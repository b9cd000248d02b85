"""The grouping heuristics that sit either side of the matcher (reference sushi.py:67-397).
They decide which events are correlated (search groups), post-process the (shift, diff) pairs the
matcher returns and, when keyframes are given, correct the result against video keyframes.
Behaviour follows the reference function for function; the reference's own unit tests for them
(tests/main.py:34-181) are ported in tests/test_grouping.py and tests/test_timing.py.

Events are duck-typed: anything with start/end/shift/diff/linked and set_shift/link_event works
(ScriptEvent here, subs.ScriptEventBase in the reference, FakeEvent in its tests).
"""
import bisect
import logging

import numpy as np

from .common import SushiError, format_time

ALLOWED_ERROR = 0.01       # sushi.py:39
MAX_GROUP_STD = 0.025      # sushi.py:40


def interpolate_nones(data, points):
    """Fill None entries of `data` by linear interpolation over `points`, edges held (sushi.py:71-93)."""
    data = data if isinstance(data, (list, tuple, set)) else list(data)
    known = {p: v for p, v in zip(points, data) if v is not None}
    if not known:
        return []
    missing = sorted({p for p, v in zip(points, data) if v is None and p not in known})
    if not any(v is None for v in data):
        return data
    xs = sorted(known)
    filled = np.interp(missing, xs, [known[x] for x in xs]) if missing else []
    known.update(zip(missing, filled))
    return [known[p] if v is None else v for p, v in zip(points, data)]


def running_median(values, window_size):
    """Median filter whose radius shrinks towards both ends (sushi.py:97-107).  Interior points use one
    vectorised sliding-window median; the 2*half border points use their own shorter windows.  np.median
    per window (middle element, or the mean of the two middle ones) is what the reference computes."""
    if window_size % 2 != 1:
        raise SushiError('Median window size should be odd')
    half = window_size // 2
    count = len(values)
    out = [None] * count
    arr = np.asarray(values)
    numeric = arr.dtype.kind in 'fiu' and count > window_size
    if numeric:
        windows = np.lib.stride_tricks.sliding_window_view(arr, window_size)
        mid = np.median(windows, axis=1)
        for i in range(half, count - half):
            out[i] = mid[i - half]
    for i in range(count):
        if out[i] is None:
            r = min(half, i, count - i - 1)
            out[i] = np.median(values[i - r:i + r + 1])
    return out


def smooth_events(events, radius):
    if not radius:
        return
    smoothed = running_median([e.shift for e in events], radius * 2 + 1)
    for e, s in zip(events, smoothed):
        e.set_shift(s, e.diff)


def _column(events, attr):
    """One attribute of many events as an array, or None when the values are not all of one numeric
    type (then NumPy's array promotion would differ from the reference's scalar-by-scalar arithmetic
    and the callers fall back to their scalar loops).  Same-typed values keep their type: matcher
    diffs are np.float32 and are compared / divided in float32 exactly like the scalars are."""
    values = [getattr(e, attr) for e in events]
    kinds = set(map(type, values))
    if len(kinds) != 1 or not issubclass(next(iter(kinds)), (float, int, np.floating, np.integer)):
        return None
    return np.array(values)


def detect_groups(events_iter):
    """Split at every jump of more than ALLOWED_ERROR between neighbours (sushi.py:120-127).  One
    vectorised difference over the shift column gives the cut points."""
    events = events_iter if isinstance(events_iter, list) else list(events_iter)
    if not events:
        raise StopIteration      # the reference calls next() on an empty iterator here
    shifts = _column(events, 'shift')
    if shifts is None:
        cuts = [i for i in range(1, len(events)) if abs(events[i].shift - events[i - 1].shift) > ALLOWED_ERROR]
    else:
        cuts = (np.flatnonzero(np.abs(shifts[1:] - shifts[:-1]) > ALLOWED_ERROR) + 1).tolist()
    bounds = [0] + cuts + [len(events)]
    return [events[a:b] for a, b in zip(bounds[:-1], bounds[1:])]


def groups_from_chapters(events, times):
    """One group per chapter; groups made only of linked events move to their parents' groups
    (sushi.py:130-161)."""
    logging.info('Chapter start points: {0}'.format([format_time(t) for t in times]))
    bounds = iter(list(times[1:]) + [36000000000])
    limit = next(bounds)
    groups = [[]]
    for e in events:
        if e.end > limit:
            groups.append([])
            while e.end > limit:
                limit = next(bounds)
        groups[-1].append(e)
    groups = [g for g in groups if g]
    orphaned = [g for g in groups if all(e.linked for e in g)]
    if orphaned:
        for g in orphaned:
            for e in g:
                parent = e.get_link_chain_end()
                next(h for h in groups if parent in h).append(e)
            del g[:]
        groups = [g for g in groups if g]
        for g in groups:
            g.sort(key=lambda e: e.start)
    return groups


def split_broken_groups(groups):
    """Chapter groups whose shifts disagree (std > MAX_GROUP_STD) fall back to automatic grouping,
    then neighbours that agree are merged again (sushi.py:164-187)."""
    fixed = []
    any_broken = False
    for g in groups:
        std = np.std([e.shift for e in g])
        if std > MAX_GROUP_STD:
            logging.warning('Shift is not consistent between {0} and {1}, most likely chapters are wrong (std: {2}). '
                            'Switching to automatic grouping.'.format(format_time(g[0].start), format_time(g[-1].end), std))
            fixed.extend(detect_groups(g))
            any_broken = True
        else:
            fixed.append(g)
    if not any_broken:
        return fixed
    merged = [list(fixed[0])]
    for g in fixed[1:]:
        tail = merged[-1]
        if abs(tail[-1].shift - g[0].shift) >= ALLOWED_ERROR \
                or np.std([e.shift for e in g + tail]) >= MAX_GROUP_STD:
            merged.append([])
        merged[-1].extend(g)
    return merged


def fix_near_borders(events):
    """Events at either end whose diff is far from the typical one are linked to the first sane
    event inwards (sushi.py:190-215)."""
    def sweep(seq, diffs, median_diff):
        # the first event whose diff is within [0.2, 5] x the typical one ends the broken run; found
        # with one vectorised ratio test over the diff column (same float type as the scalars)
        limit = min(np.median(diffs[:10]), median_diff)
        if isinstance(diffs, np.ndarray):
            ratio = diffs / limit
            sane = np.flatnonzero((0.2 < ratio) & (ratio < 5))
            first = int(sane[0]) if sane.size else None
        else:
            first = next((i for i, d in enumerate(diffs) if 0.2 < (d / limit) < 5), None)
        if first is None:
            return 0
        for b in seq[:first]:
            b.link_event(seq[first])
        return first

    diffs = _column(events, 'diff')
    if diffs is None:
        diffs = [e.diff for e in events]
    median_diff = np.median(diffs)
    n = sweep(events, diffs, median_diff)
    if n:
        logging.info('Fixing {0} border events right after {1}'.format(n, format_time(events[0].start)))
    n = sweep(events[::-1], diffs[::-1], median_diff)
    if n:
        logging.info('Fixing {0} border events right before {1}'.format(n, format_time(events[-1].end)))


def average_shifts(events):
    """Weighted mean shift of the unlinked events, weights 1 - diff (sushi.py:309-316)."""
    events = [e for e in events if not e.linked]
    shifts, diffs = _column(events, 'shift'), _column(events, 'diff')
    if shifts is None or diffs is None:
        shifts, weights = [e.shift for e in events], [1 - e.diff for e in events]
    else:
        weights = 1 - diffs                   # elementwise in the diffs' own float type, like the scalars
    avg = np.average(shifts, weights=weights)
    for e in events:
        e.set_shift(avg, e.diff)
    return avg


def merge_short_lines_into_groups(events, chapter_times, max_ts_duration, max_ts_distance):
    """Short (typesetting) lines that follow each other closely are searched as one group; long lines
    are searched alone (sushi.py:319-349)."""
    events = events if isinstance(events, (list, tuple)) else list(events)
    bounds = iter(list(chapter_times[1:]) + [100000000])
    next_chapter = next(bounds)
    taken = set()
    groups = []
    for idx, e in enumerate(events):
        if idx in taken:
            continue
        while e.end > next_chapter:
            next_chapter = next(bounds)
        if e.duration > max_ts_duration:
            groups.append([e])
            taken.add(idx)
            continue
        group, group_end = [e], e.end
        i = idx + 1
        while i < len(events) and abs(group_end - events[i].start) < max_ts_distance:
            if events[i].end < next_chapter and events[i].duration <= max_ts_duration:
                taken.add(i)
                group.append(events[i])
                group_end = max(group_end, events[i].end)
            i += 1
        groups.append(group)
    return groups


def get_distance_to_closest_kf(timestamp, keyframes):
    """Signed distance from `timestamp` to the nearest keyframe time; ties go to the earlier one (sushi.py:218-228)."""
    idx = bisect.bisect_left(keyframes, timestamp)
    if idx == 0:
        kf = keyframes[0]
    elif idx == len(keyframes):
        kf = keyframes[-1]
    else:
        before, after = keyframes[idx - 1], keyframes[idx]
        kf = after if after - timestamp < timestamp - before else before
    return kf - timestamp


def find_keyframe_shift(group, src_keytimes, dst_keytimes, src_timecodes, dst_timecodes, max_kf_distance):
    """(start, end) corrections that put a search group's edges on the destination keyframes matching
    the source ones, None where no keyframe pair is within reach (sushi.py:231-248)."""
    def get_distance(src_distance, dst_distance, limit):
        if abs(dst_distance) > limit:
            return None
        shift = dst_distance - src_distance
        return shift if abs(shift) < limit else None

    src_start = get_distance_to_closest_kf(group[0].start, src_keytimes)
    src_end = get_distance_to_closest_kf(group[-1].end + src_timecodes.get_frame_size(group[-1].end), src_keytimes)
    dst_start = get_distance_to_closest_kf(group[0].shifted_start, dst_keytimes)
    # the frame size is looked up at the UNSHIFTED end on the destination timecodes (sushi.py:242)
    dst_end = get_distance_to_closest_kf(group[-1].shifted_end + dst_timecodes.get_frame_size(group[-1].end), dst_keytimes)
    snapping_limit_start = src_timecodes.get_frame_size(group[0].start) * max_kf_distance
    snapping_limit_end = src_timecodes.get_frame_size(group[0].end) * max_kf_distance    # group[0], not group[-1] (sushi.py:245)
    return (get_distance(src_start, dst_start, snapping_limit_start),
            get_distance(src_end, dst_end, snapping_limit_end))


def find_keyframes_distances(event, src_keytimes, dst_keytimes, timecodes, max_kf_distance):
    """Separate start / end corrections of one event when both its source and shifted times sit
    near keyframes (sushi.py:251-263)."""
    def find_keyframe_distance(src_time, dst_time):
        src = get_distance_to_closest_kf(src_time, src_keytimes)
        dst = get_distance_to_closest_kf(dst_time, dst_keytimes)
        snapping_limit = timecodes.get_frame_size(src_time) * max_kf_distance
        if abs(src) < snapping_limit and abs(dst) < snapping_limit and abs(src - dst) < snapping_limit:
            return dst - src
        return 0

    return find_keyframe_distance(event.start, event.shifted_start), find_keyframe_distance(event.end, event.shifted_end)


def snap_groups_to_keyframes(events, chapter_times, max_ts_duration, max_ts_distance, src_keytimes, dst_keytimes,
                             src_timecodes, dst_timecodes, max_kf_distance, kf_mode):
    """Keyframe correction of already shifted, unlinked events (sushi.py:266-306).  Step 1 ('shift' /
    'all') moves every search group by its keyframe correction, keeping durations; step 2 ('snap' /
    'all') moves the start and end of each group's first event onto nearby keyframes."""
    if not max_kf_distance:
        return
    groups = merge_short_lines_into_groups(events, chapter_times, max_ts_duration, max_ts_distance)

    if kf_mode == 'all' or kf_mode == 'shift':
        shifts, times = [], []
        for group in groups:
            shifts.extend(find_keyframe_shift(group, src_keytimes, dst_keytimes, src_timecodes, dst_timecodes,
                                              max_kf_distance))
            times.extend((group[0].shifted_start, group[-1].shifted_end))
        shifts = interpolate_nones(shifts, times)
        if shifts:
            mean_shift = np.mean(shifts)
            pairs = zip(*(iter(shifts),) * 2)
            logging.info('Group {0}-{1} corrected by {2}'.format(format_time(events[0].start), format_time(events[-1].end),
                                                                 mean_shift))
            for group, (start_shift, end_shift) in zip(groups, pairs):
                if abs(start_shift - end_shift) > 0.001 and len(group) > 1:
                    # on a tie min() keeps the start shift
                    actual_shift = min(start_shift, end_shift, key=lambda x: abs(x - mean_shift))
                    logging.warning('Typesetting group at {0} had different shift at start/end points ({1} and {2}). '
                                    'Shifting by {3}.'.format(format_time(group[0].start), start_shift, end_shift,
                                                              actual_shift))
                    for e in group:
                        e.adjust_shift(actual_shift)
                else:
                    for e in group:
                        e.adjust_additional_shifts(start_shift, end_shift)

    if kf_mode == 'all' or kf_mode == 'snap':
        # the reference means to leave typesetting groups alone here but its check is a no-op
        # (sushi.py:301-302): every group's first event is snapped
        for group in groups:
            start_shift, end_shift = find_keyframes_distances(group[0], src_keytimes, dst_keytimes, src_timecodes,
                                                              max_kf_distance)
            if abs(start_shift) > 0.01 or abs(end_shift) > 0.01:
                logging.info('Snapping {0} to keyframes, start time by {1}, end: {2}'.format(
                    format_time(group[0].start), start_shift, end_shift))
                group[0].adjust_additional_shifts(start_shift, end_shift)


def prepare_search_groups(events, source_duration, chapter_times, max_ts_duration, max_ts_distance):
    """Link what must not be searched (comments, zero-length lines, lines past the end of the audio,
    exact duplicates), group the rest, and link groups nested inside earlier ones (sushi.py:352-397)."""
    last_unlinked = None
    for idx, e in enumerate(events):
        if e.is_comment or (e.end == e.start and not (e.start + e.duration / 2.0) > source_duration):
            target = events[idx + 1] if idx + 1 < len(events) else last_unlinked
            if not e.is_comment:
                logging.info('{0}: skipped because zero duration'.format(format_time(e.start)))
            e.link_event(target)
            continue
        if (e.start + e.duration / 2.0) > source_duration:
            logging.info('Event time outside of audio range, ignoring: %s' % e)
            e.link_event(last_unlinked)
            continue
        twin = None
        for j in range(idx - 1, -1, -1):          # walk back while the start time is the same
            x = events[j]
            if x.start != e.start:
                break
            if not x.linked and x.end == e.end:
                twin = x
                break
        if twin is not None:
            e.link_event(twin)
        else:
            last_unlinked = e

    groups = merge_short_lines_into_groups([e for e in events if not e.linked], chapter_times,
                                           max_ts_duration, max_ts_distance)
    # a group nested inside an earlier group is linked to it (nearest such group first).  When the
    # groups are ordered by start time -- the reference assumes sorted scripts -- "nearest earlier
    # group that ends at or after this one" is a previous-greater-or-equal query: a monotonic stack
    # answers it in O(N) instead of the reference's O(N^2) scan; unsorted input takes the scan.
    kept = []
    ordered = all(groups[i][0].start <= groups[i + 1][0].start for i in range(len(groups) - 1))
    stack = []                                    # indices with strictly decreasing group end
    for idx, g in enumerate(groups):
        if ordered:
            while stack and groups[stack[-1]][-1].end < g[-1].end:
                stack.pop()
            outer = groups[stack[-1]] if stack else None
            stack.append(idx)
        else:
            outer = None
            for j in range(idx - 1, -1, -1):
                x = groups[j]
                if x[0].start <= g[0].start and x[-1].end >= g[-1].end:
                    outer = x
                    break
        if outer is None:
            kept.append(g)
        else:
            for e in g:
                e.link_event(outer[0])
    return kept
