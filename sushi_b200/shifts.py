"""The shift solver that drives the matcher: a behavioural mirror of the reference's
calculate_shifts (sushi.py:400-508) with the same signature, the same constants and the same
log lines, so the grouping heuristics before and after it see identical results.

Differences are purely in how the matcher is called: the reference issues 1 + 3 (+ 3) dependent
find_substream calls per search group; here the three probes of a check (whole group, left half,
right half -- sushi.py:445-452) go to the GPU as one batch when the stream supports it
(WavStream.find_substream_many), and the fast-path searches of the coming groups are precomputed
48 at a time as whole curves (WavStream.speculate_fast_path) from which each call is answered
exactly.  Streams are duck-typed: anything with get_substream /
find_substream / duration_seconds / sample_rate works (the tests also run this solver on the
CPU oracle's streams and compare with the reference's golden results).

The solver itself is a generator (_solve) that yields the matcher work it needs and receives the
answers: a probe triple, or one fast-path search with the speculation that precedes it.
calculate_shifts answers each request with the stream's own methods, one at a time;
calculate_shifts_many runs many episodes in lockstep and answers every request that is ready in
one round -- one multi-stream launch for all probes, one for all speculations -- so the number of
GPU round trips is the maximum over the episodes instead of their sum.
"""
import logging
from itertools import chain

from .common import format_time
from .grouping import ALLOWED_ERROR

SMALL_WINDOW = 1.5          # sushi.py:410


class _GroupState(object):
    __slots__ = ('start_time', 'end_time', 'shift', 'diff')

    def __init__(self, group, shift=None, diff=None):
        self.start_time, self.end_time = group[0].start, group[-1].end
        self.shift, self.diff = shift, diff

    def log(self):
        logging.info('{0}-{1}: shift: {2:0.10f}, diff: {3:0.10f}'.format(
            format_time(self.start_time), format_time(self.end_time), self.shift, self.diff))


# Requests the solver yields (answers in brackets):
#   ('probe', [q_whole, q_left, q_right])    the three searches of a check  [three (diff, time)]
#   ('find', q, spec)                        one fast-path search, spec = (groups_list, idx, anchor, window) of the
#                                            speculation to run first, or None  [(diff, time)]
# with q = (pattern, center, window), the arguments of find_substream.
def _answer_alone(src_stream, dst_stream, request):
    """One request through the stream's own methods, exactly the calls the sequential solver makes."""
    if request[0] == 'probe':
        many = getattr(dst_stream, 'find_substream_many', None)
        return many(request[1]) if many is not None else [dst_stream.find_substream(*q) for q in request[1]]
    if request[2] is not None:
        dst_stream.speculate_fast_path(src_stream, *request[2])
    return dst_stream.find_substream(*request[1])


def _probe_triple(audio, left, right, right_offset, center, window):
    """Whole / left-half / right-half search around `center` (sushi.py:450-453)."""
    queries = [(audio, center, window), (left, center, window), (right, center + right_offset, window)]
    results = yield ('probe', queries)
    diff, whole_time = results[0]
    left_time = results[1][1]
    right_time = results[2][1] - right_offset
    agreed = abs(left_time - right_time) <= ALLOWED_ERROR and abs(whole_time - left_time) <= ALLOWED_ERROR
    return diff, whole_time, left_time, right_time, agreed


def calculate_shifts(src_stream, dst_stream, groups_list, normal_window, max_window, rewind_thresh,
                     speculative=True):
    solver = _solve(src_stream, dst_stream, groups_list, normal_window, max_window, rewind_thresh, speculative)
    answer = None
    while True:
        try:
            request = solver.send(answer)
        except StopIteration:
            return
        answer = _answer_alone(src_stream, dst_stream, request)


def calculate_shifts_many(jobs, normal_window, max_window, rewind_thresh, speculative=True, executor=None):
    """calculate_shifts over many jobs [(src_stream, dst_stream, groups_list), ...] in lockstep: every job runs on the
    host until it needs the matcher, then one round answers the requests of all of them, and every job resumes.
    Per-event results equal running calculate_shifts on each job alone (a value depends only on (template, absolute
    position), so sharing a launch changes none).  `executor(batch)` answers a round: batch = [(src, dst, request)],
    returns the answers in order; the default sends all searches out as one sb_find_multi and all speculations as one
    sb_match_curves_multi.  Returns the number of rounds."""
    executor = executor or execute_round
    solvers = [_solve(src, dst, groups, normal_window, max_window, rewind_thresh, speculative) for src, dst, groups in jobs]
    waiting = {}
    for j, solver in enumerate(solvers):
        try:
            waiting[j] = next(solver)
        except StopIteration:
            pass
    rounds = 0
    while waiting:
        order = sorted(waiting)
        answers = executor([(jobs[j][0], jobs[j][1], waiting[j]) for j in order])
        rounds += 1
        for j, answer in zip(order, answers):
            try:
                waiting[j] = solvers[j].send(answer)
            except StopIteration:
                del waiting[j]
    return rounds


def execute_round(batch):
    """The default executor of calculate_shifts_many: the speculations of the round from one sb_match_curves_multi
    (each destination's curve cache filled as speculate_fast_path fills it), then every search of the round -- probe
    triples and fast-path searches -- from one sb_find_multi; searches a cached curve answers stay on the host.
    Streams without the multi-stream surface get their requests answered one by one."""
    from .wavstream import WavStream, find_substreams, speculate_fast_path_many
    gpu = [isinstance(dst, WavStream) for _, dst, _ in batch]
    speculations = [(dst, src) + tuple(req[2]) for (src, dst, req), g in zip(batch, gpu) if g and req[0] == 'find' and req[2]]
    if speculations:
        speculate_fast_path_many(speculations)
    searches = []
    for (src, dst, req), g in zip(batch, gpu):
        if g:
            searches += [(dst,) + tuple(q) for q in (req[1] if req[0] == 'probe' else [req[1]])]
    found = iter(find_substreams(searches))
    answers = []
    for (src, dst, req), g in zip(batch, gpu):
        if not g:
            answers.append(_answer_alone(src, dst, req))
        elif req[0] == 'probe':
            answers.append([next(found) for _ in req[1]])
        else:
            answers.append(next(found))
    return answers


def _solve(src_stream, dst_stream, groups_list, normal_window, max_window, rewind_thresh, speculative):
    committed, pending = [], []
    # streams that can precompute the coming fast-path searches in one launch expose this hook; the
    # results they then return are the ones a live call would return (see WavStream.speculate_fast_path)
    speculate = getattr(dst_stream, 'speculate_fast_path', None) if speculative else None
    window = normal_window
    idx = 0
    while idx < len(groups_list):
        group = groups_list[idx]
        origin = group[0].start
        audio = src_stream.get_substream(group[0].start, group[-1].end)
        state = _GroupState(group)
        anchor = committed[-1].shift if committed else 0
        diff = found = None

        if not pending:
            if origin + anchor > dst_stream.duration_seconds:
                # past the end of the destination audio: so is everything after it (sushi.py:424-429)
                for rest in groups_list[idx:]:
                    committed.append(_GroupState(rest))
                    logging.info('{0}-{1}: outside of audio range'.format(format_time(rest[0].start), format_time(rest[-1].end)))
                break
            if SMALL_WINDOW < window:
                spec = (groups_list, idx, anchor, SMALL_WINDOW) if speculate is not None else None
                diff, found = yield ('find', (audio, origin + anchor, SMALL_WINDOW), spec)
            if found is not None and abs((found - origin) - anchor) <= ALLOWED_ERROR:
                # the shift did not move: commit straight away (sushi.py:434-443)
                state.shift, state.diff = found - origin, diff
                committed.append(state)
                state.log()
                if window != normal_window:
                    logging.info('Going back to window {0} from {1}'.format(normal_window, window))
                    window = normal_window
                idx += 1
                continue

        half = len(audio[0]) // 2
        left, right = audio[:, :half], audio[:, half:]
        right_offset = half / float(src_stream.sample_rate)
        agreed = False
        for center_shift, allowed in (
                (anchor, True),
                (pending[-1].shift if pending else None, bool(pending))):
            if agreed or not allowed or center_shift is None:
                continue
            if not origin + center_shift < dst_stream.duration_seconds:
                continue
            diff, found, left_time, right_time, agreed = yield from _probe_triple(
                audio, left, right, right_offset, origin + center_shift, window)
            logging.debug('{0}-{1}: shift: {2:0.5f} [{3:0.5f}, {4:0.5f}], search offset: {5:0.6f}'.format(
                format_time(state.start_time), format_time(state.end_time), found - origin,
                left_time - origin, right_time - origin, center_shift))

        shift = found - origin
        if not agreed:
            # not back on track: park the group; after rewind_thresh of them widen the window and
            # redo everything since the last commit (sushi.py:468-479)
            state.shift, state.diff = shift, diff
            pending.append(state)
            idx += 1
            if rewind_thresh == len(pending) and window < max_window:
                logging.warning('Detected possibly broken segment starting at {0}, increasing the window from {1} to {2}'.format(
                    format_time(pending[0].start_time), window, max_window))
                window = max_window
                idx = len(committed)
                del pending[:]
            continue

        if pending:
            logging.warning('Events from {0} to {1} will most likely be broken!'.format(
                format_time(pending[0].start_time), format_time(pending[-1].end_time)))
        pending.append(state)
        for s in pending:                       # the whole parked run takes the re-acquired shift
            s.shift, s.diff = shift, diff
            s.log()
        committed.extend(pending)
        del pending[:]
        idx += 1

    for s in pending:
        s.log()

    for idx, (group, state) in enumerate(zip(groups_list, chain(committed, pending))):
        if state.shift is None:
            for earlier in reversed(groups_list[:idx]):
                target = next((e for e in reversed(earlier) if not e.linked), None)
                if target:
                    for e in group:
                        e.link_event(target)
                    break
        else:
            for e in group:
                e.set_shift(state.shift, state.diff)
