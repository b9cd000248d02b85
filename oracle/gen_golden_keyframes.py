#!/usr/bin/env python3
"""Generate tests/golden/keyframes.npz by running THE REFERENCE ITSELF (read-only at /root/reference)
under Python 3.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose shims it reuses: importing
that module makes the reference's wav.py / subs.py loadable under Python 3, and its PY3_EDITS transform of
sushi.py (in memory only) gives the reference's snap_groups_to_keyframes and the rest of run()'s sequence.

What runs unmodified from the reference:
  * demux.Timecodes (demux.py:135-224), keyframes.parse_keyframes, chapters.get_xml_start_times
  * sushi.snap_groups_to_keyframes (sushi.py:218-306) and the run() sequence after demuxing (sushi.py:653-724),
    called function by function on reference-loaded WavStreams, after the PY3_EDITS transform

Two parts:
  (a) host snapping cases: seeded event lists with shifts, diffs and links, every kf_mode x {CFR, v1 with overrides,
      v2} x max_kf_distance in {0, 1, 2, 4}, plus corners; the reference's (_shift, _start_shift, _end_shift)
  (b) end-to-end scenarios x {uint8, float32}: the final (shifted_start, shifted_end) of every event; each scenario
      is asserted robust (a one-sample shift / 1e-5 diff change per search group moves no final time by more than
      one sample), and the seed is advanced until it is

Usage:  python oracle/gen_golden_keyframes.py          (writes tests/golden/keyframes.npz)
"""
import os
import sys
import zlib

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gen_golden  # noqa: E402  (puts the reference and the repository on sys.path, installs the py3 shims)
from gen_golden import OUT, _Event, load_reference_sushi, refsubs, refwav, synth, write_wav  # noqa: E402


def scxvid_text(key_frames, count, frame0_key=True):
    """An XviD 2-pass stat file as SCXvid writes it: three header lines, then one line per frame ('i' = keyframe)."""
    keys = set(key_frames)
    if not frame0_key:
        keys.discard(0)
    lines = ['# XviD 2pass stat file (core version 1.1.2)', '# Please do not modify this file', '']
    lines += ['{0} 1 0 0 0 0 0 0'.format('i' if f in keys else 'p') for f in range(count)]
    return '\n'.join(lines) + '\n'


def v1_text(default, overrides):
    return '# timecode format v1\nAssume {0:.6f}\n'.format(default) + ''.join(
        '{0},{1},{2:.6f}\n'.format(a, b, f) for a, b, f in overrides)


def v2_text(frame_times):
    return '# timecode format v2\n' + ''.join('{0:.3f}\n'.format(t * 1000.0) for t in frame_times)


def vfr_times(count, segments):
    """Frame start times for `count` frames; segments [(first_frame, fps), ...]."""
    times, t = [], 0.0
    for f in range(count):
        fps = [r for a, r in segments if a <= f][-1]
        times.append(t)
        t += 1.0 / fps
    return times


def _text_array(text):
    return np.frombuffer(text.encode('utf-8'), np.uint8)


def _load_side(kind, value, tmp):
    """(timecodes object) via the reference: a CFR rate or a timecodes text written to a file."""
    import demux as refdemux
    if kind == 'fps':
        return refdemux.Timecodes.cfr(value)
    with open(tmp, 'w') as f:
        f.write(value)
    return refdemux.Timecodes.from_file(tmp)


def _ref_keytimes(text, tc, tmp):
    import keyframes as refkeyframes
    with open(tmp, 'w') as f:
        f.write(text)
    return [tc.get_frame_time(f) for f in refkeyframes.parse_keyframes(tmp)]


def _nearest_frame(tc, t, count):
    times = [tc.get_frame_time(f) for f in range(count)]
    return int(np.argmin(np.abs(np.array(times) - t)))


def _host_timing(kind, rng, count):
    """(src side, dst side) as ('fps', rate) or ('text', timecodes text) for one host snapping case."""
    if kind == 'cfr':
        return ('fps', 23.976), ('fps', float(rng.choice([23.976, 25.0])))
    if kind == 'v1':
        a = int(rng.integers(100, 400))
        return (('text', v1_text(23.976, [(0, a, 29.97), (a + 300, a + 500, 59.94)])),
                ('text', v1_text(23.976, [(int(rng.integers(0, 50)), a + 100, 29.97)])))
    # v2 lists that stop before the timeline does: past their end the frame size is 0
    src = vfr_times(int(count * 0.8), [(0, 24000 / 1001.0), (300, 30000 / 1001.0), (700, 24000 / 1001.0)])
    dst = vfr_times(int(count * 0.85), [(0, 24000 / 1001.0), (500, 30000 / 1001.0)])
    return ('text', v2_text(src)), ('text', v2_text(dst))


def _host_case(rng, kind, dur=60.0):
    """Seeded events (starts near source keyframes, typesetting clusters), shifts, diffs, links, keyframe files."""
    count = int(dur * 24) + 200
    (sk, sv), (dk, dv) = _host_timing(kind, rng, count)
    tmp = '/tmp/_golden_side.txt'
    src_tc, dst_tc = _load_side(sk, sv, tmp), _load_side(dk, dv, tmp)
    frames, f = [], 0
    while f < count - 1:
        frames.append(f)
        f += int(rng.integers(20, 110))
    shift = float(rng.uniform(-3.0, 3.0))
    dst_frames = set()
    for fr in frames:
        u = rng.random()
        if u < 0.08:
            continue                                              # no matching keyframe at all
        frame = src_tc.get_frame_size(src_tc.get_frame_time(fr))
        off = rng.uniform(-1.3, 1.3) if u < 0.85 else rng.choice([-1, 1]) * rng.uniform(2.5, 5.0)
        t = src_tc.get_frame_time(fr) + shift + off * (frame or 1 / 24.0)
        if t > 0:
            dst_frames.add(_nearest_frame(dst_tc, t, count + 200))
    src_kf = scxvid_text(frames, count, frame0_key=bool(rng.random() < 0.5))
    dst_kf = scxvid_text(sorted(dst_frames), count + 200, frame0_key=bool(rng.random() < 0.5))
    src_keytimes = [src_tc.get_frame_time(x) for x in frames]
    ev = []
    t = 0.5
    while t < dur - 3:
        if rng.random() < 0.3:                                    # a typesetting cluster
            for _ in range(int(rng.integers(1, 4))):
                a = t + rng.uniform(0.0, 0.3)
                ev.append((a, a + rng.uniform(0.05, 0.4)))
                t = ev[-1][1]
            t += rng.uniform(0.3, 1.0)
            continue
        k = int(np.searchsorted(src_keytimes, t))
        if k >= len(src_keytimes) - 2:
            a = t                                                 # past the last keyframe
            b = a + rng.uniform(0.6, 3.0)
        else:
            frame = src_tc.get_frame_size(src_keytimes[k]) or 1 / 24.0
            a = src_keytimes[k] + rng.choice([0.0, 0.0, rng.uniform(-0.5, 0.5), rng.uniform(-2.5, 2.5)]) * frame
            b = src_keytimes[min(k + int(rng.integers(1, 3)), len(src_keytimes) - 1)] - frame * rng.choice([1.0, 0.0, 0.4])
            if b <= a + 0.5:
                b = a + rng.uniform(0.6, 2.0)
        ev.append((a, b))
        t = max(b, a) + rng.uniform(0.05, 1.5)
    ev.sort()
    n = len(ev)
    cuts = sorted(set(rng.integers(1, n, int(rng.integers(0, 3))).tolist()))
    bounds = [0] + cuts + [n]
    shifts = np.empty(n)
    for a, b in zip(bounds[:-1], bounds[1:]):
        shifts[a:b] = shift + rng.normal(0, 0.004)
    diffs = rng.uniform(0.0, 0.3, n)
    links = np.full(n, -1, np.int64)
    for i in range(n):
        if rng.random() < 0.12:
            j = int(rng.integers(0, n))
            if j != i and links[j] < 0:
                links[i] = j
                shifts[i] = shift + 7.0                          # replaced by the parent's shift when resolved
    chapters = [0.0] + sorted(rng.uniform(5, dur - 5, int(rng.integers(1, 4))).tolist()) if rng.random() < 0.4 else []
    return dict(events=np.array([[a, b, s, d] for (a, b), s, d in zip(ev, shifts, diffs)]), links=links,
                groups=np.array(list(zip(bounds[:-1], bounds[1:])), np.int64), chapters=np.array(chapters, np.float64),
                src=(sk, sv), dst=(dk, dv), src_kf=src_kf, dst_kf=dst_kf)


def _tie_case():
    """CFR 32 fps (frame 1/32 s, exact in binary): one typesetting group whose keyframe corrections are +1 and
    -1 frame, so both are exactly as far from their mean; the start correction must win."""
    src_frames = [0, 64, 81, 200, 300]
    dst_frames = [0, 97, 112, 250]
    ev = np.array([[2.0, 2.25, 1.0, 0.1], [2.3, 2.5, 1.0, 0.1], [6.0, 8.0, 1.0, 0.1]])
    return dict(events=ev, links=np.full(3, -1, np.int64), groups=np.array([[0, 2], [2, 3]], np.int64),
                chapters=np.array([], np.float64), src=('fps', 32.0), dst=('fps', 32.0),
                src_kf=scxvid_text(src_frames, 400), dst_kf=scxvid_text(dst_frames, 400))


def _single_kf_case():
    ev = np.array([[0.03, 1.2, 0.02, 0.1], [0.6, 0.8, 0.02, 0.1], [3.0, 4.5, 0.02, 0.2]])
    return dict(events=ev, links=np.array([-1, -1, 0]), groups=np.array([[0, 3]], np.int64),
                chapters=np.array([], np.float64), src=('fps', 23.976), dst=('fps', 23.976),
                src_kf=scxvid_text([], 200), dst_kf=scxvid_text([0], 200))


class _CountingEvent(_Event):
    """Reference event that counts which correction branch touched it (coverage of the golden cases)."""
    counts = {'adjust_shift': 0, 'additional': 0}

    def adjust_shift(self, value):
        _CountingEvent.counts['adjust_shift'] += 1
        super().adjust_shift(value)

    def adjust_additional_shifts(self, start_shift, end_shift):
        if start_shift or end_shift:
            _CountingEvent.counts['additional'] += 1
        super().adjust_additional_shifts(start_shift, end_shift)


def _ref_snap_case(sushi, case, mode, max_kf_distance, mtd=1001.0 / 24000.0 * 10):
    """Resolve links, then snap per group: sushi.py:706-711 on a host event list."""
    tmp = '/tmp/_golden_side.txt'
    src_tc, dst_tc = _load_side(*case['src'], tmp), _load_side(*case['dst'], tmp)
    src_keytimes, dst_keytimes = _ref_keytimes(case['src_kf'], src_tc, tmp), _ref_keytimes(case['dst_kf'], dst_tc, tmp)
    events = []
    for i, (a, b, s, d) in enumerate(case['events']):
        e = _CountingEvent(i, float(a), float(b), '')
        e._shift, e._diff = float(s), float(d)
        events.append(e)
    for i, j in enumerate(case['links']):
        if j >= 0:
            events[i].link_event(events[j])
    for e in (x for x in events if x.linked):
        e.resolve_link()
    for a, b in case['groups']:
        sushi.snap_groups_to_keyframes(events[a:b], list(case['chapters']), mtd, mtd, src_keytimes, dst_keytimes,
                                       src_tc, dst_tc, max_kf_distance, mode)
    return np.array([[e._shift, e._start_shift, e._end_shift] for e in events]), (src_keytimes, dst_keytimes, src_tc, dst_tc)


def _store_side(out, key, side):
    kind, value = side
    out[key + '_fps'] = np.array([value if kind == 'fps' else 0.0])
    out[key + '_tc'] = _text_array(value if kind == 'text' else '')


E2E_SCENARIOS = [
    # (a) ASS, constant shift, 23.976 both sides, grouping, kf_mode all, typesetting clusters
    dict(name='ass_const', script='.ass', dur=60.0, seed=61, shift=[(0.0, 1.52)], src=('fps', 23.976),
         dst=('fps', 23.976), chapters=None, grouping=True, kf_mode='all'),
    # (b) shift jump at a chapter boundary: XML chapters, source v2 timecodes, destination v1 with overrides
    dict(name='chapter_jump', script='.ass', dur=80.0, seed=62, shift=[(0.0, 0.75), (40.0, -1.25)], src=('v2', None),
         dst=('v1', None), chapters=[0.0, 40.0], grouping=True, kf_mode='shift'),
    # (c) no grouping, kf_mode snap, SRT, 25 fps source against 23.976 destination
    dict(name='srt_snap', script='.srt', dur=60.0, seed=63, shift=[(0.0, 2.0)], src=('fps', 25.0),
         dst=('fps', 23.976), chapters=None, grouping=False, kf_mode='snap'),
]


def _e2e_side(kind, count):
    if kind[0] == 'fps':
        return kind
    if kind[0] == 'v2':
        return ('text', v2_text(vfr_times(count, [(0, 24000 / 1001.0), (900, 30000 / 1001.0), (1300, 24000 / 1001.0)])))
    return ('text', v1_text(23.976, [(0, 240, 23.976), (600, 899, 29.97), (1500, 1599, 59.94)]))


def _e2e_inputs(sc, seed):
    """Events, script text and side files of one end-to-end scenario (seeded)."""
    from sushi_b200.common import format_time
    from sushi_b200.script import format_srt_time
    rng = np.random.default_rng(seed)
    dur = sc['dur']
    count = int(dur * 30) + 100
    tmp = '/tmp/_golden_side.txt'
    src_side, dst_side = _e2e_side(sc['src'], count), _e2e_side(sc['dst'], count + 200)
    src_tc, dst_tc = _load_side(*src_side, tmp), _load_side(*dst_side, tmp)
    shift_at = lambda t: [s for a, s in sc['shift'] if a <= t][-1]
    frames, f = [], 0
    while src_tc.get_frame_time(f) < dur:
        frames.append(f)
        f += int(rng.integers(20, 60))
    src_keytimes = [src_tc.get_frame_time(x) for x in frames]
    dst_frames = set()
    for t in src_keytimes:
        u = rng.random()
        if u < 0.06:
            continue
        frame = dst_tc.get_frame_size(t + shift_at(t))
        off = rng.uniform(-0.45, 0.45) if u < 0.88 else rng.choice([-1, 1]) * rng.uniform(3.0, 6.0)   # some out of reach
        if t + shift_at(t) + off * frame > 0:
            dst_frames.add(_nearest_frame(dst_tc, t + shift_at(t) + off * frame, count + 200))
    bounds = [a for a, _ in sc['shift'][1:]] + (sc['chapters'] or [])[1:]
    ev, k = [], 1
    while k < len(src_keytimes) - 2 and src_keytimes[k] < dur - 10:
        a = src_keytimes[k] + rng.choice([0.0, 0.0, rng.uniform(-0.3, 0.3) / 24.0])
        if rng.random() < 0.25:                                 # a typesetting cluster
            for _ in range(int(rng.integers(2, 4))):
                ev.append((a, a + rng.uniform(0.25, 0.38)))
                a = ev[-1][1] + rng.uniform(0.02, 0.1)
        else:
            j = k + int(rng.integers(1, 3))
            ev.append((a, src_keytimes[j] - rng.choice([0.0, 1 / 24.0])))
        k += int(rng.integers(1, 3))
        # nothing straddles the shift jump / chapter start: lines there cannot carry one shift
        while any(ev[-1][0] - 1.0 < x < ev[-1][1] + 1.0 for x in bounds):
            ev.pop()
            k += 1
            if not ev:
                break
        while k < len(src_keytimes) and ev and src_keytimes[k] <= ev[-1][1] + 0.2:
            k += 1
    ev = [(a, b) for a, b in ev if a > 1.0]
    if sc['script'] == '.ass':
        ev = [(round(a * 100) / 100, round(b * 100) / 100) for a, b in ev]
        from sushi_b200.script import AssScript
        lines = ['[Script Info]', 'ScriptType: v4.00+', '', '[V4+ Styles]', AssScript.STYLES_FORMAT,
                 'Style: Default,Arial,20,&H00FFFFFF,&H000000FF,&H00000000,&H00000000,0,0,0,0,100,100,0,0,1,2,2,2,10,10,10,1',
                 '', '[Events]', AssScript.EVENTS_FORMAT]
        lines += ['Dialogue: 0,{0},{1},Default,,0,0,0,,line {2}'.format(format_time(a), format_time(b), i)
                  for i, (a, b) in enumerate(ev)]
        text = '\n'.join(lines) + '\n'
    else:
        ev = [(round(a * 1000) / 1000, round(b * 1000) / 1000) for a, b in ev]
        text = '\n\n'.join('{0}\n{1} --> {2}\nline {0}'.format(i + 1, format_srt_time(a), format_srt_time(b))
                           for i, (a, b) in enumerate(ev)) + '\n'
    files = {'src_kf': scxvid_text(frames, count), 'dst_kf': scxvid_text(sorted(dst_frames), count + 200),
             'script': text}
    for key, side in (('src_tc', src_side), ('dst_tc', dst_side)):
        if side[0] == 'text':
            files[key] = side[1]
    if sc['chapters']:
        files['chapters'] = ('<?xml version="1.0"?>\n<Chapters>\n  <EditionEntry>\n' + ''.join(
            '    <ChapterAtom>\n      <ChapterTimeStart>{0:02d}:{1:02d}:{2:012.9f}</ChapterTimeStart>\n'
            '    </ChapterAtom>\n'.format(int(t // 3600), int(t // 60 % 60), t % 60) for t in sc['chapters'])
            + '  </EditionEntry>\n</Chapters>\n')
    return files, len(ev)


def _e2e_reference(sushi, sc, seed, files, st, tmpdir, perturbations=()):
    """sushi.py:653-724 after demuxing, function by function, on reference-loaded WavStreams.  Returns the final
    (shifted_start, shifted_end) per event in script order for the unperturbed run and for every perturbation
    (signs per search group applied to the shifts and diffs calculate_shifts left)."""
    import chapters as refchapters
    import demux as refdemux
    import keyframes as refkeyframes
    paths = {}
    for key, text in files.items():
        paths[key] = os.path.join(tmpdir, key + {'script': sc['script'], 'chapters': '.xml'}.get(key, '.txt'))
        with open(paths[key], 'w') as f:
            f.write(text)
    src_pcm, dst_pcm = synth.make_pair(sc['dur'], seed, sc['shift'] if len(sc['shift']) > 1 else sc['shift'][0][1])
    write_wav(os.path.join(tmpdir, 'src.wav'), src_pcm, 12000, 1)
    write_wav(os.path.join(tmpdir, 'dst.wav'), dst_pcm, 12000, 1)
    mtd = 1001.0 / 24000.0 * 10
    chapter_times = refchapters.get_xml_start_times(paths['chapters']) if sc['grouping'] and sc['chapters'] else []

    src_timecodes = refdemux.Timecodes.cfr(sc['src'][1]) if sc['src'][0] == 'fps' else refdemux.Timecodes.from_file(paths['src_tc'])
    src_keytimes = [src_timecodes.get_frame_time(f) for f in refkeyframes.parse_keyframes(paths['src_kf'])]
    dst_timecodes = refdemux.Timecodes.cfr(sc['dst'][1]) if sc['dst'][0] == 'fps' else refdemux.Timecodes.from_file(paths['dst_tc'])
    dst_keytimes = [dst_timecodes.get_frame_time(f) for f in refkeyframes.parse_keyframes(paths['dst_kf'])]
    script = (refsubs.AssScript if sc['script'] == '.ass' else refsubs.SrtScript).from_file(paths['script'])
    script.sort_by_time()
    src_stream = refwav.WavStream(os.path.join(tmpdir, 'src.wav'), sample_rate=12000, sample_type=st)
    dst_stream = refwav.WavStream(os.path.join(tmpdir, 'dst.wav'), sample_rate=12000, sample_type=st)
    search_groups = sushi.prepare_search_groups(script.events, source_duration=src_stream.duration_seconds,
                                                chapter_times=chapter_times, max_ts_duration=mtd, max_ts_distance=mtd)
    sushi.calculate_shifts(src_stream, dst_stream, search_groups, normal_window=10, max_window=30,
                           rewind_thresh=5 if sc['grouping'] else 0)
    events = script.events
    state = [(e._shift, e._diff, e._linked_event, e._start_shift, e._end_shift) for e in events]

    def post(signs):
        for e, s in zip(events, state):
            e._shift, e._diff, e._linked_event, e._start_shift, e._end_shift = s
        if signs is not None:
            for g, (ss, ds) in zip(search_groups, signs):
                for e in g:
                    if not e.linked:
                        e._shift += ss / 12000.0
                        e._diff = np.float32(e._diff + ds * 1e-5)
        if sc['grouping']:
            if chapter_times:
                groups = sushi.groups_from_chapters(events, chapter_times)
                for g in groups:
                    sushi.fix_near_borders(g)
                    sushi.smooth_events([x for x in g if not x.linked], 3)
                groups = sushi.split_broken_groups(groups)
            else:
                sushi.fix_near_borders(events)
                sushi.smooth_events([x for x in events if not x.linked], 3)
                groups = sushi.detect_groups(events)
            for g in groups:
                sushi.average_shifts(g)
            for e in (x for x in events if x.linked):
                e.resolve_link()
            for g in groups:
                sushi.snap_groups_to_keyframes(g, chapter_times, mtd, mtd, src_keytimes, dst_keytimes, src_timecodes,
                                               dst_timecodes, 2, sc['kf_mode'])
        else:
            sushi.fix_near_borders(events)
            for e in (x for x in events if x.linked):
                e.resolve_link()
            sushi.snap_groups_to_keyframes(events, chapter_times, mtd, mtd, src_keytimes, dst_keytimes, src_timecodes,
                                           dst_timecodes, 2, sc['kf_mode'])
        return np.array([[e.shifted_start, e.shifted_end] for e in events])

    base = post(None)
    moved = [post(p(len(search_groups))) for p in perturbations]
    index = np.array([e.source_index for e in events], np.int64)
    return base, moved, index, (src_pcm, dst_pcm), [[e.shift for e in g] for g in search_groups]


def _perturbation_patterns():
    pats = [lambda n, a=a, b=b: [(a, b)] * n for a in (1, -1) for b in (1, -1)]
    for k in range(4):
        pats.append(lambda n, k=k: [tuple(x) for x in np.random.default_rng(900 + k).choice([-1, 1], (n, 2))])
    return pats


def gen_keyframes():
    """Keyframe golden: (a) host snapping cases through the reference's snap_groups_to_keyframes, (b) end-to-end
    scenarios through the reference's run() sequence after demuxing, each asserted robust to the matcher's tolerance."""
    import logging
    import tempfile
    sushi = load_reference_sushi()
    logging.disable(logging.CRITICAL)
    out = {}
    # (a) host cases: every kf_mode x timecode kind x max_kf_distance, plus corners
    names = []
    cases = []
    rng = np.random.default_rng(77)
    for kind in ('cfr', 'v1', 'v2'):
        for mode in ('all', 'shift', 'snap'):
            for mkd in (0, 1, 2, 4):
                cases.append(('{0}_{1}_{2}'.format(kind, mode, mkd), _host_case(rng, kind), mode, mkd))
    noreach = _host_case(np.random.default_rng(5), 'cfr')
    noreach['dst_kf'] = scxvid_text([0], 3000)                  # nothing in reach: interpolate_nones gives []
    cases.append(('noreach_all', noreach, 'all', 2))
    cases.append(('single_kf_all', _single_kf_case(), 'all', 2))
    cases.append(('tie_shift', _tie_case(), 'shift', 2))
    cases.append(('tie_all', _tie_case(), 'all', 2))
    _CountingEvent.counts.update(adjust_shift=0, additional=0)
    interpolated = []
    real_interpolate = sushi.interpolate_nones
    sushi.interpolate_nones = lambda data, points: interpolated.append(real_interpolate(data, points)) or interpolated[-1]
    for name, case, mode, mkd in cases:
        del interpolated[:]
        res, (sk, dk, stc, dtc) = _ref_snap_case(sushi, case, mode, mkd)
        if name == 'noreach_all':
            assert interpolated == [[]], interpolated           # step 1 skipped: no keyframe pair in reach
        if name.startswith('tie'):
            g = [_Event(i, float(a), float(b), '') for i, (a, b, s, d) in enumerate(case['events'][:2])]
            for e in g:
                e._shift = 1.0
            s, e = sushi.find_keyframe_shift(g, sk, dk, stc, dtc, 2)
            assert s != e and abs(s - np.mean([s, e])) == abs(e - np.mean([s, e])), (s, e)
            assert res[0, 0] == 1.0 + s, res                      # the start correction won the tie
        p = 'a_{0}_'.format(name)
        names.append(name)
        out[p + 'events'] = case['events']
        out[p + 'links'] = np.asarray(case['links'], np.int64)
        out[p + 'groups'] = case['groups']
        out[p + 'chapters'] = case['chapters']
        out[p + 'params'] = np.array([mkd], np.float64)
        out[p + 'mode'] = _text_array(mode)
        out[p + 'src_kf'] = _text_array(case['src_kf'])
        out[p + 'dst_kf'] = _text_array(case['dst_kf'])
        _store_side(out, p + 'src', case['src'])
        _store_side(out, p + 'dst', case['dst'])
        out[p + 'result'] = res
        moved = np.abs(res[:, 1:]).sum() + np.abs(res[:, 0] - [float(case['events'][i if j < 0 else j, 2])
                                                                for i, j in enumerate(case['links'])]).sum()
        print('host', name, 'events', len(res), 'moved', round(float(moved), 4))
    sushi.interpolate_nones = real_interpolate
    assert _CountingEvent.counts['adjust_shift'] > 0 and _CountingEvent.counts['additional'] > 0, _CountingEvent.counts
    out['a_names'] = _text_array(','.join(names))

    # (b) end to end, robust to one sample of shift and 1e-5 of diff per search group
    tol = 1.0 / 12000 + 1e-9
    for sc in E2E_SCENARIOS:
        for attempt in range(20):
            seed = sc['seed'] + 100 * attempt
            files, n = _e2e_inputs(sc, seed)
            ok, runs = True, {}
            for st in ('uint8', 'float32'):
                with tempfile.TemporaryDirectory() as d:
                    base, moved, index, pcm, sg = _e2e_reference(sushi, sc, seed, files, st, d, _perturbation_patterns())
                worst = max(np.abs(m - base).max() for m in moved)
                runs[st] = (base, index, pcm)
                if worst > tol:
                    ok = False
                    print('e2e', sc['name'], 'seed', seed, st, 'not robust (moves by {0:.3g} s)'.format(worst))
                    break
            if ok:
                break
        assert ok, sc['name']
        p = 'b_{0}_'.format(sc['name'])
        spec = dict(sc, seed=seed)
        out[p + 'spec'] = _text_array(repr(spec))
        for key, text in files.items():
            out[p + key] = _text_array(text)
        src_pcm, dst_pcm = runs['uint8'][2]
        out[p + 'pcm_crc'] = np.array([zlib.crc32(src_pcm.tobytes()), zlib.crc32(dst_pcm.tobytes())], np.int64)
        for st in ('uint8', 'float32'):
            base, index, _ = runs[st]
            out[p + st + '_times'] = base
            out[p + st + '_index'] = index
        print('e2e', sc['name'], 'seed', seed, 'events', n)
    out['b_names'] = _text_array(','.join(sc['name'] for sc in E2E_SCENARIOS))
    np.savez_compressed(os.path.join(OUT, 'keyframes.npz'), **out)
    print('keyframes.npz:', len(names), 'host cases,', len(E2E_SCENARIOS), 'scenarios x 2 sample types')


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    gen_keyframes()
