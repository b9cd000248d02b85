"""Keyframe snapping on the host against the reference's own snap_groups_to_keyframes (golden
tests/golden/keyframes.npz, part a, from oracle/gen_golden_keyframes.py): seeded events with
shifts, diffs and links, every kf_mode x {CFR, v1 with overrides, v2} x max_kf_distance in
{0, 1, 2, 4}, and corners (nothing in reach, a single keyframe, events past the last keyframe and
past the end of a v2 list, an exact tie between start and end corrections, typesetting clusters,
chapters).  The port runs the same Python and NumPy operations in the same order, so every
(_shift, _start_shift, _end_shift) must be exactly equal."""
import os

import numpy as np
import pytest

from sushi_b200.events import ScriptEvent
from sushi_b200.grouping import snap_groups_to_keyframes
from sushi_b200.timing import load_keyframe_times

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'keyframes.npz'))
MAX_TS = 1001.0 / 24000.0 * 10


def text(key):
    return bytes(GOLDEN[key]).decode('utf-8')


CASES = text('a_names').split(',')


def keyframe_times(prefix, tmp_path):
    """Writes the case's keyframe and timecode texts to files and loads them the way the CLI does."""
    args = {}
    for side in ('src', 'dst'):
        (tmp_path / (side + '_kf.txt')).write_text(text(prefix + side + '_kf'))
        fps = float(GOLDEN[prefix + side + '_fps'][0])
        if fps:
            args[side + '_fps'] = fps
        else:
            (tmp_path / (side + '_tc.txt')).write_text(text(prefix + side + '_tc'))
            args[side + '_timecodes'] = str(tmp_path / (side + '_tc.txt'))
    return load_keyframe_times(str(tmp_path / 'src_kf.txt'), str(tmp_path / 'dst_kf.txt'), **args)


def test_golden_covers_the_matrix():
    for kind in ('cfr', 'v1', 'v2'):
        for mode in ('all', 'shift', 'snap'):
            for mkd in (0, 1, 2, 4):
                assert '{0}_{1}_{2}'.format(kind, mode, mkd) in CASES
    for corner in ('noreach_all', 'single_kf_all', 'tie_shift', 'tie_all'):
        assert corner in CASES


@pytest.mark.parametrize('name', CASES)
def test_snapping_equals_reference(name, tmp_path):
    p = 'a_{0}_'.format(name)
    kt = keyframe_times(p, tmp_path)
    events = []
    for i, (a, b, s, d) in enumerate(GOLDEN[p + 'events']):
        e = ScriptEvent(i, float(a), float(b))
        e._shift, e._diff = float(s), float(d)
        events.append(e)
    for i, j in enumerate(GOLDEN[p + 'links']):
        if j >= 0:
            events[i].link_event(events[int(j)])
    for e in events:                                    # run()'s order: resolve links, then snap per group
        if e.linked:
            e.resolve_link()
    chapters = [float(x) for x in GOLDEN[p + 'chapters']]
    mkd = float(GOLDEN[p + 'params'][0])
    mode = text(p + 'mode')
    for a, b in GOLDEN[p + 'groups']:
        snap_groups_to_keyframes(events[a:b], chapters, MAX_TS, MAX_TS, kt.src_keytimes, kt.dst_keytimes,
                                 kt.src_timecodes, kt.dst_timecodes, mkd, mode)
    got = [(e._shift, e._start_shift, e._end_shift) for e in events]
    want = [tuple(r) for r in GOLDEN[p + 'result']]
    assert got == want


def test_tie_keeps_the_start_correction(tmp_path):
    """One typesetting group whose start and end corrections are +1 and -1 frame (1/32 s): equally far from
    their mean, so min() keeps the start one and the whole group moves by it (adjust_shift)."""
    p = 'a_tie_shift_'
    res = GOLDEN[p + 'result']
    assert res[0, 0] == res[1, 0] == 1.0 + 1 / 32.0 and res[0, 1] == res[0, 2] == 0
