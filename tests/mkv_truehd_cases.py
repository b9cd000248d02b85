"""Matroska files with A_TRUEHD tracks for the tests, built with the writers of tests/mkv_cases.py: the AUs of a
tests/truehd_cases.py stream grouped several to a frame, in blocks with every lacing, next to a video track."""
import numpy as np

from tests import mkv_cases as mc
from tests import truehd_cases as tc


def truehd_track(case, per_frame, default=True):
    """The case's AUs, `per_frame` to a Matroska frame (times in samples)."""
    spec = mc.TrackSpec('audio', 'A_TRUEHD', b'', default, 'truehd', 'eng', 0, case.rate, case.channels, None,
                        pcm=case.pcm, pcm_bits=24)
    offs = list(case.au_offsets) + [len(case.data)]
    for k in range(0, len(case.au_offsets), per_frame):
        j = min(k + per_frame, len(case.au_offsets))
        spec.frames.append((case.data[offs[k]:offs[j]], k * case.spa, (j - k) * case.spa))
    return spec


def cases():
    """[(MkvCase, TrueHDCase)]"""
    out = []
    lac = ['none', 'xiph', 'ebml', 'fixed', 'none', 'ebml']
    for name, case, per in (('thd_stereo', tc.make('mkv_stereo', 2, 16, 48000, n_au=90, seed=60, style=tc.FULL,
                                                   restarts=(16, 5)), 3),
                            ('thd_71', tc.make('mkv_71', 8, 24, 48000, n_au=64, n_sub=3, seed=61, style=tc.FULL,
                                               restarts=(8,), objects=True), 5)):
        a = mc._timed(truehd_track(case, per), 1000.0 / case.rate)
        v = mc.video_track(20, 3)
        ab = mc._blocks_for(1, a, lambda j: (lac[j % 6], 1 + j % 3, j % 4 == 1, None))
        vb = mc._blocks_for(0, v, lambda j: ('none', 1, False, None))
        ts, clusters = mc.arrange([v, a], 250, [vb, ab])
        out.append((mc.build(name, [v, a], clusters, ts), case))
    return out


def audio_only(name, case, per=4):
    """A Matroska file holding only the case's stream as an A_TRUEHD track, `per` AUs to a frame, several laced"""
    lac = ['none', 'xiph', 'ebml', 'fixed']
    a = mc._timed(truehd_track(case, per), 1000.0 / case.rate)
    ab = mc._blocks_for(0, a, lambda j: (lac[j % 4], 1 + j % 3, j % 4 == 1, None))
    ts, clusters = mc.arrange([a], 2000, [ab])
    return mc.build(name, [a], clusters, ts)
