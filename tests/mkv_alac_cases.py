"""Matroska files with A_ALAC tracks for the tests, built with the writers of tests/mkv_cases.py: the frames of a
tests/alac_cases.py stream, one to a Matroska frame, in blocks with every lacing.  CodecPrivate is the stream's
24-byte ALACSpecificConfig."""
from tests import alac_cases as ac
from tests import mkv_cases as mc


def alac_track(case, default=True):
    spec = mc.TrackSpec('audio', 'A_ALAC', case.cfg.cookie(), default, 'alac', 'eng', 0, case.rate, case.channels,
                        case.bits, pcm=case.pcm, pcm_bits=case.bits)
    at = 0
    for f in case.frames:
        n = ac.frame_samples(case.cfg, f)
        spec.frames.append((f, at, n))
        at += n
    return spec


def audio_only(name, case):
    """A Matroska file holding only the case's stream as an A_ALAC track, several frames laced"""
    lac = ['none', 'xiph', 'ebml', 'none']
    a = mc._timed(alac_track(case), 1000.0 / case.rate)
    ab = mc._blocks_for(0, a, lambda j: (lac[j % 4], 1 + j % 3, j % 4 == 1, None))
    ts, clusters = mc.arrange([a], 2000, [ab])
    return mc.build(name, [a], clusters, ts)


def cases():
    """[(MkvCase, AlacCase)]: every ALAC case as an audio-only Matroska file"""
    return [(audio_only('mka_' + c.name, c), c) for c in ac.all_cases()]
