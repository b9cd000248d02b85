"""Matroska files with A_TTA1 tracks for the tests, built with the writers of tests/mkv_cases.py: the frames of a
tests/tta_cases.py stream (bitstream and CRC, no header or seek table), one to a Matroska frame, in SimpleBlocks and
BlockGroups with every lacing.  FFmpeg's Matroska demuxer builds the decoder's TTA header from the track and takes the
sample total from the Segment's Duration, so the cases vary it: a Duration that gives the stream's total, none, and one
that disagrees with the frames.  A track without BitDepth is built too."""
import struct

import numpy as np

from tests import mkv_cases as mc
from tests import tta_cases as tc

DURATION_1000 = b'\x44\x89\x88' + struct.pack('>d', 1000.0)        # the Duration mkv_cases.build writes


def tta_track(case, bits=True):
    spec = mc.TrackSpec('audio', 'A_TTA1', b'', True, 'tta', 'eng', 0, case.rate, case.channels,
                        case.bits if bits else None, pcm=case.pcm, pcm_bits=case.bits)
    fl = case.frame_length
    for k, f in enumerate(case.frames):
        spec.frames.append((f, k * fl, None))
    return spec


def duration_ms(samples, rate):
    """A Duration (milliseconds, TimestampScale 10^6) FFmpeg turns back into `samples` at `rate`"""
    d = samples * 1000.0 / rate
    assert (int(d * 1000000) * rate + 500000000) // 1000000000 == samples
    return d


LAYOUT = [('none', 1, False), ('xiph', 2, True), ('fixed', 2, False), ('ebml', 2, False), ('none', 1, True)]


def audio_only(name, case, duration='exact', bits=True):
    """A Matroska file holding only the case's stream as an A_TTA1 track, frames laced by LAYOUT in turn.  duration:
    'exact' (the stream's total), 'none', or a number of samples."""
    a = mc._timed(tta_track(case, bits), 1000.0 / case.rate)
    ab = mc._blocks_for(0, a, lambda j: LAYOUT[j % len(LAYOUT)][:3] + (None,))
    ts, clusters = mc.arrange([a], 2000, [ab])
    m = mc.build(name, [a], clusters, ts)
    assert m.data.count(DURATION_1000) == 1
    if duration == 'none':
        new = b'\xec\x89' + bytes(9)                                  # a Void of the same size
    else:
        total = len(case.pcm) if duration == 'exact' else duration
        new = DURATION_1000[:3] + struct.pack('>d', duration_ms(total, case.rate))
    m.data = m.data.replace(DURATION_1000, new)
    return m


def lacing_case():
    """Eight frames at 8000 Hz, the fourth and fifth silent (the same bytes, for fixed lacing), and 100 samples"""
    fl = tc.frame_length(8000)
    tone = tc.signal(np.random.default_rng([41]), 8 * fl, 1, 16, 'tone')
    pcm = np.concatenate([tone[:3 * fl], np.zeros((2 * fl, 1), np.int64), tone[5 * fl:7 * fl + 100]])
    case = tc.make_case('laced', 41, rate=8000, channels=1, pcm=pcm)
    assert case.frames[3] == case.frames[4]
    return case


def cases():
    """[(MkvCase, TtaCase, 'decoded' or 'refused')]: what the GPU decoder does with each track (a refusal names the
    last frame)"""
    by = {c.name: c for c in tc.all_cases()}
    laced = lacing_case()
    out = [(audio_only('mka_tta_laced', laced), laced, 'decoded')]
    for name in ('stereo24_noise', 'eight24_extreme', 'six16', 'rate192000'):
        out.append((audio_only('mka_tta_' + name, by[name]), by[name], 'decoded'))
    # no Duration: the decoder's last frame length is 0, so a short last frame runs past its bytes
    out.append((audio_only('mka_tta_no_duration', laced, duration='none'), laced, 'refused'))
    out.append((audio_only('mka_tta_no_duration_whole', by['eight24_extreme'], duration='none'),
                by['eight24_extreme'], 'decoded'))
    out.append((audio_only('mka_tta_duration_long', laced, duration=len(laced.pcm) + 50), laced, 'refused'))
    out.append((audio_only('mka_tta_duration_short', laced, duration=len(laced.pcm) - 50), laced, 'refused'))
    return out


def no_bitdepth(case=None):
    """An A_TTA1 file whose track has no BitDepth"""
    case = case or tc.all_cases()[0]
    return audio_only('mka_tta_no_bitdepth', case, bits=False)
