"""Matroska files with A_WAVPACK4 tracks for the tests, built with the writers of tests/mkv_cases.py: the frames of a
tests/wavpack_cases.py stream in FFmpeg's Matroska layout (block_samples, then per block flags, CRC, a size unless the
frame has one block, the sub-blocks), one to a Matroska frame, in blocks with every lacing.  CodecPrivate is the 2-byte
stream version.  Cases: mono, stereo and multichannel (several blocks per frame) streams, header stripping, and a file
cut inside its last block."""
import struct

from tests import mkv_cases as mc
from tests import wavpack_cases as wc


def wavpack_track(case, encodings=()):
    spec = mc.TrackSpec('audio', 'A_WAVPACK4', struct.pack('<H', case.st.version), True, 'wavpack', 'eng', 0,
                        case.rate, case.channels, case.bits, encodings=encodings, pcm=case.pcm, pcm_bits=case.bits)
    at = 0
    for f, n in zip(case.mkv_frames(), case.counts):
        spec.frames.append((f, at, n))
        at += n
    return spec


def audio_only(name, case, encodings=()):
    """A Matroska file holding only the case's stream as an A_WAVPACK4 track, frames laced in every way"""
    lac = ['none', 'xiph', 'ebml', 'fixed', 'none']
    a = mc._timed(wavpack_track(case, encodings), 1000.0 / case.rate)
    ab = mc._blocks_for(0, a, lambda j: (lac[j % 5], 1 + j % 3, j % 4 == 1, None))
    ts, clusters = mc.arrange([a], 2000, [ab])
    return mc.build(name, [a], clusters, ts)


def cases():
    """[(MkvCase, WvCase)]: the cases as A_WAVPACK4 files, one with header stripping, one cut inside its last block"""
    picked = [c for c in wc.all_cases() if c.name in ('mono16', 'stereo16_joint', 'stereo24', 'three24', 'six16',
                                                     'eight24', 'false_stereo16', 'mono24_custom_rate')]
    out = [(audio_only('mka_wv_' + c.name, c), c) for c in picked]
    even = wc.make_case('even', 50, counts=(500,) * 6, nterms=[4, 9, 2])
    out.append((audio_only('mka_wv_strip', even, encodings=[('strip', struct.pack('<I', 500))]), even))
    full = audio_only('mka_wv_cut', even)
    last = max(e[2] for e in full.expect[0])
    full.data = full.data[:last + 40]
    out.append((full, even))
    return out


def kept_samples(mkv, case):
    """The samples a file's whole frames hold (all of them unless the file is cut)"""
    if not mkv.name.endswith('_cut'):
        return len(case.pcm)
    last = max(e[2] for e in mkv.expect[0])
    return sum(n for (f, t, o), n in zip(mkv.expect[0], case.counts) if o < last)
