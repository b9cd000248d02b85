"""The APE writer (tests/ape_cases.py) against FFmpeg's `ape` demuxer and decoder (tests/ref_ape.py): every written
stream decodes to the writer's PCM, and ApeFile's frame table cuts the file exactly as FFmpeg's packets do.  What
FFmpeg does with each damaged or refused copy is recorded here; the refusals ApeFile makes come before the library is
loaded."""
import struct

import numpy as np
import pytest

from sushi_b200 import SushiError, _native, ape
from tests import ape_cases as ac
from tests import ref_ape

CASES = ac.all_cases()
BASE, DAMAGED = ac.damaged_cases()

# What FFmpeg makes of each damaged copy of BASE (4 stereo frames of 2000 blocks): a refusal ('demux': its demuxer
# refuses the file; 'open': its decoder does not open; 'U8': it decodes to unsigned 8 bits), or (frames it returns,
# packets its decoder refuses, whether what it returns is BASE's PCM).  Every copy is refused here.
FFMPEG = {
    'version': 'demux',               # versions 3.80 to 3.99 other than 3990 take older decoders; 3.99.x only here
    'bits8': 'U8',
    'bits32': 'open',
    'channels3': 'open',
    'level6000': 'open',
    'level1500': 'open',
    'rate_2g': 'open',
    'blocks_huge': (1, 3, False),         # frames over INT_MAX / 8 - 8 blocks are refused; the 1-block last decodes
    'seek_short': 'demux',
    'seek_backwards': (2000, 0, False),   # a frame of negative size ends the demuxing after frame 0
    'seek_past_end': (6000, 0, False),
    'crc': (8000, 0, True),               # checked only under AV_EF_CRCCHECK, so FFmpeg returns the samples
    'flags': (8000, 0, True),             # unknown flag bits are ignored
    'payload': (6000, 1, False),          # the damaged frame is refused (range decoder error) and dropped
    'cut_last': (6000, 1, False),         # the cut frame runs the range decoder past its end and is dropped
    'interim24': (6000, 0, False),        # 24-bit: see test_ffmpeg_leaves_its_predictor_past_24_bits
}


def _write(tmp_path, name, data):
    path = str(tmp_path / (name + '.ape'))
    with open(path, 'wb') as f:
        f.write(data)
    return path


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_ffmpeg_decodes_the_writer_s_pcm_and_packets_match_the_frame_table(tmp_path, case):
    path = _write(tmp_path, case.name, case.ape())
    pcm, refused = ref_ape.decode(path, case.channels, case.bits)
    assert refused == 0
    want = case.pcm if case.bits == 16 else ac.wrap24(case.pcm)
    assert pcm.shape == want.shape and np.array_equal(pcm, want)
    f = ape.ApeFile(path)
    assert list(f.offsets) == case.frame_offsets()
    packets = ref_ape.packets(path)
    assert len(packets) == len(f.offsets)
    first = int(f.offsets[0])
    for i, (_, data) in enumerate(packets):
        blocks, skip = struct.unpack_from('<II', data)
        assert blocks == (case.bpf if i + 1 < len(packets) else case.final_blocks)
        assert skip == (int(f.offsets[i]) - first) & 3
        start = int(f.offsets[i]) - skip
        end = int(f.offsets[i + 1]) if i + 1 < len(packets) else start + skip + ((f.end - int(f.offsets[i])) & ~3)
        size = min((end - start + 3) & ~3, len(f.data) - start)
        assert data[8:] == f.data[start:start + size]


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_frame_crcs_pass_ffmpeg_s_own_check(tmp_path, case):
    """The frame CRC as the writer stores it and the decoder checks it (CRC-32 of the little-endian output bytes,
    shifted right by one) is FFmpeg's: under err_detect crccheck+explode no frame of a good stream is refused."""
    path = _write(tmp_path, case.name, case.ape())
    assert ref_ape.crc_refusals(path) == (0, len(case.pcm))


def test_ffmpeg_s_crc_check_refuses_the_damaged_crc(tmp_path):
    name, data, frame, _, _ = next(d for d in DAMAGED if d[0] == 'crc')
    path = _write(tmp_path, name, data)
    assert ref_ape.crc_refusals(path) == (1, len(BASE.pcm) - BASE.bpf)


def test_ffmpeg_leaves_its_predictor_past_24_bits(tmp_path):
    """A 24-bit stereo sample past 2^23 (here 2^23 + 1, at block 500 of frame 1) makes FFmpeg's decoder try its 64-bit
    predictor mode; for this stream it then returns samples other than the stream's from the next block to the end of
    that frame, and decodes the following frame as before.  The decoder here refuses that frame; a sample of exactly
    +-2^23 decodes (case edge24)."""
    case = ac.interim_case()
    path = _write(tmp_path, case.name, case.ape())
    pcm, refused = ref_ape.decode(path, 2, 24)
    assert refused == 0 and pcm.shape == case.pcm.shape
    differ = np.nonzero((pcm != ac.wrap24(case.pcm)).any(1))[0]
    assert differ[0] == 2501 and differ[-1] < 4000


def test_coverage():
    ac.assert_coverage(CASES)


@pytest.mark.parametrize('damaged', DAMAGED, ids=lambda d: d[0])
def test_what_ffmpeg_does_with_each_damaged_copy(tmp_path, damaged):
    name, data, _, _, _ = damaged
    path = _write(tmp_path, name, data)
    pcm, refused = ref_ape.decode(path, 2, 16)
    want = FFMPEG[name]
    if pcm is None:
        assert refused == want
    else:
        assert (len(pcm), refused, pcm.shape == BASE.pcm.shape and np.array_equal(pcm, BASE.pcm)) == want


@pytest.mark.parametrize('damaged', [d for d in DAMAGED if not d[4]], ids=lambda d: d[0])
def test_refusals_come_before_the_library_is_loaded(tmp_path, monkeypatch, damaged):
    name, data, _, regex, _ = damaged
    path = _write(tmp_path, name, data)

    def no_library(*a, **k):
        raise AssertionError('the library was loaded')

    monkeypatch.setattr(_native, 'load_library', no_library)
    monkeypatch.setattr(_native, 'lib', no_library)
    with pytest.raises(SushiError, match=regex):
        ape.ApeFile(path).select_audio()


def test_detection_by_content(tmp_path):
    from sushi_b200 import inputs
    case = next(c for c in CASES if c.head)
    path = _write(tmp_path, 'tagged', case.ape())
    renamed = tmp_path / 'tagged.bin'
    renamed.write_bytes(open(path, 'rb').read())
    reader, name = inputs.open_input(str(renamed))
    assert name == 'APE' and isinstance(reader, ape.ApeFile)
    assert not ape.is_ape(str(tmp_path / 'missing.ape'))
