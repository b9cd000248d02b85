"""The FLAC encoder of tests/flac_cases.py against an independent decoder (FFmpeg's libavcodec, oracle/ref_flac.py):
every case decodes to exactly the PCM it was built from.  Each damaged file is checked to be damaged the way it
claims: the CRC it breaks no longer matches, the gap is there, the file ends inside its last frame, the STREAMINFO
total is off by one."""
import numpy as np
import pytest

from oracle import ref_flac
from sushi_b200.wavstream import FlacFile
from tests import flac_cases as fc

CASES = fc.all_cases()
BASE, CORRUPT = fc.corrupt_cases()


@pytest.mark.parametrize('case', CASES + [BASE], ids=lambda c: c.name)
def test_libavcodec_decodes_the_encoder_pcm(tmp_path, case):
    path = case.write(tmp_path)
    got, sfmt = ref_flac.decode(path, case.channels, len(case.pcm))
    # 16-bit FLAC comes back as S16, 24-bit as S32 with the sample in the top 24 bits
    if len(case.pcm):
        assert sfmt == (ref_flac.AV_SAMPLE_FMT_S16 if case.bits == 16 else ref_flac.AV_SAMPLE_FMT_S32)
    assert np.array_equal(ref_flac.decode_pcm(path, case.channels, case.bits, len(case.pcm)), case.pcm)


@pytest.mark.parametrize('case', CASES + [BASE], ids=lambda c: c.name)
def test_metadata_reader(tmp_path, case):
    info = FlacFile(case.write(tmp_path))
    assert (info.channels_count, info.bits_per_sample, info.framerate) == (case.channels, case.bits, case.rate)
    assert info.frame_offset == int(case.offsets[0])
    assert info.total_samples in (0, len(case.pcm))


def test_metadata_blocks_and_id3_are_skipped(tmp_path):
    by = {c.name: c for c in CASES}
    blocks = FlacFile(by['metadata_blocks'].write(tmp_path)).blocks
    assert blocks == ['STREAMINFO', 'SEEKTABLE', 'VORBIS_COMMENT', 'PADDING', 'PICTURE', 'APPLICATION']
    assert by['id3_prefix_total_unknown'].flac.startswith(b'ID3')


def _frame_bytes(case, k):
    return case.flac[int(case.offsets[k]):int(case.offsets[k + 1])]


@pytest.mark.parametrize('case', CORRUPT, ids=lambda c: c.name)
def test_corrupt_case_is_damaged_as_described(case):
    kind, k, where, _ = case.corrupt
    good = BASE.flac
    if kind == 'crc8':
        head = case.flac[where:where + 16]
        n = 4 + len(fc.utf8_number(k))
        assert fc.crc8(head[:n]) != head[n] and fc.crc8(good[where:where + n]) == good[where + n]
        assert len(case.flac) == len(good) and sum(a != b for a, b in zip(case.flac, good)) == 1
    elif kind == 'crc16':
        frame = case.flac[int(BASE.offsets[k]):int(BASE.offsets[k + 1])]
        assert fc.crc16_many([frame[:-2]])[0] != int.from_bytes(frame[-2:], 'big')
        assert fc.crc16_many([_frame_bytes(BASE, k)[:-2]])[0] == int.from_bytes(_frame_bytes(BASE, k)[-2:], 'big')
        assert len(case.flac) == len(good)
    elif kind == 'gap':
        end = int(BASE.offsets[k + 1])
        assert case.flac[:end] == good[:end] and case.flac[end:end + 3] == b'\0\0\0' and case.flac[end + 3:] == good[end:]
    elif kind in ('truncated', 'truncated_header'):
        assert good.startswith(case.flac) and int(BASE.offsets[k]) < len(case.flac) < int(BASE.offsets[k + 1])
        assert len(good) == int(BASE.offsets[-1]) and k == len(BASE.frames) - 1
    elif kind == 'total':
        assert len(case.flac) == len(good)
        def total(d):
            return int.from_bytes(d[18:26], 'big') & ((1 << 36) - 1)
        assert total(good) == len(BASE.pcm) and total(case.flac) == len(BASE.pcm) + 1
    else:
        raise AssertionError(kind)


def test_unsupported_depth_case_is_valid_flac(tmp_path):
    case = fc.unsupported_bits_case()
    path = case.write(tmp_path)
    assert FlacFile(path).bits_per_sample == 20
    assert np.array_equal(ref_flac.decode_pcm(path, case.channels, 20, len(case.pcm)), case.pcm)
