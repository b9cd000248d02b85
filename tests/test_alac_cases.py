"""FFmpeg's `alac` decoder, driven through ctypes, decodes every stream of tests/alac_cases.py (in an A_ALAC Matroska
file) to the PCM the writer meant, so the writer's streams pin the decoder's arithmetic to FFmpeg's."""
import numpy as np
import pytest

from oracle import ref_flac
from tests import alac_cases as ac
from tests import mkv_alac_cases as mac

PAIRS = mac.cases()


def test_cases_cover_the_decoder():
    ac.assert_coverage([c for _, c in PAIRS])


@pytest.mark.parametrize('pair', PAIRS, ids=lambda p: p[1].name)
def test_ffmpeg_decodes_the_case_to_its_pcm(tmp_path, pair):
    mkv, case = pair
    out = ref_flac.decode_pcm(mkv.write(tmp_path), case.channels, case.bits, len(case.pcm))
    assert np.array_equal(out, case.pcm)
    assert np.array_equal(ac.to16(out, case.bits), case.pcm16)


def test_bytes_after_end_are_ignored(tmp_path):
    """FFmpeg decodes a frame with bytes after its END element as it decodes the frame without them."""
    case = [c for _, c in PAIRS if 'trailing_bytes' in c.used][0]
    stripped = ac.AlacCase('stripped', case.cfg, [f.rstrip(b'\xa5\x00\x17') if f.endswith(b'\xa5\x00\x17') else f
                                                  for f in case.frames], case.pcm, set())
    a = ref_flac.decode_pcm(mac.audio_only('with', case).write(tmp_path), case.channels, case.bits, len(case.pcm))
    b = ref_flac.decode_pcm(mac.audio_only('without', stripped).write(tmp_path), case.channels, case.bits,
                            len(case.pcm))
    assert np.array_equal(a, b)
