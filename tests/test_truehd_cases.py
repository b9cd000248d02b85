"""FFmpeg's TrueHD decoder (libavcodec through ctypes, tests/ref_truehd.py) decodes every undamaged stream of
tests/truehd_cases.py to the writer's PCM, and every Matroska file of tests/mkv_truehd_cases.py through its Matroska
demuxer.  This pins the writer's reading of the format against an independent decoder, including which substream is
decoded and the channel order: the output is substream min(n - 1, 2) in the layout of the 13-bit (8-channel
presentation) arrangement, in FFmpeg's native channel order, and a fourth (object) substream is skipped."""
import numpy as np
import pytest

from tests import mkv_truehd_cases as mtc
from tests import ref_truehd
from tests import truehd_cases as tc

CASES = tc.all_cases()


def test_writer_covers_the_coding_tools():
    tc.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_ffmpeg_decodes_the_writer_pcm(tmp_path, case):
    got = ref_truehd.decode(case.write(tmp_path), case.channels)
    assert got.shape == case.pcm.shape
    assert np.array_equal(got, case.pcm), int(np.count_nonzero(got != case.pcm))


def test_channel_order_is_ffmpegs_native_order():
    # 7.1 with back surrounds: the restart header counts L R C LFE Ls Rs Lb Rb, FFmpeg outputs FL FR FC LFE BL BR SL SR
    assert tc.channel_codes(tc.ARRANGE2[8]) == [0, 1, 2, 3, 6, 7, 4, 5]
    assert any(c.channels == 8 and c.n_sub >= 3 for c in CASES)


@pytest.mark.parametrize('pair', mtc.cases(), ids=lambda p: p[0].name)
def test_ffmpeg_decodes_matroska_truehd_tracks(tmp_path, pair):
    mkv, case = pair
    got = ref_truehd.decode(mkv.write(tmp_path), case.channels, raw=False)
    assert np.array_equal(got, case.pcm)
