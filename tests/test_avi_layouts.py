"""The channel layout the AVI reader gives --ffmpeg-audio, held to FFmpeg's: for every PCM and MP2 stream of
tests/avi_cases.py (plain WAVEFORMATEX, WAVEFORMATEXTENSIBLE with and without a channel mask, 1 to 8 channels), the
mask AviFile's Audio names for its channel count equals the layout FFmpeg's decoder reports (or, where it reports
none, the default layout the ffmpeg command line assumes), as tests/test_swr_layouts.py holds the other readers."""
import pytest

from sushi_b200 import avi
from tests import avi_cases as ac
from tests import ref_mp4


def _streams():
    return [(c, i) for c in ac.good_cases() for i, _ in c.audio()]


@pytest.mark.parametrize('pair', _streams(), ids=lambda p: '%s_%d' % (p[0].name, p[1]))
def test_layout_equals_ffmpegs(tmp_path, pair):
    case, sid = pair
    path = case.write(tmp_path)
    audio = avi.AviFile(path).select_audio(sid)
    out, _, _, mask, rate = ref_mp4._decode(path, sid, None)
    assert audio.layout[out.shape[1]] == mask
    assert rate == case.streams[sid].case.rate if case.streams[sid].case else rate == avi.AviFile(path).tracks[sid].rate
