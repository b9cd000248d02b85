"""Raw MPEG audio files on the CPU: sushi_b200.mpa against FFmpeg's `mp3` demuxer and `mp2` decoder
(tests/ref_mp4.decode_s16 decodes the file as the ffmpeg command line does).  The bytes the reader hands to the decoder
(ID3v2 tags in front skipped, APEv2 and ID3v1 tags at the end left out) decode, through the CPU build of sb_mp2.cuh,
to FFmpeg's samples, a stream starting mid-frame and one cut inside its last frame included; layer III is refused by
name before the library is loaded."""
import numpy as np
import pytest

from sushi_b200 import _native, inputs, mpa
from sushi_b200.common import SushiError
from tests import mpa_cases
from tests import ref_mp4
from tests import ref_ps
from tests.test_mp2_cases import decode, emu  # noqa: F401  (the CPU build of sb_mp2.cuh)

CASES = mpa_cases.all_cases()


@pytest.mark.parametrize('case', CASES, ids=lambda c: c[0])
def test_reader_hands_over_what_ffmpeg_decodes(emu, tmp_path, monkeypatch, case):  # noqa: F811
    name, data, c, stream = case
    path = tmp_path / (name + '.mp2')
    path.write_bytes(data)
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))
    reader, fmt = inputs.open_input(str(path))
    assert fmt == 'MPEG audio' and reader.select_audio().label == 'MP2'
    assert reader.data[reader.start:reader.end] == stream
    assert [s['codec'] for s in ref_ps.streams(str(path))] == ['mp2']
    want, mask, rate = ref_mp4.decode_s16(str(path), 0)
    assert rate == c.rate and mask == {1: 0x4, 2: 0x3}[c.channels]
    got, cut = decode(emu, stream)
    assert got is not None, cut
    assert cut == (name == 'cut_tail')
    assert np.array_equal(got, want)


def test_layer3_is_refused_by_name(tmp_path):
    path = tmp_path / 'x.mpa'
    path.write_bytes(mpa_cases.layer3())
    with pytest.raises(SushiError, match=r'x.mpa is MPEG audio layer III \(MP3\), which cannot be decoded here'):
        mpa.MpegAudioFile(str(path))
    assert mpa.is_mpeg_audio('a.M2A') and not mpa.is_mpeg_audio('a.mp3')
