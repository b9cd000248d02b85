"""AVI files on the CPU: the writer of tests/avi_cases.py and sushi_b200.avi against FFmpeg's `avi` demuxer
(tests/ref_avi.py):
  - FFmpeg reads every case as intended: each audio stream's packets are the payloads the writer put in its chunks,
    across JUNK, LIST rec, ix##, idx1, zero-size and odd-sized chunks and OpenDML segments;
  - the stream list AviFile reads (ids, kinds, codec names) equals FFmpeg's on every case;
  - selection, and every refusal by codec name, before the library is loaded;
  - the --ffmpeg-audio fields: 16-bit PCM and MP2 convert, 24-bit is refused, and PCM's channel layout is what FFmpeg's
    decoder reports (the extensible header's mask, else the default layout)."""
import numpy as np
import pytest

from sushi_b200 import _native, avi, inputs, swr
from sushi_b200.common import SushiError
from tests import avi_cases as ac
from tests import ref_avi

GOOD = ac.good_cases()
REFUSED = ac.refused_cases()


@pytest.fixture
def no_library(monkeypatch):
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))


@pytest.mark.parametrize('case', GOOD + [r[0] for r in REFUSED] + [ac.partial_frame_case()[0]], ids=repr)
def test_ffmpeg_reads_the_case_as_written(tmp_path, case):
    path = case.write(tmp_path)
    for i, s in case.audio():
        assert b''.join(ref_avi.packets(path, i)) == s.es


@pytest.mark.parametrize('case', GOOD + [r[0] for r in REFUSED], ids=repr)
def test_stream_list_equals_ffmpeg(tmp_path, case):
    path = case.write(tmp_path)
    f = avi.AviFile(path)
    assert [dict(id=s.id, kind=s.kind, codec=s.codec) for s in f.streams_all] == ref_avi.streams(path)
    assert f.movi == case.movi_extents() and f.chapters == []
    assert inputs.open_input(path)[1] == 'AVI'


def test_opendml_cases_have_what_they_should():
    odml = [c for c in GOOD if c.segments > 1]
    assert len(odml) == 2
    for c in odml:
        assert c.data.count(b'AVIX') == c.segments - 1 and b'indx' in c.data and b'ix00' in c.data
    assert any(c.rec for c in GOOD) and any(c.junk for c in GOOD) and any(not c.idx1 for c in GOOD)
    assert any(len(x) & 1 for c in GOOD for s in c.streams for x in s.chunks)
    assert any(len(x) == 0 for c in GOOD for _, s in c.audio() for x in s.chunks)


def test_selection_and_refusals(tmp_path, no_library):
    two = avi.AviFile(next(c for c in GOOD if c.name == 'two_audio_preload').write(tmp_path))
    with pytest.raises(SushiError, match='More than one audio stream found'):
        two.select_audio(None)
    assert two.select_audio(1).label == 'PCM' and two.select_audio(2).id == 2
    with pytest.raises(SushiError, match="Stream with index 0 doesn't exist"):
        two.select_audio(0)
    subs = avi.AviFile(next(c for c in GOOD if c.name == 'mp2_cbr_subs').write(tmp_path))
    assert subs.select_audio().label == 'MP2'
    assert subs.select('subtitles', None).script_type == 'none'
    for case, sid, regex in REFUSED:
        with pytest.raises(SushiError, match=r'^Audio track {0} {1}, which cannot be decoded here'.format(sid, regex)):
            avi.AviFile(case.write(tmp_path)).select_audio()
    l3 = ac.mp2_stream(ac._mp2('avi_l3', 404, 10, bitrate_index=10, mode=0), True)
    l3.chunks = [bytes([f[0], (f[1] & ~0x06) | 0x02]) + f[2:] for f in l3.chunks]
    l3.es = b''.join(l3.chunks)
    case = ac.AviCase('layer3', [ac.video_stream(np.random.default_rng([1]), 5), l3],
                      ac.interleave([ac.video_stream(np.random.default_rng([1]), 5), l3], None))
    with pytest.raises(SushiError, match=r'^Audio track 1 is MPEG audio layer III \(MP3\), which cannot be decoded'):
        avi.AviFile(case.write(tmp_path)).select_audio()
    bad = tmp_path / 'x.avi'
    bad.write_bytes(b'RIFF\x04\x00\x00\x00WAVE')
    assert not avi.is_avi(str(bad))
    with pytest.raises(SushiError, match='not an AVI file'):
        avi.AviFile(str(bad))


def test_ffmpeg_audio_fields(tmp_path, no_library):
    """16-bit PCM and MP2 convert; 24-bit PCM gets the S32 refusal"""
    for name, track, fmt in (('pcm16_every_frame', 1, 'S16'), ('mp2_vbr_odml', 1, 'S16'),
                             ('pcm24_51_half_second', 1, 'S32')):
        a = avi.AviFile(next(c for c in GOOD if c.name == name).write(tmp_path)).select_audio(track)
        assert a.fmt == fmt
        if fmt == 'S16':
            swr.check(a)
        else:
            with pytest.raises(SushiError, match='decodes to S32'):
                swr.check(a)
