"""The TAK writer (tests/tak_cases.py) against FFmpeg's `tak` demuxer, parser and decoder (tests/ref_tak.py): every
written stream decodes to the writer's PCM, and the frame table (the CPU run of the sync stage) cuts the file exactly
where FFmpeg's packets do.  What FFmpeg does with each damaged or refused copy is recorded here; the refusals TakFile
makes come before the library is loaded."""
import numpy as np
import pytest

from sushi_b200 import SushiError, _native, tak
from tests import ref_tak
from tests import tak_cases as tc
from tests.test_kernel_emulation_tak import build, frame_table

CASES = tc.all_cases()
BASE, DAMAGED = tc.damaged_cases()

# What FFmpeg makes of each damaged copy of BASE (4 stereo frames of 1024 samples): a refusal ('demux': its demuxer
# refuses the file; 'open': its decoder does not open), or (samples it returns, packets its decoder refuses).  Every
# copy is refused here.
FFMPEG = {
    'bits8': (4096, 0),               # the decoder takes its parameters from the frames' stream info, not STREAMINFO
    'channels7': (4096, 0),
    'stereo_codec_3ch': (4096, 0),
    'data_type1': (4096, 0),
    'codec3': (4096, 0),
    'frame_type12': 'demux',
    'frame_type6_6k': 'demux',
    'no_streaminfo': 'open',
    'streaminfo_crc': (4096, 0),      # the demuxer checks the block CRC only under AV_EF_EXPLODE
    'last_frame_past_end': (4096, 0),
    'data_crc': (4096, 0),            # checked only under AV_EF_CRCCHECK
    'trailing': (4096, 0),            # bytes after the data CRC are ignored
    'cut_last': (4096, 0),            # the reader reads zeros past the packet
    'shift': (3072, 1),
    'subframes': (3072, 1),
    'order': (3072, 1),
    'coding': (3072, 1),
    'short_decor': (3072, 1),
    'mcdparams': (2048, 1),
    'metadata': (3072, 0),            # not a frame start for the parser: the frame is merged into the one before
    'contradicts': (2048, 2),
    'number_gap': (4096, 0),          # frame numbers are not checked
    'no_info_first': (0, 4),          # without stream info the decoder knows no codec type
    'total': (4096, 0),
}


def _write(tmp_path, name, data):
    path = str(tmp_path / (name + '.tak'))
    with open(path, 'wb') as f:
        f.write(data)
    return path


@pytest.fixture(scope='module')
def emu():
    return build()


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_ffmpeg_decodes_the_writer_s_pcm_and_packets_match_the_frame_table(emu, tmp_path, case):
    path = _write(tmp_path, case.name, case.tak())
    pcm, refused = ref_tak.decode(path, case.channels, case.bits)
    assert refused == 0
    assert pcm.shape == case.pcm.shape and np.array_equal(pcm, case.pcm)
    f = tak.TakFile(path)
    frames = frame_table(emu, f)
    packets = ref_tak.packets(path)
    assert [p for p, _ in packets] == [s for s, _ in frames]
    for (start, end), (pos, data) in zip(frames, packets):
        # FFmpeg's last packet runs to the end of the file: a trailing tag without LAST_FRAME is in it
        assert data[:end - start] == f.data[start:end]
        assert len(data) == end - start or (end == f.audio_end and len(data) == len(f.data) - start)


def test_ffmpeg_checks_the_data_crc_under_crccheck(tmp_path):
    good = _write(tmp_path, 'good', BASE.tak())
    assert ref_tak.crc_refusals(good) == (0, 4096)
    bad = _write(tmp_path, 'bad', next(d[1] for d in DAMAGED if d[0] == 'data_crc'))
    assert ref_tak.crc_refusals(bad) == (1, 3072)


@pytest.mark.parametrize('damaged', DAMAGED, ids=lambda d: d[0])
def test_what_ffmpeg_does_with_each_damaged_copy(tmp_path, damaged):
    name, data = damaged[:2]
    path = _write(tmp_path, name, data)
    channels = 3 if name == 'mcdparams' else 2
    pcm, refused = ref_tak.decode(path, channels, 16)
    got = refused if pcm is None else (len(pcm), refused)
    assert got == FFMPEG[name]


@pytest.mark.parametrize('damaged', [d for d in DAMAGED if not d[4]], ids=lambda d: d[0])
def test_host_refusals_come_before_the_library(tmp_path, monkeypatch, damaged):
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))
    name, data, _, regex, _ = damaged
    with pytest.raises(SushiError, match=regex):
        tak.TakFile(_write(tmp_path, name, data))


@pytest.mark.parametrize('name', ['mc6_plain', 'mc6_chained', 'dmode1', 'order4'])
def test_reader_layout_is_ffmpeg_s(tmp_path, name):
    case = next(c for c in CASES if c.name == name)
    path = _write(tmp_path, name, case.tak())
    assert tak.TakFile(path).layout == ref_tak.layout(path)
