"""The command line's refusals on TTA inputs, all before the GPU is touched: every copy of a .tta file the host reader
refuses (encrypted, other formats, 8-bit, 9 channels, damaged header or seek table, a cut file), and A_TTA1 tracks
WavStream refuses before the library is loaded (no BitDepth, 8 bits, 9 channels, the host loader)."""
import pytest

from sushi_b200 import _native, cli, wavstream
from sushi_b200 import matroska as mk
from sushi_b200.common import SushiError
from tests import mkv_cases as mc
from tests import mkv_tta_cases as mtc
from tests import tta_cases as tc


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def script(tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    path = tmp_path / 'in.ass'
    path.write_text('[Script Info]\n')
    return str(path)


@pytest.fixture
def no_library(monkeypatch):
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))


@pytest.mark.parametrize('damaged', [d for d in tc.damaged_cases()[1] if not d[4]], ids=lambda d: d[0])
def test_tta_refusals(tmp_path, script, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.tta')
    src.write_bytes(data)
    dst = tmp_path / 'dst.tta'
    dst.write_bytes(tc.all_cases()[0].tta())
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(src), '--dst', str(dst), '--script', script])
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(dst), '--dst', str(src), '--script', script])
    assert not list(tmp_path.glob('*.wav'))


@pytest.mark.parametrize('damaged', [d for d in tc.damaged_cases()[1] if not d[4]], ids=lambda d: d[0])
def test_tta_refusals_come_before_the_library(tmp_path, no_library, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.tta')
    src.write_bytes(data)
    with pytest.raises(SushiError, match=regex):
        wavstream.WavStream(str(src))


def _track_file(tmp_path, name, case, channels=None, bits=None, drop_bits=False):
    spec = mtc.tta_track(case, bits=not drop_bits)
    spec.channels = channels or spec.channels
    spec.bits = None if drop_bits else (bits or spec.bits)
    a = mc._timed(spec, 1000.0 / case.rate)
    ts, clusters = mc.arrange([a], 2000, [mc._blocks_for(0, a, lambda j: ('none', 1, False, None))])
    return mc.build(name, [a], clusters, ts).write(tmp_path, '.mka')


@pytest.mark.parametrize('kw, regex', [
    (dict(drop_bits=True), 'Audio track 0 is TTA without BitDepth, which cannot be decoded here'),
    (dict(bits=8), 'Audio track 0 is TTA at 8 bits, which cannot be decoded here'),
    (dict(channels=9), 'Audio track 0 is TTA with 9 channels, which cannot be decoded here'),
])
def test_matroska_track_refusals_come_before_the_library(tmp_path, no_library, script, kw, regex):
    case = tc.all_cases()[1]
    path = _track_file(tmp_path, 'bad', case, **kw)
    with pytest.raises(SushiError, match=regex):
        wavstream.WavStream(path)
    good = mtc.audio_only('good', case).write(tmp_path, '.mka')
    with pytest.raises(SushiError, match=regex):
        run(['--src', path, '--dst', good, '--script', script])
    with mk.MatroskaFile(good) as f:
        assert mk.audio_codec(f.select('audio', None)) == 'tta'


def test_host_loader_is_refused_before_the_library(tmp_path, no_library):
    case = tc.all_cases()[0]
    path = tmp_path / 'a.tta'
    path.write_bytes(case.tta())
    with pytest.raises(SushiError, match="TTA input needs loader='gpu'"):
        wavstream.WavStream(str(path), loader='host')
    mka = mtc.audio_only('a', case).write(tmp_path, '.mka')
    with pytest.raises(SushiError, match="TTA input needs loader='gpu'"):
        wavstream.WavStream(mka, loader='host')


def test_unknown_codec_refusal_lists_tta(tmp_path):
    case = tc.all_cases()[0]
    spec = mtc.tta_track(case)
    spec.codec = 'A_AAC'
    a = mc._timed(spec, 1000.0 / case.rate)
    ts, clusters = mc.arrange([a], 2000, [mc._blocks_for(0, a, lambda j: ('none', 1, False, None))])
    path = mc.build('aac', [a], clusters, ts).write(tmp_path, '.mka')
    with mk.MatroskaFile(path) as f:
        with pytest.raises(SushiError, match=r'Audio track 0 is A_AAC, which cannot be decoded here \(FLAC, TrueHD, '
                                             r'ALAC, WavPack, TTA and'):
            mk.audio_codec(f.select('audio', None))
