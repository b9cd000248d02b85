"""The command line's refusals on WavPack inputs, all before the GPU is touched: every copy of a .wv file the host
reader refuses (hybrid, float, DSD, 1- and 4-byte samples, extended precision, a broken block chain), an A_WAVPACK4
track of an unsupported stream version, and the name of the codec in the refusal of a track nothing here decodes.  A
Matroska track's flags are refused by WavStream before the library is loaded."""
import struct

import pytest

from sushi_b200 import _native, cli, wavstream
from sushi_b200 import matroska as mk
from sushi_b200.common import SushiError
from tests import mkv_cases as mc
from tests import mkv_wavpack_cases as mwc
from tests import wavpack_cases as wc


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def script(tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    path = tmp_path / 'in.ass'
    path.write_text('[Script Info]\n')
    return str(path)


@pytest.mark.parametrize('damaged', [d for d in wc.damaged_cases()[1] if not d[4]], ids=lambda d: d[0])
def test_wv_refusals(tmp_path, script, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.wv')
    src.write_bytes(data)
    dst = tmp_path / 'dst.wv'
    dst.write_bytes(wc.all_cases()[0].wv())
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(src), '--dst', str(dst), '--script', script])
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(dst), '--dst', str(src), '--script', script])


def _track_file(tmp_path, case, version=0x407, flag=0):
    frames = case.mkv_frames()
    if flag:
        frames = [f[:4] + struct.pack('<I', struct.unpack_from('<I', f, 4)[0] | flag) + f[8:] for f in frames]
    spec = mc.TrackSpec('audio', 'A_WAVPACK4', struct.pack('<H', version), True, 'wavpack', 'eng', 0, case.rate,
                        case.channels, case.bits, pcm=case.pcm, pcm_bits=case.bits)
    at = 0
    for f, n in zip(frames, case.counts):
        spec.frames.append((f, at, n))
        at += n
    a = mc._timed(spec, 1000.0 / case.rate)
    ts, clusters = mc.arrange([a], 2000, [mc._blocks_for(0, a, lambda j: ('none', 1, False, None))])
    return mc.build('v%x_%x' % (version, flag), [a], clusters, ts).write(tmp_path, '.mka')


def test_matroska_version_is_refused(tmp_path, script):
    case = wc.all_cases()[1]
    good = mwc.audio_only('good', case).write(tmp_path, '.mka')
    bad = _track_file(tmp_path, case, version=0x401)
    with pytest.raises(SushiError, match='Audio track 0 is WavPack stream version 0x401, which cannot be decoded here'):
        run(['--src', bad, '--dst', good, '--script', script])
    with mk.MatroskaFile(good) as f:
        assert mk.audio_codec(f.select('audio', None)) == 'wavpack'


@pytest.mark.parametrize('flag, kind', [(wc.HYBRID, 'hybrid'), (wc.FLOAT, 'float'), (wc.DSD, 'DSD')])
def test_matroska_flags_are_refused_before_the_library(tmp_path, monkeypatch, flag, kind):
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))
    path = _track_file(tmp_path, wc.all_cases()[1], flag=flag)
    with pytest.raises(SushiError, match=r'Audio track 0 is WavPack \(%s\), which cannot be decoded here' % kind):
        wavstream.WavStream(path)


def test_wv_host_loader_is_refused_before_the_library(tmp_path, monkeypatch):
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))
    path = tmp_path / 'a.wv'
    path.write_bytes(wc.all_cases()[0].wv())
    with pytest.raises(SushiError, match="WavPack input needs loader='gpu'"):
        wavstream.WavStream(str(path), loader='host')
