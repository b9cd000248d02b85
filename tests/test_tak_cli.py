"""The command line's refusals on TAK inputs, all before the GPU is touched: every copy of a .tak file the host reader
refuses (8 bits, 7 channels, 3 channels in the mono/stereo codec, other data types, codec types and frame size types, a
missing or corrupt STREAMINFO, a LAST_FRAME past the end), as source and as destination, and the same copies through
WavStream before the library is loaded."""
import pytest

from sushi_b200 import _native, cli, wavstream
from sushi_b200.common import SushiError
from tests import tak_cases as tc


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


HOST = [d for d in tc.damaged_cases()[1] if not d[4]]


@pytest.mark.parametrize('damaged', HOST, ids=lambda d: d[0])
def test_tak_refusals(tmp_path, script, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.tak')
    src.write_bytes(data)
    dst = tmp_path / 'dst.tak'
    dst.write_bytes(tc.all_cases()[0].tak())
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(src), '--dst', str(dst), '--script', script])
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(dst), '--dst', str(src), '--script', script])
    assert not list(tmp_path.glob('*.wav'))


@pytest.mark.parametrize('damaged', HOST, ids=lambda d: d[0])
def test_tak_refusals_come_before_the_library(tmp_path, no_library, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.tak')
    src.write_bytes(data)
    with pytest.raises(SushiError, match=regex):
        wavstream.WavStream(str(src))


def test_tak_needs_a_gpu_loader(tmp_path, no_library):
    src = tmp_path / 'a.tak'
    src.write_bytes(tc.all_cases()[0].tak())
    with pytest.raises(SushiError, match="TAK input needs loader='gpu'"):
        wavstream.WavStream(str(src), loader='host')
