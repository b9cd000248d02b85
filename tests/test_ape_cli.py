"""The command line's refusals on Monkey's Audio inputs, all before the GPU is touched: every copy of a .ape file the
host reader refuses (other versions, 8 and 32 bits, 3 channels, compression levels FFmpeg does not open, a seek table
cut short or inconsistent), as source and as destination, and the same copies through WavStream before the library is
loaded."""
import pytest

from sushi_b200 import _native, cli, wavstream
from sushi_b200.common import SushiError
from tests import ape_cases as ac


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


HOST = [d for d in ac.damaged_cases()[1] if not d[4]]


@pytest.mark.parametrize('damaged', HOST, ids=lambda d: d[0])
def test_ape_refusals(tmp_path, script, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.ape')
    src.write_bytes(data)
    dst = tmp_path / 'dst.ape'
    dst.write_bytes(ac.all_cases()[0].ape())
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(src), '--dst', str(dst), '--script', script])
    with pytest.raises(SushiError, match=regex):
        run(['--src', str(dst), '--dst', str(src), '--script', script])
    assert not list(tmp_path.glob('*.wav'))


@pytest.mark.parametrize('damaged', HOST, ids=lambda d: d[0])
def test_ape_refusals_come_before_the_library(tmp_path, no_library, damaged):
    name, data, _, regex, _ = damaged
    src = tmp_path / (name + '.ape')
    src.write_bytes(data)
    with pytest.raises(SushiError, match=regex):
        wavstream.WavStream(str(src))


def test_ape_needs_a_gpu_loader(tmp_path, no_library):
    src = tmp_path / 'a.ape'
    src.write_bytes(ac.all_cases()[0].ape())
    with pytest.raises(SushiError, match="APE input needs loader='gpu'"):
        wavstream.WavStream(str(src), loader='host')

