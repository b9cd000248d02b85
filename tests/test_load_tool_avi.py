"""tools/load.py's `avi` entry on the CPU: its file at 1 minute opens as an AVI file with two movi-bearing RIFF lists
when its first list is kept small, passes select_audio(), and holds 48 kHz stereo PCM of the bit depth written."""
import importlib.util
import os

import pytest

from sushi_b200 import avi, inputs
from tests import avi_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location('load_tool', os.path.join(ROOT, 'tools', 'load.py'))
load = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(load)


@pytest.mark.parametrize('bits', [16, 24])
def test_avi_entry_builds_files_its_reader_opens(tmp_path, bits):
    assert load.cases('avi', None, None) == [(90, 16), (90, 24)]
    rows = load.ALL_FORMATS['avi'].build(str(tmp_path), 1, bits)
    assert [r['input'] for r, _ in rows] == ['avi (PCM)']
    reader, got = inputs.open_input(rows[0][1])
    assert got == 'AVI' and len(reader.movi) == 1
    s = reader.tracks[reader.select_audio().id]
    assert (s.channels, s.rate, s.codec) == (2, 48000, 'pcm_s%dle' % bits)
    assert rows[0][0]['bytes'] > 60 * 48000 * 2 * bits // 8


def test_long_file_splits_into_opendml_segments(tmp_path):
    path = str(tmp_path / 'odml.avi')
    pcm = avi_cases.long_file(path, 0.5, 16, seg_bytes=1 << 20)
    f = avi.AviFile(path)
    assert len(f.movi) > 1 and len(f.movi) == open(path, 'rb').read().count(b'AVIX') + 1
    assert pcm.shape == (30 * 48000, 2)
