"""tools/load.py's `tak` entry on the CPU: its files at 1 minute open as the formats they are meant to be, pass
select_audio(), and, where the reader knows them, hold 48 kHz stereo of the length written.  One 12 000-sample (250 ms)
frame repeated for a minute is 240 frames; the WAV holds the same samples."""
import importlib.util
import os

import pytest

from sushi_b200 import tak, flac, inputs, wav

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location('load_tool', os.path.join(ROOT, 'tools', 'load.py'))
load = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(load)

NAMES = {'tak': 'TAK', 'flac': 'FLAC', 'wav': 'WAV'}
SAMPLES = {'tak': 240 * 12000, 'wav': 240 * 12000, 'flac': 2880100}


def reported(reader):
    if isinstance(reader, tak.TakFile):
        return reader.channels, reader.rate, reader.samples
    if isinstance(reader, wav.DownmixedWavFile):
        return reader.channels_count, reader.framerate, reader.frames_count
    if isinstance(reader, flac.FlacFile):
        return reader.channels_count, reader.framerate, reader.total_samples
    return None


@pytest.mark.parametrize('bits', [16, 24])
def test_tak_entry_builds_files_its_readers_open(tmp_path, bits):
    assert load.cases('tak', None, None) == [(24, 16), (24, 24), (90, 16), (90, 24)]
    for row, path in load.ALL_FORMATS['tak'].build(str(tmp_path), 1, bits):
        reader, got = inputs.open_input(path)
        try:
            assert got == NAMES[row['input']], (row, path)
            assert reader.select_audio() is not None
            assert reported(reader) == (2, 48000, SAMPLES[row['input']]), (row, path)
        finally:
            if hasattr(reader, 'close'):
                reader.close()
