"""tools/load.py's `ape` entry on the CPU: its files at 1 minute open as the formats they are meant to be, pass
select_audio(), and, where the reader knows them, hold 48 kHz stereo of the length written.  One 1 179 648-block frame
repeated for a minute is 2 frames; the WAV holds the same samples."""
import importlib.util
import os

import pytest

from sushi_b200 import ape, flac, inputs, wav

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location('load_tool', os.path.join(ROOT, 'tools', 'load.py'))
load = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(load)

NAMES = {'ape': 'APE', 'flac': 'FLAC', 'wav': 'WAV'}
SAMPLES = {'ape': 2 * 1179648, 'wav': 2 * 1179648, 'flac': 2880100}


def reported(reader):
    if isinstance(reader, ape.ApeFile):
        return reader.channels, reader.rate, reader.samples
    if isinstance(reader, wav.DownmixedWavFile):
        return reader.channels_count, reader.framerate, reader.frames_count
    if isinstance(reader, flac.FlacFile):
        return reader.channels_count, reader.framerate, reader.total_samples
    return None


@pytest.mark.parametrize('bits', [16, 24])
def test_ape_entry_builds_files_its_readers_open(tmp_path, bits):
    assert load.cases('ape', None, None) == [(24, 16), (24, 24), (90, 16), (90, 24)]
    for row, path in load.ALL_FORMATS['ape'].build(str(tmp_path), 1, bits):
        reader, got = inputs.open_input(path)
        try:
            assert got == NAMES[row['input']], (row, path)
            assert reader.select_audio() is not None
            assert reported(reader) == (2, 48000, SAMPLES[row['input']]), (row, path)
        finally:
            if hasattr(reader, 'close'):
                reader.close()
