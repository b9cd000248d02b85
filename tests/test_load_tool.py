"""tools/load.py's builders against the product's host path: every format's files, written at 1 minute (mkv and ts
with their 24-minute shapes), open as the format they are meant to be and pass select_audio(); where a reader reports
the channel count, rate and sample count, they are what the builder wrote.  The files are not loaded, so no GPU is
needed; this is what fails when a change to a tests/*_cases.py helper breaks the tool."""
import importlib.util
import os

import pytest

from sushi_b200 import flac, inputs, tta, wav, wavpack

_spec = importlib.util.spec_from_file_location(
    'load_tool', os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools', 'load.py'))
load = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(load)

# input kind -> the format name open_input gives its file
FORMAT_NAMES = {'flac': 'FLAC', 'wav': 'WAV', 'mkv': 'Matroska', 'truehd': 'TrueHD', 'm2ts': 'transport stream',
                'alac': 'MP4', 'wavpack': 'WavPack', 'tta': 'TTA', 'mp2 (program stream)': 'program stream',
                'flac 24-bit stereo (Ogg)': 'Ogg', 'mp2 (Matroska)': 'Matroska', 'flac stereo': 'FLAC'}

# (format, input kind) -> samples per channel of the 1-minute file, where its reader reports them.  The FLAC file of
# 4608-sample frames ends in a 100-sample frame; ALAC's WAV is 43 whole repetitions of 16 frames of 4096; TTA's is 57
# frames of 50 155 and a last frame of 1000.
SAMPLES = {('flac', 'flac'): 2880100, ('flac', 'wav'): 2880100, ('mkv', 'flac'): 2880000,
           ('truehd', 'wav'): 2880000, ('truehd', 'flac'): 2880100, ('ts', 'wav'): 2880000,
           ('alac', 'flac'): 2880100, ('alac', 'wav'): 2818048,
           ('wavpack', 'wavpack'): 2880000, ('wavpack', 'flac'): 2880100, ('wavpack', 'wav'): 2880000,
           ('tta', 'tta'): 2859835, ('tta', 'flac'): 2880100, ('tta', 'wav'): 2859835,
           ('swr', 'flac stereo'): 2880100}


def reported(reader):
    """(channels, rate, samples per channel) of a reader that knows them before decoding, else None."""
    if isinstance(reader, wav.DownmixedWavFile):
        return reader.channels_count, reader.framerate, reader.frames_count
    if isinstance(reader, flac.FlacFile):
        return reader.channels_count, reader.framerate, reader.total_samples
    if isinstance(reader, tta.TTAFile):
        return reader.channels, reader.rate, reader.samples
    if isinstance(reader, wavpack.WavPackFile):
        return reader.stream.channels, reader.stream.rate, reader.samples
    return None


@pytest.fixture
def no_device(monkeypatch):
    """The SM count (for TrueHD's threads per SM) is the device's; there is none here."""
    monkeypatch.setattr(load, 'sm_count', lambda: None)


def build(name, directory):
    if name == 'mkv':
        return load.build_mkv(directory, 1, None, mbps=load.MKV_RATES[24, None])
    if name == 'ts':
        return load.build_ts(directory, 1, 16, video=load.TS_FILLER[24, 16])
    fmt = load.FORMATS[name]
    return fmt.build(directory, 1, fmt.bits[0] if fmt.bits else None)


@pytest.mark.parametrize('name', sorted(load.FORMATS))
def test_every_format_builds_files_its_reader_opens(tmp_path, no_device, name):
    files = build(name, str(tmp_path))
    for row, path in files:
        if row['input'] in load.LEGS:
            continue
        reader, got = inputs.open_input(path)
        try:
            assert got == FORMAT_NAMES[row['input']], (row, path)
            assert reader.select_audio() is not None
            if (name, row['input']) in SAMPLES:
                assert reported(reader) == (2, 48000, SAMPLES[name, row['input']]), (row, path)
            else:
                assert reported(reader) is None, (row, path)
        finally:
            if hasattr(reader, 'close'):
                reader.close()


def test_lengths_outside_a_shape_table_are_refused():
    assert load.cases('ts', [24], [24]) == [(24, 24)]
    assert load.cases('mkv', None, [16]) == [(24, None), (90, None)]
    with pytest.raises(ValueError, match='mkv has shapes'):
        load.cases('mkv', [30], None)
    with pytest.raises(ValueError, match='truehd is built at 16 bits only'):
        load.cases('truehd', None, [24])
