"""The format table (sushi_b200/inputs.py): one small file of every format the test writers produce opens with the reader
the table's detection order gives it, by content where the format has a content mark, and its select_audio() names the
codec and the stream without loading the library."""
import shutil

import pytest

from sushi_b200 import _native, flac, inputs, matroska, mp4, mpegts, truehd, tta, wav, wavpack
from tests import alac_cases, flac_cases, mkv_alac_cases, mkv_cases, mkv_truehd_cases, mkv_tta_cases, mkv_wavpack_cases
from tests import mp4_cases, truehd_cases, ts_cases, tta_cases, wavpack_cases


def _write(tmp_path, name, data):
    path = tmp_path / name
    path.write_bytes(data)
    return str(path)


def _mkv_track(tmp_path, codec):
    """(path, stream id) of a Matroska test file's first track of `codec`."""
    for case in mkv_cases.audio_cases():
        for sid in case.audio_ids():
            if case.specs[sid].codec == codec:
                return case.write(tmp_path), sid


def _mp4(tmp_path, name):
    return next(c for c in mp4_cases.good_cases() if c.name == name).write(tmp_path), None


# name -> (file and track, format name, reader class, label, whether a stream id comes back)
FILES = {
    'wav': (lambda d: (flac_cases.named_cases()[0].write_wav(d), None), 'WAV', wav.DownmixedWavFile, None, False),
    'flac': (lambda d: (flac_cases.named_cases()[0].write(d), None), 'FLAC', flac.FlacFile, 'FLAC', False),
    'thd': (lambda d: (truehd_cases.named_cases()[0].write(d), None), 'TrueHD', truehd.TrueHDFile, 'TrueHD', False),
    'wv': (lambda d: (_write(d, 'a.wv', wavpack_cases.all_cases()[0].wv()), None), 'WavPack', wavpack.WavPackFile,
           'WavPack', False),
    'tta': (lambda d: (_write(d, 'a.tta', tta_cases.all_cases()[0].tta()), None), 'TTA', tta.TTAFile, 'TTA', False),
    'mka_flac': (lambda d: _mkv_track(d, 'A_FLAC'), 'Matroska', matroska.MatroskaFile, 'FLAC', True),
    'mka_pcm': (lambda d: _mkv_track(d, 'A_PCM/INT/LIT'), 'Matroska', matroska.MatroskaFile, None, True),
    'mka_truehd': (lambda d: (mkv_truehd_cases.audio_only('t', truehd_cases.named_cases()[0]).write(d, '.mka'), None),
                   'Matroska', matroska.MatroskaFile, 'TrueHD', True),
    'mka_alac': (lambda d: (mkv_alac_cases.audio_only('a', alac_cases.all_cases()[0]).write(d, '.mka'), None),
                 'Matroska', matroska.MatroskaFile, 'ALAC', True),
    'mka_wavpack': (lambda d: (mkv_wavpack_cases.audio_only('w', wavpack_cases.all_cases()[0]).write(d, '.mka'), None),
                    'Matroska', matroska.MatroskaFile, 'WavPack', True),
    'mka_tta': (lambda d: (mkv_tta_cases.audio_only('t', tta_cases.all_cases()[0]).write(d, '.mka'), None),
                'Matroska', matroska.MatroskaFile, 'TTA', True),
    'm4a_alac': (lambda d: _mp4(d, 'm4a_alac'), 'MP4', mp4.Mp4File, 'ALAC', True),
    'mp4_flac': (lambda d: _mp4(d, 'mp4_flac'), 'MP4', mp4.Mp4File, 'FLAC', True),
    'mp4_pcm': (lambda d: _mp4(d, 'mp4_ipcm'), 'MP4', mp4.Mp4File, None, True),
    'm2ts_lpcm': (lambda d: (ts_cases.case('bd_stereo16_48k').write(d), None), 'transport stream',
                  mpegts.TransportStream, 'BD-LPCM', True),
    'm2ts_truehd': (lambda d: (ts_cases.case('bd_truehd').write(d), 1), 'transport stream', mpegts.TransportStream,
                    'TrueHD', True),
}


@pytest.fixture
def no_library(monkeypatch):
    monkeypatch.setattr(_native, 'lib', lambda *a, **kw: pytest.fail('the library was loaded'))


@pytest.mark.parametrize('key', sorted(FILES))
def test_every_format_opens_with_its_reader(tmp_path, no_library, key):
    make, name, reader_class, label, has_id = FILES[key]
    path, track = make(tmp_path)
    reader, got_name = inputs.open_input(path)
    try:
        assert (type(reader), got_name) == (reader_class, name)
        audio = reader.select_audio(track)
        assert audio.label == label
        assert (audio.pcm is not None, audio.decode is None) == (label is None, label is None)
        if has_id:
            assert audio.id == (reader.select('audio', track).id if track is None else track)
        else:
            assert audio.id is None
        # an opened container passes through; an opened raw-file reader is not an input
        if name in ('Matroska', 'MP4', 'transport stream'):
            assert inputs.open_input(reader) == (reader, name)
    finally:
        if hasattr(reader, 'close'):
            reader.close()


@pytest.mark.parametrize('key, suffix', [('flac', '.wav'), ('wv', '.flac'), ('tta', '.wav'), ('mka_flac', '.mp4'),
                                         ('m4a_alac', '.mkv'), ('wav', '.flac'), ('wav', '.bin')])
def test_content_decides_not_the_extension(tmp_path, key, suffix):
    make, name, reader_class = FILES[key][:3]
    path = shutil.copy(make(tmp_path)[0], str(tmp_path / ('renamed' + suffix)))
    reader, got_name = inputs.open_input(path)
    assert (type(reader), got_name) == (reader_class, name)
    if hasattr(reader, 'close'):
        reader.close()


def test_detection_order_and_extensions():
    assert [f.name for f in inputs.FORMATS] == ['transport stream', 'MP4', 'Matroska', 'TrueHD', 'WavPack', 'TTA',
                                                'FLAC', 'WAV']
    extensions = [e for f in inputs.FORMATS for e in f.extensions]
    assert len(extensions) == len(set(extensions))
    assert {f.name for f in inputs.FORMATS if f.opens_as} == {'transport stream', 'MP4', 'Matroska'}
