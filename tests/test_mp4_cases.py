"""sushi_b200/mp4.py against FFmpeg's mov demuxer (tests/ref_mp4.py) on every file of tests/mp4_cases.py: streams,
ids, kinds, default flags and codec names; chapters; each audio sample's bytes, order and file offset; what a cut
copy keeps.  FFmpeg's decoders give back the writer's PCM from the same files.  Refused and damaged copies are
refused, naming the track, box and byte offset."""
import re
import struct

import numpy as np
import pytest

from sushi_b200 import mp4
from sushi_b200.common import SushiError
from tests import mp4_cases as m
from tests import ref_mp4

GOOD = m.good_cases()


def _kinds(streams):
    return [('other' if k == 'data' else k, c, d) for k, c, d in streams]


def test_cases_cover_the_reader():
    m.assert_coverage(GOOD)


@pytest.mark.parametrize('case', GOOD, ids=lambda c: c.name)
def test_streams_chapters_and_samples_agree_with_ffmpeg(tmp_path, case):
    path = case.write(tmp_path)
    ref = ref_mp4.demux(path)
    assert ref.streams == case.expect
    with mp4.Mp4File(path) as f:
        kinds = [('other' if t.kind == 'data' else t.kind, t.codec, t.default) for t in f.tracks]
        assert kinds == _kinds(ref.streams)
        assert f.chapters == ref.chapters == case.chapters
        for sid in case.audio_ids():
            t = f.track(sid)
            table = f.frames(t)
            packets = ref.track(sid)
            assert table.data == b''.join(p for p, _ in packets)
            assert list(table.block) == [pos for _, pos in packets]
            if t.codec in ('alac', 'flac'):
                assert [bytes(table.frame(i)) for i in range(len(table))] == [p for p, _ in packets]


@pytest.mark.parametrize('case', GOOD, ids=lambda c: c.name)
def test_ffmpeg_decodes_the_writers_pcm(tmp_path, case):
    path = case.write(tmp_path)
    for sid in case.audio_ids():
        t = case.traks[sid]
        out, refused = ref_mp4.decode_pcm(path, sid, t.channels, t.bits)
        assert refused == 0 and np.array_equal(out, t.pcm)


@pytest.mark.parametrize('pair', m.refused_cases(), ids=lambda p: p[0].name)
def test_refused_files_name_the_reason(tmp_path, pair):
    case, regex = pair
    path = case.write(tmp_path)
    with pytest.raises(SushiError, match=regex):
        with mp4.Mp4File(path) as f:
            t = f.select('audio', None)
            mp4.audio_codec(t)
            f.check_edits(t)


@pytest.mark.parametrize('pair', m.damaged_cases(), ids=lambda p: p[0].name)
def test_damage_is_refused_naming_box_and_offset(tmp_path, pair):
    case, regex = pair
    path = case.write(tmp_path)
    with pytest.raises(SushiError) as e:
        with mp4.Mp4File(path) as f:
            f.frames(f.select('audio', None))
    assert re.search(regex, str(e.value)), str(e.value)


@pytest.mark.parametrize('pair', m.cut_cases(), ids=lambda p: p[0].name)
def test_cut_copy_keeps_what_ffmpeg_keeps(tmp_path, pair, caplog):
    case, length = pair
    path = str(tmp_path / ('cut_' + case.name + case.suffix))
    with open(path, 'wb') as f:
        f.write(case.data[:length])
    ref = ref_mp4.demux(path)
    with mp4.Mp4File(path) as f:
        assert f.cut
        for sid in case.audio_ids():
            t = f.track(sid)
            table = f.frames(t)
            out, refused = ref_mp4.decode_pcm(path, sid, case.traks[sid].channels, case.traks[sid].bits)
            width = case.traks[sid].channels * (case.traks[sid].bits // 8)
            if t.codec in ('alac', 'flac'):
                # FFmpeg hands the decoder the partial last sample, which it refuses; the reader drops it
                whole = [p for p, _ in ref.track(sid)][:len(table)]
                assert [bytes(table.frame(i)) for i in range(len(table))] == whole
                assert refused <= 1
                n = len(out)
            else:
                n = len(table.data) // width
                assert table.data == b''.join(p for p, _ in ref.track(sid))[:n * width]
            assert n == len(out) and np.array_equal(out, case.traks[sid].pcm[:n])
    assert 'cut' in caplog.text


def test_sparse_file_past_4_gib(tmp_path):
    path = str(tmp_path / 'sparse.m4a')
    case = m.sparse_file(path)
    ref = ref_mp4.demux(path)
    with mp4.Mp4File(path) as f:
        table = f.frames(f.select('audio', None))
        assert table.block[0] > 2 ** 32
        assert table.data == b''.join(p for p, _ in ref.track(0)) == case.data
        assert f.bytes_read < 1 << 20


def test_wav_whose_size_field_spells_a_box_name_is_not_mp4(tmp_path):
    """A RIFF size field of b'free' (a WAV of about 1.7 GB) does not make the file an MP4: only the header matters."""
    path = tmp_path / 'big.wav'
    path.write_bytes(b'RIFF' + b'free' + b'WAVEfmt ' + bytes(100))
    assert not mp4.is_mp4(str(path))
    path.write_bytes(struct.pack('>I', 24) + b'ftypM4A ' + bytes(16))
    assert mp4.is_mp4(str(path))


@pytest.mark.parametrize('name', ['tkhd', 'mdhd', 'hdlr', 'stsd', 'mvhd'])
def test_box_too_short_for_its_fields_is_refused_naming_it(tmp_path, name):
    """A leaf box cut short (its size shrunk, the bytes it gives up made into a `free` box) is refused with a message
    naming the box and its offset, not a Python exception."""
    data = bytearray(m.good_cases()[0].data)
    at = data.index(name.encode()) - 4
    size = struct.unpack('>I', data[at:at + 4])[0]
    keep = 12 if name != 'stsd' else 16
    struct.pack_into('>I', data, at, keep)
    struct.pack_into('>I4s', data, at + keep, size - keep, b'free')
    path = tmp_path / 'short.m4a'
    path.write_bytes(bytes(data))
    with pytest.raises(SushiError, match=r"box '%s' at byte offset %d is too short|sample descriptions" % (name, at)):
        with mp4.Mp4File(str(path)) as f:
            mp4.audio_codec(f.select('audio', None))
