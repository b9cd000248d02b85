"""FFmpeg's `tta` demuxer, Matroska demuxer and `tta` decoder, driven through ctypes, against tests/tta_cases.py and
sushi_b200/tta.py: every .tta case and every A_TTA1 track decodes to the PCM the writer meant; the host's frame tables
hold FFmpeg's packets (bytes and file positions); and what FFmpeg does with each damaged or refused copy, and with each
Matroska Duration case, is recorded beside the refusal this project gives instead (DESIGN.md section 2)."""
import numpy as np
import pytest

from sushi_b200 import SushiError
from sushi_b200 import matroska as mk
from sushi_b200 import tta
from tests import mkv_tta_cases as mtc
from tests import ref_tta as ref
from tests import tta_cases as tc

CASES = tc.all_cases()
MKV = mtc.cases()
BASE, DAMAGED = tc.damaged_cases()
# (samples FFmpeg decodes, packets its decoder refuses) for each damaged copy, or (None, why it gives none): the base
# holds 19718 samples, two frames of 8359 and one of 3000.  Its demuxer checks the header and seek-table CRCs (the
# default err_detect of libavformat is crccheck); its decoder checks no frame CRC (that default is 0), cuts a frame
# short at the last frame's length when only the CRC is left, and refuses a frame that runs out of bits.
FFMPEG = {
    'header_crc': (None, 'demux'), 'seek_crc': (None, 'demux'), 'frame_crc': (19718, 0), 'bitstream_past': (11359, 1),
    'not_on_crc': (19718, 0), 'sizes_past': (8359, 2), 'sizes_short': (16718, 1), 'cut_last_frame': (16718, 1),
    'seek_table_past_file': (None, 'demux'), 'encrypted': (None, 'open'), 'format3': (None, 'open'),
    '8-bit': (None, 'U8'), '9-channels': (2000, 0), 'early_end': (16716, 0),
}
# samples FFmpeg drops from each Matroska track: the last frame when Duration does not give its length
MKV_DROPPED = {'mka_tta_no_duration': 100, 'mka_tta_duration_long': 100, 'mka_tta_duration_short': 100}


def _write(tmp_path, name, data):
    path = str(tmp_path / (name + '.tta'))
    with open(path, 'wb') as f:
        f.write(data)
    return path


def test_cases_cover_the_decoder():
    tc.assert_coverage(CASES)


def test_frame_length_is_ffmpegs():
    """256 * rate / 245 at every rate the cases use, and a last frame of total % length (a whole frame at 0)"""
    for case in CASES:
        fl = tta.frame_length(case.rate)
        assert fl == 256 * case.rate // 245
        assert [len(f) for f in case.frames] and len(case.frames) == -(-len(case.pcm) // fl)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_ffmpeg_decodes_the_tta_file_to_its_pcm(tmp_path, case):
    out, refused = ref.decode(_write(tmp_path, case.name, case.tta()), case.channels, case.bits)
    assert refused == 0
    assert np.array_equal(out, case.pcm)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_frame_table_holds_ffmpegs_packets(tmp_path, case):
    path = _write(tmp_path, case.name, case.tta())
    f = tta.TTAFile(path)
    packets = ref.packets(path)
    assert [p for p, _ in packets] == [int(w) for w in f.where]
    ends = list(f.offsets[1:]) + [len(f.audio)]
    assert [d for _, d in packets] == [f.audio[int(a):int(b)] for a, b in zip(f.offsets, ends)]
    assert list(f.config) == [case.channels, case.bits, case.rate, case.frame_length, len(case.pcm) % case.frame_length]


@pytest.mark.parametrize('pair', MKV, ids=lambda p: p[0].name)
def test_ffmpeg_decodes_the_matroska_track(tmp_path, pair):
    mkv, case, outcome = pair
    out, refused = ref.decode(mkv.write(tmp_path), case.channels, case.bits)
    dropped = MKV_DROPPED.get(mkv.name, 0)
    assert (outcome == 'refused') == bool(dropped)
    assert refused == (1 if dropped else 0)
    assert np.array_equal(out, case.pcm[:len(case.pcm) - dropped])


@pytest.mark.parametrize('pair', MKV, ids=lambda p: p[0].name)
def test_matroska_frame_table_holds_ffmpegs_packets(tmp_path, pair):
    mkv, case, _ = pair
    path = mkv.write(tmp_path)
    with mk.MatroskaFile(path) as f:
        t = f.select('audio', None)
        assert mk.audio_codec(t) == 'tta'
        frames = f.frames([t.id])[t.id]
    assert [d for _, d in ref.packets(path)] == [frames.frame(i) for i in range(len(frames))] == list(case.frames)


def test_matroska_duration_gives_the_last_frame_length(tmp_path):
    """Duration * TimestampScale, rescaled to the rate, modulo the frame length; 0 without a Duration"""
    for mkv, case, _ in MKV:
        with mk.MatroskaFile(mkv.write(tmp_path)) as f:
            t = f.select('audio', None)
            config = tta.matroska_config(t, f.timestamp_scale, f.duration)
        fl = case.frame_length
        if mkv.name.endswith('no_duration') or mkv.name.endswith('no_duration_whole'):
            assert f.duration is None and config[4] == 0
        elif mkv.name.endswith('duration_long'):
            assert config[4] == (len(case.pcm) + 50) % fl
        elif mkv.name.endswith('duration_short'):
            assert config[4] == (len(case.pcm) - 50) % fl
        else:
            assert config[4] == len(case.pcm) % fl
        assert list(config[:4]) == [case.channels, case.bits, case.rate, fl]


def test_matroska_track_without_bit_depth(tmp_path):
    """FFmpeg's decoder does not open (its header says 0 bits); the track is refused by name"""
    path = mtc.no_bitdepth().write(tmp_path)
    assert ref.decode(path, 1, 16) == (None, 'open')
    with mk.MatroskaFile(path) as f:
        with pytest.raises(SushiError, match='Audio track 0 is TTA without BitDepth, which cannot be decoded here'):
            mk.audio_codec(f.select('audio', None))


@pytest.mark.parametrize('damaged', DAMAGED, ids=lambda d: d[0])
def test_what_ffmpeg_does_with_each_damaged_copy(tmp_path, damaged):
    name, data, frame, regex, kernel = damaged
    path = _write(tmp_path, name, data)
    out, refused = ref.decode(path, 9 if name == '9-channels' else 1 if name == 'early_end' else 2, 16)
    assert (None if out is None else len(out), refused) == FFMPEG[name]
    if not kernel:
        with pytest.raises(SushiError, match=regex):
            tta.TTAFile(path)
    else:
        tta.TTAFile(path)                      # header and seek table are sound: the GPU decoder refuses the frame


def test_tags_end_the_audio_as_for_ffmpeg(tmp_path):
    """An ID3v2 tag in front is skipped; an APEv2 or ID3v1 tag after the last frame ends the audio"""
    for case in CASES:
        if case.head or case.tail:
            f = tta.TTAFile(_write(tmp_path, 'a', case.tta()))
            bare = tta.TTAFile(_write(tmp_path, 'b', case.tta()[len(case.head):len(case.tta()) - len(case.tail)]))
            assert f.audio == bare.audio and np.array_equal(f.offsets, bare.offsets)
            assert np.array_equal(f.where, bare.where + len(case.head))
            assert tta.is_tta(_write(tmp_path, 'c', case.tta()))
