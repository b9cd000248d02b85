"""The transport stream writer (tests/ts_cases.py) and sushi_b200.mpegts against FFmpeg's mpegts demuxer and its
pcm_bluray / truehd decoders (tests/ref_ts.py), on the CPU:
  - the stream list mpegts.py reads (ids, PIDs, kinds, codec names, no default flag) equals FFmpeg's after
    avformat_open_input; after avformat_find_stream_info too, except that FFmpeg's content probe may give a codec to
    a stream whose type it does not know (mpegts.py leaves such a stream without codec, and never decodes it);
  - FFmpeg decodes every BD-LPCM and TrueHD stream to the writer's PCM (channels possibly reordered: the loader takes
    their mean), routes PES packets with stream_id_extension 0x76 to the AC-3 stream and every other to TrueHD;
  - on the cut copies FFmpeg keeps what the product is specified to keep: every whole PES before the cut, and the whole
    sample frames of the last PES whose whole packets survive;
  - selection, refusals and the damaged PAT / PMT read as specified."""
import numpy as np
import pytest

from sushi_b200 import mpegts
from sushi_b200.common import SushiError
from tests import ref_ts
from tests import ts_cases as tsc

CASES = tsc.all_cases()
OPENED = [c for c in CASES if not c.refused]


@pytest.mark.parametrize('case', OPENED, ids=lambda c: c.name)
def test_stream_list_equals_ffmpeg(tmp_path, case):
    path = case.write(tmp_path)
    ts = mpegts.TransportStream(path)
    assert ts.packet_size == case.psize
    mine = [dict(pid=s.pid, kind=s.kind, codec=s.codec, default=s.default) for s in ts.streams_all]
    assert [s.id for s in ts.streams_all] == list(range(len(mine)))
    assert mine == ref_ts.streams(path)
    probed = ref_ts.streams(path, find_info=True)
    assert [s['pid'] for s in probed] == [s['pid'] for s in mine]
    for a, b in zip(mine, probed):
        assert a == b or a['codec'] == 'none', (a, b)


def test_hdmv_and_private_types_follow_ffmpeg():
    c = tsc.case('bd_truehd')
    # TrueHD: FFmpeg adds an AC-3 stream right after it, on the same PID, taking the next id
    assert [(s.stream_type, s.kind) for s in c.streams] == [(0x1B, 'video'), (0x83, 'truehd')]
    no = tsc.case('ts_no_hdmv')
    assert not no.hdmv and [s.stream_type for s in no.streams] == [0x1B, 0x80, 0x83, 0x81, 0x0F]


@pytest.mark.parametrize('case', [c for c in OPENED if c.audio() and c.hdmv and c.name != 'bd_stereo20_48k'],
                         ids=lambda c: c.name)
def test_ffmpeg_decodes_every_stream_to_the_writers_pcm(tmp_path, case):
    path = case.write(tmp_path)
    ts = mpegts.TransportStream(path)
    for s in case.audio():
        st = next(t for t in ts.streams_all if t.pid == s.pid and t.codec in mpegts.DECODED)
        got = ref_ts.decode(path, st.id, s.channels)
        assert ref_ts.same_up_to_channel_order(s.pcm, got), (s.pid, got.shape, s.pcm.shape)


def test_ffmpeg_refuses_20_bit_lpcm(tmp_path):
    # FFmpeg's pcm_bluray decoder refuses every 20-bit packet ("unsupported sample depth"): nothing is decoded
    path = tsc.case('bd_stereo20_48k').write(tmp_path)
    assert len(ref_ts.decode(path, 0, 2)) == 0


def test_ffmpeg_routes_the_ac3_substream_by_stream_id_extension(tmp_path):
    case = tsc.case('bd_truehd')
    path = case.write(tmp_path)
    thd = next(s for s in case.streams if s.kind == 'truehd')
    pk = ref_ts.packets(path)
    ids = [s.id for s in mpegts.TransportStream(path).streams_all if s.pid == tsc.AUDIO_PID]
    ac3 = b''.join(d for i, d in pk if i == ids[1])
    want = b''.join(p[thd.header_len:] for p, f in zip(thd.pes, thd.pes_frames) if f is None)
    assert ac3 == want and len(ac3) > 0


@pytest.mark.parametrize('case', tsc.cut_cases(), ids=lambda c: c.name)
def test_ffmpeg_keeps_what_a_cut_copy_is_specified_to_keep(tmp_path, case):
    path = case.write(tmp_path)
    s = next(x for x in case.streams if x.kind == 'lpcm')
    sid = next(t.id for t in mpegts.TransportStream(path).streams_all if t.pid == s.pid)
    want = case.expected(s)
    assert 0 < len(want) < len(s.pcm) and len(want) not in np.cumsum(s.pes_frames)   # the last PES is cut
    assert ref_ts.same_up_to_channel_order(want, ref_ts.decode(path, sid, s.channels))


def test_selection_follows_the_reference(tmp_path):
    ts = mpegts.TransportStream(tsc.case('bd_two_lpcm').write(tmp_path))
    with pytest.raises(SushiError, match='More than one audio stream found'):
        ts.select('audio', None)
    assert ts.select('audio', 2).pid == tsc.AUDIO_PID + 1
    with pytest.raises(SushiError, match="Stream with index 0 doesn't exist"):
        ts.select('audio', 0)
    assert mpegts.audio_codec(ts.select('audio', 1)) == 'pcm_bluray'
    assert ts.select('subtitles', None).script_type == 'hdmv_pgs_subtitle'
    assert ts.chapters == []
    with pytest.raises(SushiError, match='No subtitles streams found'):
        mpegts.TransportStream(tsc.case('bd_8ch24_48k').write(tmp_path)).select('subtitles', None)


def test_lossy_streams_are_refused_by_codec_name(tmp_path):
    ts = mpegts.TransportStream(tsc.case('bd_lossy').write(tmp_path))
    for sid, codec in ((0, 'ac3'), (1, 'dts')):
        with pytest.raises(SushiError, match=r'^Audio track {0} is {1}, which cannot be decoded here'.format(sid, codec)):
            mpegts.audio_codec(ts.select('audio', sid))
    thd = mpegts.TransportStream(tsc.case('bd_truehd').write(tmp_path))
    assert mpegts.audio_codec(thd.select('audio', 1)) == 'truehd'
    with pytest.raises(SushiError, match='Audio track 2 is ac3'):
        mpegts.audio_codec(thd.select('audio', 2))


def test_refusals_of_the_head(tmp_path):
    with pytest.raises(SushiError, match='has 2 programs'):
        mpegts.TransportStream(tsc.case('bd_two_programs').write(tmp_path))
    bad = tmp_path / 'x.m2ts'
    bad.write_bytes(b'\0' * 4000)
    with pytest.raises(SushiError, match='not a transport stream'):
        mpegts.TransportStream(str(bad))
    for c in tsc.damaged_cases():
        if c.name.endswith(('_pat_crc', '_pmt_crc')):
            with pytest.raises(SushiError, match=r'{0} at byte offset {1}: CRC-32 mismatch'.format(*c.damage)):
                mpegts.TransportStream(c.write(tmp_path))
    assert mpegts.is_transport_stream('A.M2TS') and mpegts.is_transport_stream('b.mts') and \
        not mpegts.is_transport_stream('c.mkv')


def test_damaged_copies_change_what_they_claim(tmp_path):
    # every damaged copy differs from its base in one byte of the packet it names (or of the PES's first packet)
    for c in tsc.damaged_cases():
        base = tsc.case('bd_stereo16_48k' if c.psize == 192 else 'ts_stereo24_48k')
        diff = [i for i in range(len(c.data)) if c.data[i] != base.data[i]] if len(c.data) < 10 ** 6 else []
        assert len(diff) == 1, c.name
