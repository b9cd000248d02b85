"""FFmpeg's `ogg` demuxer for the tests: libavformat from the opencv wheel (oracle/ref_flac.libs()), driven through
ctypes, as tests/ref_ps.py drives the `mpeg` demuxer.

`streams(path)` gives FFmpeg's stream list after avformat_find_stream_info (what `ffmpeg -i` lists), `chapters(path)`
the chapter starts in seconds, `packets(path, index)` the payload of every packet of one stream as av_read_frame returns
them (a FLAC stream's header packets are not among them).  Samples come from tests/ref_mp4.decode_s16.  Test
infrastructure only: the product never imports this."""
from tests import ref_mp4, ref_ps, ref_ts


def streams(path):
    """[{kind, codec}] in FFmpeg's stream order (the `ogg` demuxer gives each stream its index as its id, which is
    checked)"""
    out = ref_ps.streams(path)
    assert [s['id'] for s in out] == list(range(len(out))), out
    return [dict(kind=s['kind'], codec=s['codec']) for s in out]


def chapters(path):
    return ref_mp4.demux(path, packets=False).chapters


def packets(path, index):
    """the bytes of every packet of stream `index`, in order"""
    return [d for i, d in ref_ts.packets(path) if i == index]
