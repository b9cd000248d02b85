"""FFmpeg's `mpeg` (program stream) and `mp3` (raw MPEG audio) demuxers for the tests: libavformat from the opencv
wheel (oracle/ref_flac.libs()), driven through ctypes.

`streams(path)` gives FFmpeg's stream list after avformat_open_input and avformat_find_stream_info (what `ffmpeg -i`
lists); `packets(path, index)` the payload of every packet of one stream, as av_read_frame returns them.  The samples
of the `mp2` decoder come from tests/ref_mp4.decode_s16, which decodes any input the same way.  The struct fields read
are those tests/ref_ts.py reads (libavformat 62), with the same checks: a stream's index is its position, a packet's
stream index is in range.  Test infrastructure only: the product never imports this."""
import ctypes

from oracle import ref_flac
from tests import ref_ts

_i32, _ptr = ref_flac._i32, ref_flac._ptr


def streams(path):
    """[{id, kind, codec}] in FFmpeg's stream order"""
    fmt = ref_flac.libs()[0]
    ctx = _open(path)
    try:
        _, codec, _ = ref_flac.libs()
        out = []
        for i in range(_i32(ctx.value + 44)):
            st = _ptr(_ptr(ctx.value + 48) + 8 * i)
            assert _i32(st + 8) == i, 'AVStream.index'
            par = _ptr(st + 16)
            out.append(dict(id=_i32(st + 12), kind=ref_ts.AVMEDIA_TYPES.get(_i32(par), 'other'),
                            codec=codec.avcodec_get_name(_i32(par + 4)).decode()))
        return out
    finally:
        fmt.avformat_close_input(ctypes.byref(ctx))


def _open(path):
    ctx = ref_ts._open(path, True)
    return ctx


def packets(path, index):
    """the bytes of every packet of stream `index`, in order"""
    return [d for i, d in ref_ts.packets(path) if i == index]
