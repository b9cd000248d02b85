"""Independent Matroska demuxer for the tests: FFmpeg's libavformat, driven through ctypes (the libraries of the
opencv-python wheel, loaded by oracle/ref_flac.py).

`demux(path)` opens the file with avformat_open_input and reads every packet with av_read_frame, giving the stream
list (media type, codec name, default disposition, time base), every packet (stream, pts, duration, bytes) and the
chapters (start, time base).  Only a few struct fields are read, at their offsets in these library versions
(libavformat / libavcodec 62):
    AVFormatContext.nb_streams +44, .streams +48, .nb_chapters +72, .chapters +80;
    AVStream.index +8, .codecpar +16, .time_base +32, .disposition +64;  AVCodecParameters.codec_type +0, .codec_id +4;
    AVPacket.pts +8, .data +24, .size +32, .stream_index +36, .duration +64;  AVChapter.id +0, .time_base +8, .start +16.
Each is asserted against something known (a stream's index is its position; a track's time base is the file's
TimestampScale over 10^9 (FFmpeg lists attachments as streams after the tracks); a chapter's time base is 1/10^9; a
packet's stream index is in range), so a wrong offset fails loudly instead of returning garbage.  Test infrastructure only: the product never imports this."""
import ctypes
from fractions import Fraction

from oracle import ref_flac

AVMEDIA_TYPES = {0: 'video', 1: 'audio', 3: 'subtitles', 4: 'attachment'}
AV_DISPOSITION_DEFAULT = 1
AV_NOPTS_VALUE = -(1 << 63)


def _i32(addr):
    return ctypes.c_int32.from_address(addr).value


def _i64(addr):
    return ctypes.c_int64.from_address(addr).value


def _ptr(addr):
    return ctypes.c_void_p.from_address(addr).value


class Demuxed(object):
    """streams: [(type, codec name, default)]; packets: [(stream, pts in ns or None, duration in ns, bytes)];
    chapters: [start in ns]."""

    def __init__(self, streams, packets, chapters):
        self.streams, self.packets, self.chapters = streams, packets, chapters

    def track(self, sid):
        return [(p[3], p[1]) for p in self.packets if p[0] == sid]


def demux(path, timestamp_scale):
    fmt, codec, _ = ref_flac.libs()
    codec.avcodec_get_name.argtypes = [ctypes.c_int]
    codec.avcodec_get_name.restype = ctypes.c_char_p
    ctx = ctypes.c_void_p()
    rc = fmt.avformat_open_input(ctypes.byref(ctx), path.encode(), None, None)
    if rc < 0:
        raise RuntimeError('avformat_open_input(%s) failed: %d' % (path, rc))
    pkt = ctypes.c_void_p()
    try:
        base = ctx.value
        nb = _i32(base + 44)
        streams, tbs = [], []
        want_tb = Fraction(timestamp_scale, 10 ** 9)
        for i in range(nb):
            st = _ptr(_ptr(base + 48) + 8 * i)
            assert _i32(st + 8) == i, 'AVStream.index'
            par = _ptr(st + 16)
            tb = Fraction(_i32(st + 32), _i32(st + 36))
            kind = AVMEDIA_TYPES.get(_i32(par), 'other')
            assert tb == want_tb or kind == 'attachment', ('AVStream.time_base', tb, want_tb)
            tbs.append(tb)
            streams.append((kind, codec.avcodec_get_name(_i32(par + 4)).decode(),
                            bool(_i32(st + 64) & AV_DISPOSITION_DEFAULT)))
        chapters = []
        for i in range(_i32(base + 72)):
            ch = _ptr(_ptr(base + 80) + 8 * i)
            assert (_i32(ch + 8), _i32(ch + 12)) == (1, 10 ** 9), 'AVChapter.time_base'
            assert _i64(ch) != 0, 'AVChapter.id'
            chapters.append(_i64(ch + 16))
        packets = []
        pkt = ctypes.c_void_p(codec.av_packet_alloc())
        while fmt.av_read_frame(ctx, pkt) >= 0:
            p = pkt.value
            sid, size = _i32(p + 36), _i32(p + 32)
            assert 0 <= sid < nb and size >= 0, 'AVPacket.stream_index / size'
            pts = _i64(p + 8)
            data = ctypes.string_at(_ptr(p + 24), size) if size else b''
            packets.append((sid, None if pts == AV_NOPTS_VALUE else int(pts * tbs[sid] * 10 ** 9),
                            int(_i64(p + 64) * tbs[sid] * 10 ** 9), data))
            codec.av_packet_unref(pkt)
        return Demuxed(streams, packets, chapters)
    finally:
        if pkt:
            codec.av_packet_free(ctypes.byref(pkt))
        fmt.avformat_close_input(ctypes.byref(ctx))
