"""Independent MP4 / QuickTime demuxer and decoder for the tests: FFmpeg's mov demuxer and its decoders, driven through
ctypes on the libraries oracle/ref_flac.py loads.

`demux(path)` gives the stream list (media type, codec name, default disposition), the chapters (start in seconds,
from each chapter's own time base) and every packet (stream, bytes, file position).  `decode(path, sid, channels)`
decodes one stream's packets, skipping a packet the decoder refuses as the ffmpeg command line does, and asserts
the sample format it reads.  Struct offsets, as in tests/ref_mkv.py (libavformat / libavcodec 62):
    AVFormatContext.nb_streams +44, .streams +48, .nb_chapters +72, .chapters +80;
    AVStream.index +8, .codecpar +16, .disposition +64;  AVCodecParameters.codec_type +0, .codec_id +4;
    AVPacket.data +24, .size +32, .stream_index +36, .pos +72;  AVChapter.time_base +8, .start +16;
    AVFrame.data[] +0, .nb_samples +112, .format +116.
Test infrastructure only: the product never imports this."""
import ctypes

import numpy as np

from oracle import ref_flac

AVMEDIA_TYPES = {0: 'video', 1: 'audio', 2: 'data', 3: 'subtitles', 4: 'attachment'}
AV_DISPOSITION_DEFAULT = 1
FORMATS = {1: (np.int16, False), 2: (np.int32, False), 6: (np.int16, True), 7: (np.int32, True)}


def _i32(addr):
    return ctypes.c_int32.from_address(addr).value


def _i64(addr):
    return ctypes.c_int64.from_address(addr).value


def _ptr(addr):
    return ctypes.c_void_p.from_address(addr).value


class Demuxed(object):
    def __init__(self, streams, chapters, packets):
        self.streams, self.chapters, self.packets = streams, chapters, packets

    def track(self, sid):
        return [(p[1], p[2]) for p in self.packets if p[0] == sid]


def _open(path):
    fmt, codec, _ = ref_flac.libs()
    codec.avcodec_get_name.argtypes = [ctypes.c_int]
    codec.avcodec_get_name.restype = ctypes.c_char_p
    ctx = ctypes.c_void_p()
    rc = fmt.avformat_open_input(ctypes.byref(ctx), path.encode(), None, None)
    if rc < 0:
        raise RuntimeError('avformat_open_input(%s) failed: %d' % (path, rc))
    return ctx


def demux(path, packets=True):
    fmt, codec, _ = ref_flac.libs()
    ctx = _open(path)
    pkt = ctypes.c_void_p()
    try:
        base = ctx.value
        nb = _i32(base + 44)
        streams = []
        for i in range(nb):
            st = _ptr(_ptr(base + 48) + 8 * i)
            assert _i32(st + 8) == i, 'AVStream.index'
            par = _ptr(st + 16)
            streams.append((AVMEDIA_TYPES.get(_i32(par), 'other'), codec.avcodec_get_name(_i32(par + 4)).decode(),
                            bool(_i32(st + 64) & AV_DISPOSITION_DEFAULT)))
        chapters = []
        for i in range(_i32(base + 72)):
            ch = _ptr(_ptr(base + 80) + 8 * i)
            num, den = _i32(ch + 8), _i32(ch + 12)
            assert num > 0 and den > 0, 'AVChapter.time_base'
            chapters.append(float('%f' % (_i64(ch + 16) * num / den)))
        out = []
        if packets:
            pkt = ctypes.c_void_p(codec.av_packet_alloc())
            while fmt.av_read_frame(ctx, pkt) >= 0:
                p = pkt.value
                sid, size = _i32(p + 36), _i32(p + 32)
                assert 0 <= sid < nb and size >= 0, 'AVPacket.stream_index / size'
                out.append((sid, ctypes.string_at(_ptr(p + 24), size) if size else b'', _i64(p + 72)))
                codec.av_packet_unref(pkt)
        return Demuxed(streams, chapters, out)
    finally:
        if pkt:
            codec.av_packet_free(ctypes.byref(pkt))
        fmt.avformat_close_input(ctypes.byref(ctx))


def decode(path, sid, channels):
    """-> (samples (n, channels) int64 as FFmpeg returns them, sample format, packets refused)."""
    fmt, codec, util = ref_flac.libs()
    ctx = _open(path)
    dec = pkt = frame = ctypes.c_void_p()
    chunks, sfmt, refused = [], None, 0
    try:
        fmt.avformat_find_stream_info(ctx, None)
        par = _ptr(_ptr(_ptr(ctx.value + 48) + 8 * sid) + 16)
        c = codec.avcodec_find_decoder(_i32(par + 4))
        assert c, 'no decoder'
        dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
        assert codec.avcodec_parameters_to_context(dec, par) >= 0
        assert codec.avcodec_open2(dec, c, None) >= 0
        pkt = ctypes.c_void_p(codec.av_packet_alloc())
        frame = ctypes.c_void_p(util.av_frame_alloc())

        def drain():
            nonlocal sfmt
            while codec.avcodec_receive_frame(dec, frame) == 0:
                n, f = _i32(frame.value + 112), _i32(frame.value + 116)
                assert f in FORMATS, 'unexpected sample format %d' % f
                assert sfmt in (None, f)
                sfmt = f
                dt, planar = FORMATS[f]
                size = np.dtype(dt).itemsize
                if planar:
                    planes = [np.frombuffer((ctypes.c_char * (n * size)).from_address(_ptr(frame.value + 8 * ch)), dt)
                              for ch in range(channels)]
                    chunks.append(np.stack(planes, 1).astype(np.int64))
                else:
                    buf = (ctypes.c_char * (n * channels * size)).from_address(_ptr(frame.value))
                    chunks.append(np.frombuffer(buf, dt).astype(np.int64).reshape(n, channels))
        while fmt.av_read_frame(ctx, pkt) >= 0:
            if _i32(pkt.value + 36) == sid:
                if codec.avcodec_send_packet(dec, pkt) < 0:
                    refused += 1
                drain()
            codec.av_packet_unref(pkt)
        codec.avcodec_send_packet(dec, None)
        drain()
    finally:
        if frame:
            util.av_frame_free(ctypes.byref(frame))
        if pkt:
            codec.av_packet_free(ctypes.byref(pkt))
        if dec:
            codec.avcodec_free_context(ctypes.byref(dec))
        fmt.avformat_close_input(ctypes.byref(ctx))
    out = np.concatenate(chunks) if chunks else np.zeros((0, channels), np.int64)
    return out, sfmt, refused


def decode_pcm(path, sid, channels, bits):
    """The decoded samples at their own bit depth (S32 samples shifted down), with the refused packet count."""
    out, sfmt, refused = decode(path, sid, channels)
    if sfmt in (2, 7):
        out = out >> (32 - bits)
    return out, refused
