"""FFmpeg's TrueHD decoder for the tests: libavformat / libavcodec from the opencv wheel, driven through ctypes with the
prototypes and struct offsets of oracle/ref_flac.py (whose `decode` this follows).  A raw stream is opened with the
`truehd` demuxer named explicitly (its probe gives short streams a low score); a Matroska file goes through the
Matroska demuxer.  FFmpeg returns TrueHD as AV_SAMPLE_FMT_S32 with the 24-bit sample in the top bits; `decode` returns
the samples shifted down to their 24-bit values, in FFmpeg's channel order.  Test infrastructure only."""
import ctypes

import numpy as np

from oracle import ref_flac

AV_SAMPLE_FMT_S32 = 2
AVMEDIA_TYPE_AUDIO = 1


def _lib():
    fmt, codec, util = ref_flac.libs()
    fmt.av_find_input_format.argtypes = [ctypes.c_char_p]
    fmt.av_find_input_format.restype = ctypes.c_void_p
    return fmt, codec, util


def decode(path, channels, raw=None, log_level=None):
    """-> (frames, channels) int64 24-bit samples FFmpeg's decoder returns.  raw: open with the `truehd` demuxer
    (default: when the name ends in .thd).  Raises RuntimeError when FFmpeg refuses a packet."""
    fmt, codec, util = _lib()
    if log_level is not None:
        util.av_log_set_level(log_level)
    if raw is None:
        raw = str(path).endswith('.thd')
    ifmt = fmt.av_find_input_format(b'truehd') if raw else None
    ctx = ctypes.c_void_p()
    rc = fmt.avformat_open_input(ctypes.byref(ctx), str(path).encode(), ifmt, None)
    if rc < 0:
        raise RuntimeError('avformat_open_input(%s) failed: %d' % (path, rc))
    dec = pkt = frame = ctypes.c_void_p()
    chunks = []
    try:
        if fmt.avformat_find_stream_info(ctx, None) < 0:
            raise RuntimeError('avformat_find_stream_info failed')
        nb = ref_flac._i32(ctx.value + 44)
        pars = [ref_flac._ptr(ref_flac._ptr(ref_flac._ptr(ctx.value + 48) + 8 * i) + 16) for i in range(nb)]
        audio = [i for i in range(nb) if ref_flac._i32(pars[i]) == AVMEDIA_TYPE_AUDIO]
        assert len(audio) == 1, 'expected one audio stream among %d' % nb
        index, par = audio[0], pars[audio[0]]
        c = codec.avcodec_find_decoder(ref_flac._i32(par + 4))
        assert c
        dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
        assert codec.avcodec_parameters_to_context(dec, par) >= 0
        assert codec.avcodec_open2(dec, c, None) >= 0
        pkt = ctypes.c_void_p(codec.av_packet_alloc())
        frame = ctypes.c_void_p(util.av_frame_alloc())

        def drain():
            while codec.avcodec_receive_frame(dec, frame) == 0:
                n, f = ref_flac._i32(frame.value + 112), ref_flac._i32(frame.value + 116)
                assert f == AV_SAMPLE_FMT_S32, 'unexpected sample format %d' % f
                buf = (ctypes.c_char * (n * channels * 4)).from_address(ref_flac._ptr(frame.value))
                chunks.append(np.frombuffer(buf, np.int32).reshape(n, channels).astype(np.int64) >> 8)
        while fmt.av_read_frame(ctx, pkt) >= 0:
            if ref_flac._i32(pkt.value + 36) != index:
                codec.av_packet_unref(pkt)
                continue
            rc = codec.avcodec_send_packet(dec, pkt)
            codec.av_packet_unref(pkt)
            if rc < 0 and rc != ref_flac.AVERROR_EAGAIN:
                raise RuntimeError('avcodec_send_packet failed: %d' % rc)
            drain()
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
        if log_level is not None:
            util.av_log_set_level(-8)
    return np.concatenate(chunks) if chunks else np.zeros((0, channels), np.int64)
