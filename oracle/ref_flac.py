"""Independent FLAC decoder for the tests: FFmpeg's libavformat / libavcodec, driven through ctypes.

The opencv-python wheel ships FFmpeg's libraries (libavformat / libavcodec / libavutil, major version 62) in
`opencv_python_headless.libs/` beside `cv2/`; cv2 itself cannot read audio, so the calls go to the libraries directly:
avformat_open_input, then av_read_frame -> avcodec_send_packet -> avcodec_receive_frame until the end, and a drain.
Only a few struct fields are read, at their offsets in these library versions:
    AVFormatContext.nb_streams +44, .streams +48;  AVStream.codecpar +16;
    AVCodecParameters.codec_type +0, .codec_id +4;  AVPacket.stream_index +36;
    AVFrame.data[0..7] +0, .nb_samples +112, .format +116.
`decode` asserts the decoded sample count, so a wrong offset fails loudly instead of returning garbage.

FFmpeg returns 16-bit FLAC as AV_SAMPLE_FMT_S16 and 24-bit FLAC as AV_SAMPLE_FMT_S32 with the sample in the top 24
bits (interleaved; the planar formats are handled too).  Test infrastructure only: the product never imports this."""
import ctypes
import glob
import os

import numpy as np

AV_SAMPLE_FMT_S16, AV_SAMPLE_FMT_S32, AV_SAMPLE_FMT_S16P, AV_SAMPLE_FMT_S32P = 1, 2, 6, 7
AVERROR_EAGAIN = -11
AVMEDIA_TYPE_AUDIO = 1
_libs = None


def _find_libs():
    import cv2
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(cv2.__file__))), 'opencv_python_headless.libs')
    found = {}
    for name in ('avutil', 'avcodec', 'avformat'):
        hits = sorted(glob.glob(os.path.join(d, 'lib%s-*.so*' % name)))
        if not hits:
            raise RuntimeError('lib%s not found in %s' % (name, d))
        found[name] = hits[0]
    return found


def libs():
    """(libavformat, libavcodec, libavutil) with the prototypes this module uses."""
    global _libs
    if _libs is not None:
        return _libs
    paths = _find_libs()
    util = ctypes.CDLL(paths['avutil'], mode=ctypes.RTLD_GLOBAL)
    codec = ctypes.CDLL(paths['avcodec'], mode=ctypes.RTLD_GLOBAL)
    fmt = ctypes.CDLL(paths['avformat'], mode=ctypes.RTLD_GLOBAL)
    vp, vpp = ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)
    fmt.avformat_open_input.argtypes = [vpp, ctypes.c_char_p, vp, vp]
    fmt.avformat_open_input.restype = ctypes.c_int
    fmt.avformat_find_stream_info.argtypes = [vp, vp]
    fmt.avformat_find_stream_info.restype = ctypes.c_int
    fmt.av_read_frame.argtypes = [vp, vp]
    fmt.av_read_frame.restype = ctypes.c_int
    fmt.avformat_close_input.argtypes = [vpp]
    codec.avcodec_find_decoder.argtypes = [ctypes.c_int]
    codec.avcodec_find_decoder.restype = vp
    codec.avcodec_alloc_context3.argtypes = [vp]
    codec.avcodec_alloc_context3.restype = vp
    codec.avcodec_parameters_to_context.argtypes = [vp, vp]
    codec.avcodec_parameters_to_context.restype = ctypes.c_int
    codec.avcodec_open2.argtypes = [vp, vp, vp]
    codec.avcodec_open2.restype = ctypes.c_int
    codec.avcodec_send_packet.argtypes = [vp, vp]
    codec.avcodec_send_packet.restype = ctypes.c_int
    codec.avcodec_receive_frame.argtypes = [vp, vp]
    codec.avcodec_receive_frame.restype = ctypes.c_int
    codec.avcodec_free_context.argtypes = [vpp]
    codec.av_packet_alloc.restype = vp
    codec.av_packet_unref.argtypes = [vp]
    codec.av_packet_free.argtypes = [vpp]
    util.av_frame_alloc.restype = vp
    util.av_frame_free.argtypes = [vpp]
    util.av_log_set_level.argtypes = [ctypes.c_int]
    util.av_log_set_level(-8)                 # AV_LOG_QUIET: an undecodable attached picture is not our concern
    _libs = (fmt, codec, util)
    return _libs


def _i32(addr):
    return ctypes.c_int32.from_address(addr).value


def _ptr(addr):
    return ctypes.c_void_p.from_address(addr).value


def decode(path, channels, expected_frames):
    """-> (samples, format): (expected_frames, channels) int32 as FFmpeg returns them (S16 values, or S32 values with
    the sample in the top bits), and FFmpeg's sample format."""
    fmt, codec, util = libs()
    ctx = ctypes.c_void_p()
    rc = fmt.avformat_open_input(ctypes.byref(ctx), path.encode(), None, None)
    if rc < 0:
        raise RuntimeError('avformat_open_input(%s) failed: %d' % (path, rc))
    dec = pkt = frame = ctypes.c_void_p()
    chunks, sfmt = [], None
    try:
        if fmt.avformat_find_stream_info(ctx, None) < 0:
            raise RuntimeError('avformat_find_stream_info failed')
        # the audio stream (an attached PICTURE block shows up as a video stream)
        nb = _i32(ctx.value + 44)
        pars = [_ptr(_ptr(_ptr(ctx.value + 48) + 8 * i) + 16) for i in range(nb)]
        audio = [i for i in range(nb) if _i32(pars[i]) == AVMEDIA_TYPE_AUDIO]
        assert len(audio) == 1, 'expected one audio stream among %d' % nb
        index, par = audio[0], pars[audio[0]]
        codec_id = _i32(par + 4)
        c = codec.avcodec_find_decoder(codec_id)
        assert c, 'no decoder for codec id %d' % codec_id
        dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
        assert codec.avcodec_parameters_to_context(dec, par) >= 0
        assert codec.avcodec_open2(dec, c, None) >= 0
        pkt = ctypes.c_void_p(codec.av_packet_alloc())
        frame = ctypes.c_void_p(util.av_frame_alloc())

        def drain():
            nonlocal sfmt
            while codec.avcodec_receive_frame(dec, frame) == 0:
                n = _i32(frame.value + 112)
                f = _i32(frame.value + 116)
                assert sfmt in (None, f)
                sfmt = f
                if f in (AV_SAMPLE_FMT_S16, AV_SAMPLE_FMT_S32):
                    dt = np.int16 if f == AV_SAMPLE_FMT_S16 else np.int32
                    buf = (ctypes.c_char * (n * channels * np.dtype(dt).itemsize)).from_address(_ptr(frame.value))
                    chunks.append(np.frombuffer(buf, dt).astype(np.int32).reshape(n, channels).copy())
                elif f in (AV_SAMPLE_FMT_S16P, AV_SAMPLE_FMT_S32P):
                    dt = np.int16 if f == AV_SAMPLE_FMT_S16P else np.int32
                    planes = []
                    for ch in range(channels):
                        buf = (ctypes.c_char * (n * np.dtype(dt).itemsize)).from_address(_ptr(frame.value + 8 * ch))
                        planes.append(np.frombuffer(buf, dt).astype(np.int32))
                    chunks.append(np.stack(planes, 1))
                else:
                    raise AssertionError('unexpected sample format %d' % f)
        while fmt.av_read_frame(ctx, pkt) >= 0:
            if _i32(pkt.value + 36) != index:
                codec.av_packet_unref(pkt)
                continue
            rc = codec.avcodec_send_packet(dec, pkt)
            codec.av_packet_unref(pkt)
            if rc < 0 and rc != AVERROR_EAGAIN:
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
    out = np.concatenate(chunks) if chunks else np.zeros((0, channels), np.int32)
    assert out.shape == (expected_frames, channels), (out.shape, expected_frames, channels)
    return out, sfmt


def decode_pcm(path, channels, bits, expected_frames):
    """The decoded samples at their own bit depth, (frames, channels) int64."""
    out, sfmt = decode(path, channels, expected_frames)
    out = out.astype(np.int64)
    if sfmt in (AV_SAMPLE_FMT_S32, AV_SAMPLE_FMT_S32P):
        out >>= 32 - bits
    elif bits != 16:
        raise AssertionError('%d-bit FLAC came back as 16-bit samples' % bits)
    return out
