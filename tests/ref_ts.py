"""FFmpeg's mpegts demuxer and its pcm_bluray / truehd decoders for the tests: libavformat / libavcodec from the opencv
wheel (oracle/ref_flac.libs()), driven through ctypes.

`streams(path, find_info)` gives FFmpeg's stream list, after avformat_open_input alone or also after
avformat_find_stream_info (`ffmpeg -i` runs both); `packets(path)` every packet (stream index, bytes); `decode(path,
index, channels)` the samples FFmpeg's decoder returns for one stream, as int16 (S16 as it is, S32 its top 16 bits).
Only a few struct fields are read, at their offsets in these library versions (libavformat / libavcodec 62):
    AVFormatContext.nb_streams +44, .streams +48;  AVStream.index +8, .id +12, .codecpar +16, .time_base +32,
    .disposition +64;  AVCodecParameters.codec_type +0, .codec_id +4;  AVPacket.data +24, .size +32, .stream_index +36;
    AVFrame.data[0] +0, .nb_samples +112, .format +116.
Each is asserted against something known: a stream's index is its position, its id is the PID the writer gave it,
its time base is 1/90000, a packet's stream index is in range, a frame's format is S16 or S32.  Test infrastructure
only: the product never imports this."""
import ctypes

import numpy as np

from oracle import ref_flac

AVMEDIA_TYPES = {0: 'video', 1: 'audio', 2: 'data', 3: 'subtitles', 4: 'attachment'}
AV_DISPOSITION_DEFAULT = 1
AV_SAMPLE_FMT_S16, AV_SAMPLE_FMT_S32 = 1, 2
_i32, _ptr = ref_flac._i32, ref_flac._ptr


def _open(path, find_info):
    fmt, codec, util = ref_flac.libs()
    codec.avcodec_get_name.argtypes = [ctypes.c_int]
    codec.avcodec_get_name.restype = ctypes.c_char_p
    ctx = ctypes.c_void_p()
    rc = fmt.avformat_open_input(ctypes.byref(ctx), str(path).encode(), None, None)
    if rc < 0:
        raise RuntimeError('avformat_open_input(%s) failed: %d' % (path, rc))
    if find_info and fmt.avformat_find_stream_info(ctx, None) < 0:
        fmt.avformat_close_input(ctypes.byref(ctx))
        raise RuntimeError('avformat_find_stream_info failed')
    return ctx


def _streams(ctx):
    _, codec, _ = ref_flac.libs()
    out = []
    nb = _i32(ctx.value + 44)
    for i in range(nb):
        st = _ptr(_ptr(ctx.value + 48) + 8 * i)
        assert _i32(st + 8) == i, 'AVStream.index'
        assert (_i32(st + 32), _i32(st + 36)) == (1, 90000), 'AVStream.time_base'
        par = _ptr(st + 16)
        out.append(dict(pid=_i32(st + 12), kind=AVMEDIA_TYPES.get(_i32(par), 'other'),
                        codec=codec.avcodec_get_name(_i32(par + 4)).decode(),
                        default=bool(_i32(st + 64) & AV_DISPOSITION_DEFAULT), par=par))
    return out


def streams(path, find_info=False):
    """[{pid, kind, codec, default}] in FFmpeg's stream order."""
    fmt = ref_flac.libs()[0]
    ctx = _open(path, find_info)
    try:
        return [{k: v for k, v in s.items() if k != 'par'} for s in _streams(ctx)]
    finally:
        fmt.avformat_close_input(ctypes.byref(ctx))


def packets(path):
    """[(stream index, bytes)] as av_read_frame returns them (after avformat_find_stream_info)."""
    fmt, codec, _ = ref_flac.libs()
    ctx = _open(path, True)
    pkt = ctypes.c_void_p(codec.av_packet_alloc())
    out = []
    try:
        nb = _i32(ctx.value + 44)
        while fmt.av_read_frame(ctx, pkt) >= 0:
            sid, size = _i32(pkt.value + 36), _i32(pkt.value + 32)
            assert 0 <= sid < nb and size >= 0, 'AVPacket.stream_index / size'
            out.append((sid, ctypes.string_at(_ptr(pkt.value + 24), size) if size else b''))
            codec.av_packet_unref(pkt)
    finally:
        codec.av_packet_free(ctypes.byref(pkt))
        fmt.avformat_close_input(ctypes.byref(ctx))
    return out


def decode(path, index, channels):
    """(frames, channels) int16: the top 16 bits of what FFmpeg's decoder returns for stream `index`.  Packets the
    decoder refuses are skipped, as the ffmpeg command line skips them."""
    fmt, codec, util = ref_flac.libs()
    ctx = _open(path, True)
    dec = pkt = frame = ctypes.c_void_p()
    chunks = []
    try:
        par = _streams(ctx)[index]['par']
        c = codec.avcodec_find_decoder(_i32(par + 4))
        assert c
        dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
        assert codec.avcodec_parameters_to_context(dec, par) >= 0
        assert codec.avcodec_open2(dec, c, None) >= 0
        pkt = ctypes.c_void_p(codec.av_packet_alloc())
        frame = ctypes.c_void_p(util.av_frame_alloc())

        def drain():
            while codec.avcodec_receive_frame(dec, frame) == 0:
                n, f = _i32(frame.value + 112), _i32(frame.value + 116)
                assert f in (AV_SAMPLE_FMT_S16, AV_SAMPLE_FMT_S32), 'unexpected sample format %d' % f
                width = 2 if f == AV_SAMPLE_FMT_S16 else 4
                buf = (ctypes.c_char * (n * channels * width)).from_address(_ptr(frame.value))
                a = np.frombuffer(buf, np.int16 if width == 2 else np.int32).reshape(n, channels)
                chunks.append(a.copy() if width == 2 else (a >> 16).astype(np.int16))
        while fmt.av_read_frame(ctx, pkt) >= 0:
            if _i32(pkt.value + 36) != index:
                codec.av_packet_unref(pkt)
                continue
            codec.avcodec_send_packet(dec, pkt)
            codec.av_packet_unref(pkt)
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
    return np.concatenate(chunks) if chunks else np.zeros((0, channels), np.int16)


def same_up_to_channel_order(a, b):
    """True when b's columns are a's in some order (FFmpeg returns some BD-LPCM layouts reordered)."""
    if a.shape != b.shape:
        return False
    used = set()
    for c in range(a.shape[1]):
        match = next((d for d in range(b.shape[1]) if d not in used and np.array_equal(a[:, c], b[:, d])), None)
        if match is None:
            return False
        used.add(match)
    return True
