"""FFmpeg's APE demuxing and decoding for the tests, through the ctypes driver of tests/ref_mp4.py (libavformat /
libavcodec 62): `packets(path)` are the ape demuxer's packets with their file positions, `decode(path, channels, bits)`
the `ape` decoder's samples at their own width with the count of packets it refused, or the reason it gave none.
FFmpeg's decoder gives S16P for 16-bit streams and S32P, the sample in the top 24 bits, for 24-bit ones.  Each packet
is the demuxer's 8-byte prefix (block count and skip, little-endian) and the frame's 32-bit words.  Test
infrastructure only."""
from tests import ref_mp4


def packets(path):
    """[(file position, packet bytes)] of the stream"""
    return [(pos, data) for data, pos in ref_mp4.demux(path).track(0)]


def decode(path, channels, bits):
    """(samples (n, channels) int64 at `bits` bits, packets FFmpeg's decoder refused), or (None, why) when FFmpeg
    gives no samples at all: 'demux' when its demuxer refuses the file, 'open' when its decoder does not open, 'U8'
    for its unsigned 8-bit output"""
    try:
        return ref_mp4.decode_pcm(path, 0, channels, bits)
    except RuntimeError as e:
        if 'avformat_open_input' not in str(e):
            raise
        return None, 'demux'
    except AssertionError as e:
        text = str(e)
        if 'unexpected sample format' in text and ' 5' in text:
            return None, 'U8'
        if not text:                           # avcodec_open2 failed
            return None, 'open'
        raise


def crc_refusals(path):
    """(packets FFmpeg's decoder refuses, frames it returns) with `err_detect crccheck+explode` set on the decoder, so
    that a frame whose CRC disagrees is refused rather than only logged: FFmpeg's own test of the frame CRC."""
    import ctypes
    from oracle import ref_flac
    fmt, codec, util = ref_flac.libs()
    util.av_opt_set.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    util.av_opt_set.restype = ctypes.c_int
    ctx = ref_mp4._open(path)
    dec = pkt = frame = ctypes.c_void_p()
    refused = frames = 0
    try:
        fmt.avformat_find_stream_info(ctx, None)
        par = ref_mp4._ptr(ref_mp4._ptr(ref_mp4._ptr(ctx.value + 48)) + 16)
        c = codec.avcodec_find_decoder(ref_mp4._i32(par + 4))
        dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
        assert codec.avcodec_parameters_to_context(dec, par) >= 0
        assert util.av_opt_set(dec, b'err_detect', b'crccheck+explode', 0) >= 0
        assert codec.avcodec_open2(dec, c, None) >= 0
        pkt = ctypes.c_void_p(codec.av_packet_alloc())
        frame = ctypes.c_void_p(util.av_frame_alloc())

        def drain():
            nonlocal refused, frames
            while True:
                rc = codec.avcodec_receive_frame(dec, frame)
                if rc == 0:
                    frames += ref_mp4._i32(frame.value + 112)
                    continue
                if rc not in (-11, -541478725):          # EAGAIN, EOF: nothing more for now
                    refused += 1
                    continue
                return

        while fmt.av_read_frame(ctx, pkt) >= 0:
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
    return refused, frames
