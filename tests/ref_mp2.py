"""FFmpeg's `mp2` decoder (the fixed-point one, libavcodec 62 from the opencv wheel, oracle/ref_flac.libs()) for the
tests, driven through ctypes: `decode_packets(packets)` sends each byte string as one packet, as a demuxer with
FFmpeg's MPEG audio parser hands frames over, and returns the samples with the decoder's sample format, channel
layout and rate.  The decoder returns S16P (planar); AVFrame.data[] +0, .nb_samples +112, .format +116 are read, and
the format is asserted.  Test infrastructure only: the product never imports this."""
import ctypes

import numpy as np

from oracle import ref_flac
from tests import ref_mp4

AV_SAMPLE_FMT_S16P = 6


def _decoder():
    fmt, codec, util = ref_flac.libs()
    codec.avcodec_find_decoder_by_name.argtypes = [ctypes.c_char_p]
    codec.avcodec_find_decoder_by_name.restype = ctypes.c_void_p
    codec.av_new_packet.argtypes = [ctypes.c_void_p, ctypes.c_int]
    return codec, util, codec.avcodec_find_decoder_by_name(b'mp2')


def decode_packets(packets):
    """-> (samples (n, channels) int16, channel mask, rate, packets refused)"""
    codec, util, c = _decoder()
    dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
    pkt = ctypes.c_void_p(codec.av_packet_alloc())
    frame = ctypes.c_void_p(util.av_frame_alloc())
    chunks, refused, channels = [], 0, None
    try:
        assert codec.avcodec_open2(dec, c, None) >= 0

        def drain():
            nonlocal channels
            while codec.avcodec_receive_frame(dec, frame) == 0:
                n, f = ref_flac._i32(frame.value + 112), ref_flac._i32(frame.value + 116)
                assert f == AV_SAMPLE_FMT_S16P, f
                channels = ref_mp4.decoder_layout(dec)[1]
                planes = [np.frombuffer((ctypes.c_char * (2 * n)).from_address(ref_flac._ptr(frame.value + 8 * ch)),
                                        np.int16) for ch in range(channels)]
                chunks.append(np.stack(planes, 1).copy())
        for p in packets:
            assert codec.av_new_packet(pkt, len(p)) == 0
            ctypes.memmove(ref_flac._ptr(pkt.value + 24), p, len(p))
            if codec.avcodec_send_packet(dec, pkt) < 0:
                refused += 1
            codec.av_packet_unref(pkt)
            drain()
        codec.avcodec_send_packet(dec, None)
        drain()
        mask = ref_mp4.decoder_layout(dec)[0]
        rate = ctypes.c_int64()
        util.av_opt_get_int.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int64)]
        assert util.av_opt_get_int(dec, b'ar', 0, ctypes.byref(rate)) >= 0
    finally:
        util.av_frame_free(ctypes.byref(frame))
        codec.av_packet_free(ctypes.byref(pkt))
        codec.avcodec_free_context(ctypes.byref(dec))
    out = np.concatenate(chunks) if chunks else np.zeros((0, channels or 1), np.int16)
    return out, mask, rate.value, refused
