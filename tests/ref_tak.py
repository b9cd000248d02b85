"""FFmpeg's TAK demuxing and decoding for the tests, through the ctypes driver of tests/ref_mp4.py (libavformat /
libavcodec 62): `packets(path)` are the tak demuxer's packets (cut by FFmpeg's tak parser) with their file positions,
`decode(path, channels, bits)` the `tak` decoder's samples at their own width with the count of packets it refused, or
the reason it gave none.  FFmpeg's decoder gives S16P for 16-bit streams and S32P, the sample in the top 24 bits, for
24-bit ones.  Test infrastructure only."""
from tests import ref_ape, ref_mp4


def packets(path):
    """[(file position, packet bytes)] of the stream"""
    return [(pos, data) for data, pos in ref_mp4.demux(path).track(0)]


def decode(path, channels, bits):
    """(samples (n, channels) int64 at `bits` bits, packets FFmpeg's decoder refused), or (None, why): 'demux' when its
    demuxer refuses the file, 'open' when its decoder does not open, 'U8' for its unsigned 8-bit output"""
    return ref_ape.decode(path, channels, bits)


def layout(path):
    """the channel mask of FFmpeg's decoder after it decoded the stream (its default layout when it reports none): the
    layout the ffmpeg command line hands libswresample"""
    return ref_mp4._decode(path, 0, None)[3]


def crc_refusals(path):
    """(packets FFmpeg's decoder refuses, frames it returns) under `err_detect crccheck+explode`"""
    return ref_ape.crc_refusals(path)
