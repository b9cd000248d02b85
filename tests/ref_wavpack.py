"""FFmpeg's WavPack demuxing and decoding for the tests, through the ctypes driver of tests/ref_mp4.py (libavformat /
libavcodec 62): `packets(path)` are the wv or Matroska demuxer's packets split back into blocks, `decode(path, channels,
bits)` the `wavpack` decoder's samples at their own width with the count of packets it refused.  FFmpeg's decoder gives
S16P for 2-byte streams and S32P, the sample in the top bits, for 3-byte ones.  Test infrastructure only."""
import struct

from tests import ref_mp4


def packets(path):
    """[(file position, [(block_samples, flags, crc, sub-block bytes)])]: one entry per packet, its blocks in order"""
    out = []
    for data, pos in ref_mp4.demux(path).track(0):
        blocks, at = [], 0
        while at + 32 <= len(data):
            assert data[at:at + 4] == b'wvpk'
            size = struct.unpack_from('<I', data, at + 4)[0] + 8
            count, flags, crc = struct.unpack_from('<III', data, at + 20)
            blocks.append((count, flags, crc, data[at + 32:at + size]))
            at += size
        assert at == len(data)
        out.append((pos, blocks))
    return out


def decode(path, channels, bits):
    """(samples (n, channels) int64 at `bits` bits, packets FFmpeg's decoder refused)"""
    return ref_mp4.decode_pcm(path, 0, channels, bits)
