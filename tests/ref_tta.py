"""FFmpeg's TTA demuxing and decoding for the tests, through the ctypes driver of tests/ref_mp4.py (libavformat /
libavcodec 62): `packets(path)` are the tta or Matroska demuxer's packets with their file positions, `decode(path,
channels, bits)` the `tta` decoder's samples at their own width with the count of packets it refused, or the reason it
gave none.  FFmpeg's decoder gives S16 for 16-bit streams and S32, the sample in the top 24 bits, for 24-bit ones.
Test infrastructure only."""
from tests import ref_mp4


def packets(path):
    """[(file position, packet bytes)] of the first stream"""
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
        if 'unexpected sample format 0' in text:
            return None, 'U8'
        if not text:                           # avcodec_open2 failed
            return None, 'open'
        raise
