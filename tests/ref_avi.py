"""FFmpeg's `avi` demuxer and its `pcm_*` / `mp2` decoders for the tests, through the ctypes driver of tests/ref_mp4.py
(libavformat / libavcodec 62, from oracle/ref_flac.libs()).

`streams(path)` gives the stream list as avformat_open_input leaves it ([{id, kind, codec}] in FFmpeg's order; the
test videos are random bytes, which stream probing cannot decode, so the list is the demuxer's own);
`packets(path, index)` the bytes of every packet of one stream, as av_read_frame returns them; `decode_s16` and
`decode_pcm` are tests/ref_mp4.py's.  Test infrastructure only: the product never imports this."""
from tests import ref_mp4

decode_s16 = ref_mp4.decode_s16
decode_pcm = ref_mp4.decode_pcm
decoder_layout = ref_mp4.decoder_layout


def streams(path):
    """[{id, kind, codec}] in FFmpeg's stream order"""
    return [dict(id=i, kind=k, codec=c) for i, (k, c, _) in enumerate(ref_mp4.demux(path, packets=False).streams)]


def packets(path, index):
    """the bytes of every packet of stream `index`, in order"""
    return [d for d, _ in ref_mp4.demux(path).track(index)]
