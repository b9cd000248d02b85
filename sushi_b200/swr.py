"""--ffmpeg-audio: load a non-WAV input as the reference's demuxing call writes it.  For any input that is not a WAV
file the reference runs `ffmpeg -i <input> -map 0:<id> -ar <sample rate> -ac 1 -acodec pcm_s16le` (demux.py:31-40) and
reads the mono WAV that writes; libswresample decides what the matcher sees.  In this mode the decoded PCM goes through
sb_pcm_swr, which gives that WAV's samples bit for bit for sources FFmpeg decodes to S16, and is then loaded as such a
WAV is.  The channel layout tables here are those of FFmpeg's decoders (tests/test_swr_layouts.py holds each reader to
FFmpeg's)."""
import ctypes

from . import _native
from ._nvtx import nvtx_range
from .common import SushiError

# av_channel_layout_default: the layout ffmpeg assumes for a decoder that gives none (container PCM)
DEFAULT = {1: 0x4, 2: 0x3, 3: 0xb, 4: 0x107, 5: 0x37, 6: 0x3f, 7: 0x70f, 8: 0x63f}
# the FLAC decoder's table by channel count
FLAC = {1: 0x4, 2: 0x3, 3: 0x7, 4: 0x33, 5: 0x607, 6: 0x60f, 7: 0x70f, 8: 0x63f}
# the ALAC decoder's table (its channels already in FFmpeg's order)
ALAC = {1: 0x4, 2: 0x3, 3: 0x7, 4: 0x107, 5: 0x37, 6: 0x3f, 7: 0x13f, 8: 0xff}
# the TTA decoder's table (5 channels: none, so the default)
TTA = {1: 0x4, 2: 0x3, 3: 0xb, 4: 0x33, 5: 0x37, 6: 0x3f, 7: 0x13f, 8: 0x6cf}
# mono and stereo, where a decoder's layout does not depend on metadata this project does not read
PLAIN = {1: 0x4, 2: 0x3}


def audio_format(bits, layouts):
    """The Audio fields of an integer source of `bits` bits that FFmpeg decodes to S16 up to 16 bits and to S32 above,
    with the channel layout table `layouts`."""
    return {'fmt': 'S16' if bits <= 16 else 'S32', 'bits': bits, 'layout': layouts}


def check(audio):
    """SushiError unless FFmpeg decodes `audio` to S16, the sources --ffmpeg-audio converts exactly; before any GPU
    work.  It names the track, the codec and, where the reader knows it, the bit depth."""
    what = '{0}{1}'.format(audio.path, '' if audio.id is None else ' track {0}'.format(audio.id))
    codec = audio.label or 'PCM'
    if audio.fmt is None:
        raise SushiError('{0}: --ffmpeg-audio cannot tell which sample format FFmpeg decodes this {1} stream to before '
                         'decoding it'.format(what, codec))
    if audio.fmt != 'S16':
        depth = '' if audio.bits is None else 'of {0} bits '.format(audio.bits)
        raise SushiError('{0}: --ffmpeg-audio takes only sources FFmpeg decodes to 16-bit samples (S16); this {1} '
                         'stream {2}decodes to S32'.format(what, codec, depth))


def convert(device, h, audio, sample_rate):
    """The sb_pcm handle `h` of `audio`'s decoded samples (destroyed here; the reader's check(frames) runs on it first)
    -> a new handle holding the mono `sample_rate` samples the ffmpeg command line writes for it."""
    lib = _native.lib(device)
    try:
        frames, channels, rate = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
        _native.check(lib.sb_pcm_info(h, ctypes.byref(frames), ctypes.byref(channels), ctypes.byref(rate)),
                      'sb_pcm_info')
        if audio.check is not None:
            audio.check(frames.value)
        layout = (audio.layout or {}).get(channels.value)
        if layout is None:
            raise SushiError('{0}: --ffmpeg-audio does not know FFmpeg\'s channel layout of this {1}-channel {2} '
                             'stream'.format(audio.path, channels.value, audio.label or 'PCM'))
        out = ctypes.c_void_p()
        with nvtx_range('sushi_b200: sb_pcm_swr'):
            _native.check(lib.sb_pcm_swr(h, layout, sample_rate, ctypes.byref(out)), 'sb_pcm_swr')
        return out
    finally:
        lib.sb_pcm_destroy(h)
