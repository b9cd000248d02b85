"""Raw MPEG audio files on the host (`.mp2`, `.mpa`, `.m2a`), as FFmpeg's `mp3` demuxer reads them: ID3v2 tags in
front are skipped, and an ID3v1 tag and an APEv2 tag at the end end the audio.  The demuxer starts at the first frame
header the next one confirms; the bytes from there go to the GPU as one stream (sb_mp2_decode_stream), split at its
headers as FFmpeg's parser splits it.  Layer II is decoded; layer I and III
are refused by name before the GPU is touched."""
import ctypes
import logging

import numpy as np

from . import _native, swr
from .common import Audio, SushiError
from .flac import id3v2_size
from .mpegps import LAYERS, first_header
from .wavpack import tag_start

MPA_EXTENSIONS = ('.mp2', '.mpa', '.m2a')
KBPS = ((0, 32, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, 384),
        (0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160))
RATES = (44100, 48000, 32000)
MASK = 0xFFFE0CCF                 # what two frames of one stream share: sync, version, layer, rate, channel mode


def frame_size(h):
    """Bytes of the layer II frame with header h, or 0 when h is not one"""
    bi, ri, lsf = (h >> 12) & 15, (h >> 10) & 3, 0 if (h >> 19) & 1 else 1
    if (h & 0xFFE00000) != 0xFFE00000 or (h >> 19) & 3 == 1 or (h >> 17) & 3 != 2 or bi in (0, 15) or ri == 3:
        return 0
    return KBPS[lsf][bi] * 144000 // (RATES[ri] >> lsf) + ((h >> 9) & 1)


def sync_start(data):
    """Where FFmpeg's mp3 demuxer starts reading: the first layer II header followed, one frame on, by a header of
    the same stream, within the first 64 kB; 0 when there is none"""
    for i in range(min(len(data) - 3, 64 * 1024)):
        h = int.from_bytes(data[i:i + 4], 'big')
        n = frame_size(h)
        if n and i + n + 4 <= len(data):
            h2 = int.from_bytes(data[i + n:i + n + 4], 'big')
            if frame_size(h2) and (h & MASK) == (h2 & MASK):
                return i
    return 0


def is_mpeg_audio(path):
    """True for a raw MPEG audio file's name; MpegAudioFile then decides from the content."""
    return str(path).lower().endswith(MPA_EXTENSIONS)


class MpegAudioFile(object):
    """A raw MPEG audio file: its bytes, and where the audio starts and ends.  As FFmpeg's mp3 demuxer does, the audio
    starts at the first frame the next frame confirms: bytes before it (a file cut from a stream mid-frame) are
    skipped, so the first whole frame decodes."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.data = data = f.read()
        start = 0
        while True:                                       # consecutive ID3v2 tags
            n = id3v2_size(data[start:start + 10])
            if not n:
                break
            start += n
        self.start, self.end = start, max(start, tag_start(data))
        h = first_header(data[self.start:self.end])
        if h is None:
            raise SushiError('{0}: no MPEG audio frame header'.format(path))
        self.layer = (h >> 17) & 3
        if self.layer != 2:
            raise SushiError('{0} is MPEG audio {1}, which cannot be decoded here (MP2 can): convert it to FLAC or WAV '
                             'first'.format(path, LAYERS[self.layer]))
        self.start += sync_start(memoryview(data)[self.start:self.end])

    def select_audio(self, track=None):
        return Audio('MP2', path=self.path, decode=self._decode, **swr.audio_format(16, swr.PLAIN))

    def _decode(self, device):
        buf = np.frombuffer(self.data, dtype=np.uint8)
        cut = ctypes.c_int32()
        h = _native.decode(device, 'sb_mp2_decode_stream', ctypes.c_void_p(buf.ctypes.data + self.start),
                           self.end - self.start, self.start, ctypes.byref(cut))
        if cut.value:
            logging.warning('{0}: the file ends inside its last MP2 frame; it is decoded with zeros for what is '
                            'missing'.format(self.path))
        return h
