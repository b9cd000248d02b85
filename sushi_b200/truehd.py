"""Dolby TrueHD streams on the host: recognising a raw .thd file and reading its first major sync (sample rate, samples
per access unit, substreams, the decoded presentation's channel count) for the refusals WavStream gives before the GPU
is touched.  The decode itself, and every check of the stream, is sb_truehd_decode on the GPU."""
import numpy as np

from . import _native
from .common import Audio, SushiError

SYNC_TRUEHD = b'\xf8\x72\x6f\xba'
SYNC_MLP = b'\xf8\x72\x6f\xbb'
THD_EXTENSIONS = ('.thd',)
# FFmpeg's channel count of each of the 13 channel-arrangement groups
GROUP_CHANNELS = (2, 1, 1, 2, 2, 2, 2, 1, 1, 2, 2, 1, 1)


def rate_of(code):
    return 0 if code == 0xF else (44100 if code & 8 else 48000) << (code & 7)


class MajorSync(object):
    """The first access unit's major sync.  The decoded presentation is substream min(n - 1, 2) in the layout of the
    13-bit (8-channel presentation) arrangement, as FFmpeg's decoder gives it without a downmix."""

    def __init__(self, data, name):
        if len(data) < 36:
            raise SushiError('{0}: too short for a TrueHD stream'.format(name))
        sync = data[4:32]
        if data[4:8] == SYNC_MLP:
            raise SushiError('{0}: MLP (DVD-Audio) is not supported, only Dolby TrueHD'.format(name))
        if data[4:8] != SYNC_TRUEHD:
            raise SushiError('{0}: not a TrueHD stream (no major sync in its first access unit)'.format(name))
        rate_code = sync[4] >> 4
        self.sample_rate = rate_of(rate_code)
        self.samples_per_au = 40 << (rate_code & 7)
        self.substreams = sync[16] >> 4
        arrangement = ((sync[6] & 0x1F) << 8) | sync[7]
        self.channels = sum(GROUP_CHANNELS[i] for i in range(13) if arrangement >> i & 1)
        if not self.sample_rate or self.samples_per_au > 160:
            raise SushiError('{0}: TrueHD sample rate code {1} is not supported'.format(name, rate_code))
        if not 1 <= self.substreams <= 4:
            raise SushiError('{0}: TrueHD with {1} substreams is not supported'.format(name, self.substreams))
        if not 1 <= self.channels <= 8:
            raise SushiError('{0}: TrueHD channel arrangement 0x{1:04x} is not supported (1 to 8 channels)'.format(
                name, arrangement))
        self.bits_per_sample = 24


def is_truehd(path):
    """True for a raw TrueHD (.thd) file name, or an .mlp one (which is then refused by name)."""
    return str(path).lower().endswith(THD_EXTENSIONS + ('.mlp',))


class TrueHDFile(object):
    """A raw TrueHD stream: the file's bytes and its first major sync; an .mlp file is refused."""

    def __init__(self, path):
        if str(path).lower().endswith('.mlp'):
            raise SushiError('{0}: MLP (DVD-Audio) is not supported, only Dolby TrueHD'.format(path))
        self.path = path
        with open(path, 'rb') as f:
            self.data = f.read()
        self.sync = MajorSync(self.data, path)

    def select_audio(self, track=None):
        # one block holding every access unit; a negative file offset makes messages name each unit's own offset
        return Audio('TrueHD', path=self.path, fmt='S32', decode=lambda device: decode(
            device, self.data, np.zeros(1, np.int64), np.full(1, -1, np.int64)))


def decode(device, data, offsets, blocks):
    """sb_truehd_decode on the blocks of access units at `offsets` in `data`; blocks[i] is the file offset errors
    name."""
    return _native.decode_frames(device, 'sb_truehd_decode', data, offsets, blocks)
