"""TAK (.tak) on the host: the `tBaK` marker and the metadata blocks of a raw file, turned into the config
sb_tak_decode_file decodes on the GPU.

Integer TAK of 16 or 24 bits, 1 to 6 channels, in either codec type FFmpeg decodes (mono/stereo and multichannel), is
decoded.  8-bit streams, more than 6 channels (FFmpeg's decoder refuses them), other data types, codec types and frame
size types FFmpeg does not decode, and a missing or corrupt STREAMINFO are refused by name here, before the GPU is
touched.  The frames are found, chained and checked on the GPU.

As FFmpeg's demuxer does, the audio starts after the metadata's END block (after an optional ID3v2 tag and `tBaK`)
and ends where LAST_FRAME says, or, without one, at the end of the file less a trailing APEv2 or ID3v1 tag (FFmpeg's
parser leaves such a tag in the last packet, where the decoder never reads it)."""
import ctypes

import numpy as np

from . import _native, swr, wavpack
from .common import Audio, SushiError
from .flac import id3v2_size

TAK_EXTENSIONS = ('.tak',)
MAX_CHANNELS = 6
CODECS = {2: 'mono/stereo', 4: 'multichannel'}
STREAMINFO, LAST_FRAME, ENCODER, MD5, END = 1, 7, 4, 6, 0
# FFmpeg's tak_channel_layouts: TAK speaker code -> channel mask bit (codes past the table add nothing)
SPEAKERS = (0, 0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40, 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000, 0x2000, 0x4000, 0x8000,
            0x10000, 0x20000)
FRAME_TYPES = (3, 4, 6, 8, 4096, 8192, 16384, 512, 1024, 2048)


def is_tak(path):
    """True for a file that starts with `tBaK`, or with an ID3v2 tag and then `tBaK`."""
    try:
        with open(path, 'rb') as f:
            head = f.read(10)
            skip = id3v2_size(head)
            if skip:
                f.seek(skip)
                head = f.read(4)
    except (OSError, TypeError):
        return False
    return head[:4] == b'tBaK'


def _refuse(name, why):
    raise SushiError('{0} is {1}, which cannot be decoded here (integer TAK of 16 or 24 bits with 1 to 6 channels '
                     'can): convert it to FLAC or WAV first'.format(name, why))


def crc24(data):
    """FFmpeg's CRC-24 of TAK (poly 0x864CFB from 0xCE04B7), as the stored little-endian value"""
    r = 0xB704CE
    for b in data:
        r ^= b << 16
        for _ in range(8):
            r = ((r << 1) ^ (0x864CFB if r & 0x800000 else 0)) & 0xFFFFFF
    return r


class _Bits(object):
    """FFmpeg's little-endian bit reader over bytes (zeros past them)"""

    def __init__(self, data):
        self.v, self.pos = int.from_bytes(data, 'little'), 0

    def get(self, n):
        x = (self.v >> self.pos) & ((1 << n) - 1)
        self.pos += n
        return x


def frame_samples(rate, frame_type):
    """FFmpeg's tak_get_nb_samples: samples per frame, 0 where FFmpeg refuses the frame size type at that rate"""
    if frame_type >= len(FRAME_TYPES):
        return 0
    q = FRAME_TYPES[frame_type]
    n, top = (rate * q >> 5, 16384) if frame_type <= 3 else (q, rate * 8 >> 5)
    return n if 0 < n <= top else 0


class TakFile(object):
    """A raw .tak file: its bytes, where its audio starts and ends, and the decoder config."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.data = data = f.read()
        at = id3v2_size(data[:10])
        if data[at:at + 4] != b'tBaK':
            raise SushiError('{0}: not a TAK file'.format(path))
        at += 4
        label = '{0}: TAK'.format(path)
        info = last = None
        while True:
            if at + 4 > len(data):
                raise SushiError('{0} metadata runs past the end of the file'.format(label))
            kind, size = data[at] & 0x7F, int.from_bytes(data[at + 1:at + 4], 'little')
            at += 4
            if kind == END:
                break
            body = data[at:at + size]
            if len(body) < size:
                raise SushiError('{0} metadata block {1} runs past the end of the file'.format(label, kind))
            if kind in (STREAMINFO, LAST_FRAME, ENCODER, MD5) and size <= 3:
                raise SushiError('{0} metadata block {1} of {2} bytes is too short'.format(label, kind, size))
            if kind == STREAMINFO:
                if info is not None:
                    raise SushiError('{0} has two STREAMINFO blocks'.format(label))
                if crc24(body[:-3]) != int.from_bytes(body[-3:], 'little'):
                    raise SushiError('{0} STREAMINFO is corrupt (CRC mismatch)'.format(label))
                info = body[:-3]
            elif kind == LAST_FRAME:
                if size != 11:
                    raise SushiError('{0} LAST_FRAME block of {1} bytes is invalid (11)'.format(label, size))
                b = _Bits(body[:8])
                last = (b.get(40), b.get(24))
            at += size
        if info is None:
            raise SushiError('{0} has no STREAMINFO'.format(label))
        b = _Bits(info)
        codec = b.get(6)
        b.get(4)
        frame_type = b.get(4)
        samples = b.get(35)
        data_type = b.get(3)
        rate = b.get(18) + 6000
        bits = b.get(5) + 8
        channels = b.get(4) + 1
        mask = 0
        if b.get(1):
            b.get(5)
            if b.get(1):
                for _ in range(channels):
                    code = b.get(6)
                    mask |= SPEAKERS[code] if code < len(SPEAKERS) else 0
        if data_type:
            _refuse(path, 'TAK of data type {0} (not integer PCM)'.format(data_type))
        if codec not in CODECS:
            _refuse(path, 'TAK of codec type {0}'.format(codec))
        if bits != 16 and bits != 24:
            _refuse(path, 'TAK at {0} bits'.format(bits))
        if channels > MAX_CHANNELS or (codec == 2 and channels > 2):
            _refuse(path, 'TAK with {0} channels ({1} codec)'.format(channels, CODECS[codec]))
        if not frame_samples(rate, frame_type):
            _refuse(path, 'TAK of frame size type {0}, invalid at {1} Hz'.format(frame_type, rate))
        if mask and bin(mask).count('1') != channels:
            _refuse(path, 'TAK whose channel layout (mask 0x{0:x}) does not give its {1} channels'.format(
                mask, channels))
        if samples < 1:
            raise SushiError('{0} stream info gives no samples'.format(label))
        self.audio_start = at
        if last is not None:
            self.audio_end = at + last[0] + last[1]
            if self.audio_end > len(data):
                raise SushiError('{0} LAST_FRAME ends at byte offset {1}, past the end of the file ({2} bytes)'.format(
                    label, self.audio_end, len(data)))
        else:
            self.audio_end = wavpack.tag_start(data)
        if self.audio_end <= self.audio_start:
            raise SushiError('{0} has no audio after its metadata'.format(label))
        self.channels, self.bits, self.rate, self.codec, self.samples = channels, bits, rate, codec, samples
        self.frame_type, self.mask = frame_type, mask
        # FFmpeg's decoder reports the stream info's layout when it gives one, the default layout otherwise
        self.layout = mask or swr.DEFAULT[channels]
        self.config = np.array([channels, bits, rate, codec, frame_type, samples & 0xFFFFFFFF, samples >> 32, mask],
                               np.int64).astype(np.int32)

    def select_audio(self, track=None):
        return Audio('TAK', path=self.path, decode=self._decode,
                     **swr.audio_format(self.bits, {self.channels: self.layout}))

    def _decode(self, device):
        buf = np.frombuffer(self.data, dtype=np.uint8)
        return _native.decode(device, 'sb_tak_decode_file', buf.ctypes.data_as(ctypes.c_void_p), len(self.data),
                              self.audio_start, self.audio_end, self.config.ctypes.data_as(_native.c_i32p))

