"""Monkey's Audio (.ape) on the host: the descriptor, the header and the seek table of a raw file, turned into the frame
table sb_ape_decode_frames decodes on the GPU.

File version 3990 (Monkey's Audio 3.99 and later) at compression levels 1000 (fast) to 5000 (insane), 16 or 24 bits,
mono or stereo, is decoded.  Other versions, 8- and 32-bit streams, more than two channels, compression levels FFmpeg
does not open, and a seek table that is cut short or inconsistent are refused by name here, before the GPU is touched.
The frame headers, the range coder and each frame's CRC are checked on the GPU.

The frame table is each frame's byte offset in the file (its seek-table entry plus any ID3v2 tag in front; the first
frame's from the header sizes, as FFmpeg's demuxer takes it) and the config sb_ape_decode_frames takes: channels,
bits, rate, compression level, blocks per frame and the last frame's blocks.  As FFmpeg's demuxer does, the last frame
runs to the end of the file less its stored WAV tail, so a trailing APEv2 or ID3v1 tag is part of its bytes (the range
decoder never reaches it)."""
import ctypes
import struct

import numpy as np

from . import _native, swr, wavpack
from .common import Audio, SushiError
from .flac import id3v2_size

APE_EXTENSIONS = ('.ape',)
VERSION = 3990
LEVELS = (1000, 2000, 3000, 4000, 5000)
MAX_RATE = (1 << 31) - 1
MAX_BLOCKS = (1 << 31) // 8 - 9            # FFmpeg's decoder refuses a frame above INT_MAX / 2 / 4 - 8 blocks
_DESCRIPTOR = struct.Struct('<4sHHIIIIIII16s')
_HEADER = struct.Struct('<HHIIIHHI')


def is_ape(path):
    """True for a file that starts with `MAC `, or with an ID3v2 tag and then `MAC `."""
    try:
        with open(path, 'rb') as f:
            head = f.read(10)
            skip = id3v2_size(head)
            if skip:
                f.seek(skip)
                head = f.read(4)
    except (OSError, TypeError):
        return False
    return head[:4] == b'MAC '


def _refuse(name, why):
    raise SushiError('{0} is {1}, which cannot be decoded here (Monkey\'s Audio 3.99 of 16 or 24 bits, mono or stereo, '
                     'at compression levels 1000 to 5000 can): convert it to FLAC or WAV first'.format(name, why))


class ApeFile(object):
    """A raw .ape file: its bytes, where its frames start (`offsets`, file offsets), where the last one ends (`end`:
    the file less its WAV tail) and the decoder config."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.data = data = f.read()
        at = id3v2_size(data[:10])
        if len(data) < at + 6 or data[at:at + 4] != b'MAC ':
            raise SushiError('{0}: not a Monkey\'s Audio file'.format(path))
        version = struct.unpack_from('<H', data, at + 4)[0]
        if version != VERSION:
            _refuse(path, 'Monkey\'s Audio file version {0}.{1:02d} ({2})'.format(version // 1000,
                                                                                   (version % 1000) // 10, version))
        if len(data) < at + _DESCRIPTOR.size:
            raise SushiError('{0}: APE descriptor cut short'.format(path))
        (_, _, _, desc_len, header_len, table_len, wav_header_len, _, _, wav_tail_len,
         _) = _DESCRIPTOR.unpack_from(data, at)
        if desc_len < 52 or len(data) < at + desc_len + _HEADER.size:
            raise SushiError('{0}: APE header cut short'.format(path))
        (level, _, bpf, final, frames, bits, channels, rate) = _HEADER.unpack_from(data, at + desc_len)
        if bits not in (16, 24):
            _refuse(path, 'Monkey\'s Audio at {0} bits'.format(bits))
        if not 1 <= channels <= 2:
            _refuse(path, 'Monkey\'s Audio with {0} channels'.format(channels))
        if level not in LEVELS:
            _refuse(path, 'Monkey\'s Audio at compression level {0}'.format(level))
        if not 1 <= rate <= MAX_RATE:
            raise SushiError('{0}: APE sample rate {1} is not supported (1 to {2})'.format(path, rate, MAX_RATE))
        if bpf > MAX_BLOCKS:
            raise SushiError('{0}: APE frames of {1} blocks are not supported (FFmpeg refuses more than {2})'.format(
                path, bpf, MAX_BLOCKS))
        if frames == 0 or bpf == 0 or not 1 <= final <= bpf:
            raise SushiError('{0}: APE header gives {1} frames of {2} blocks, the last of {3}: not a stream'.format(
                path, frames, bpf, final))
        label = '{0}: APE'.format(path)
        if table_len // 4 < frames:
            raise SushiError('{0} seek table of {1} entries is cut short: the header gives {2} frames'.format(
                label, table_len // 4, frames))
        table = at + desc_len + header_len
        if table + 4 * frames > len(data):
            raise SushiError('{0} seek table of {1} frames runs past the end of the file'.format(label, frames))
        seek = np.frombuffer(data, '<u4', frames, table).astype(np.int64) + at
        first = at + desc_len + header_len + table_len + wav_header_len
        offsets = seek.copy()
        offsets[0] = first
        self.end = end = len(data) - wav_tail_len
        audio_end = min(end, wavpack.tag_start(data))
        back = np.nonzero(np.diff(offsets) <= 0)[0]
        if len(back):
            f = int(back[0]) + 1
            raise SushiError('{0} seek table is inconsistent: frame {1} at byte offset {2} does not follow frame {3} '
                             'at byte offset {4}'.format(label, f, int(offsets[f]), f - 1, int(offsets[f - 1])))
        past = np.nonzero(offsets >= audio_end)[0]
        if len(past):
            f = int(past[0])
            raise SushiError('{0} seek table is inconsistent: frame {1} at byte offset {2} starts past the end of the '
                             'audio at byte {3}'.format(label, f, int(offsets[f]), audio_end))
        self.channels, self.bits, self.rate, self.level = channels, bits, rate, level
        self.samples = (frames - 1) * bpf + final
        self.offsets = offsets
        self.config = np.array([channels, bits, rate, level, bpf, final], np.int32)

    def select_audio(self, track=None):
        return Audio('APE', path=self.path, decode=self._decode, **swr.audio_format(self.bits, swr.PLAIN))

    def _decode(self, device):
        # the file's bytes as read, up to the end of the last frame: frames at their file offsets, no copy
        buf = np.frombuffer(self.data, dtype=np.uint8)
        offsets = self.offsets.ctypes.data_as(_native.c_i64p)
        return _native.decode(device, 'sb_ape_decode_frames', buf.ctypes.data_as(ctypes.c_void_p), self.end, offsets,
                              offsets, len(self.offsets), self.config.ctypes.data_as(_native.c_i32p))
