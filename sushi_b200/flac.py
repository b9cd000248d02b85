"""FLAC streams on the host: recognising a .flac file, reading its metadata blocks (or the ones a container track
carries as its codec configuration), and the calls that decode the frames on the GPU (sb_flac_decode_file finds a
file's frames by their sync codes, sb_flac_decode_frames takes them where a container lists them)."""
import ctypes
import struct

import numpy as np

from . import _native, swr
from .common import Audio, SushiError

FLAC_MAGIC = b'fLaC'
FLAC_BLOCK_NAMES = {0: 'STREAMINFO', 1: 'PADDING', 2: 'APPLICATION', 3: 'SEEKTABLE', 4: 'VORBIS_COMMENT', 5: 'CUESHEET',
                    6: 'PICTURE'}


def id3v2_size(head):
    """Bytes of an ID3v2 tag at the start of `head` (header, syncsafe size, optional footer), or 0 if there is none."""
    if len(head) < 10 or head[0:3] != b'ID3':
        return 0
    size = (head[6] & 0x7F) << 21 | (head[7] & 0x7F) << 14 | (head[8] & 0x7F) << 7 | (head[9] & 0x7F)
    return 10 + size + (10 if head[5] & 0x10 else 0)


def is_flac(path):
    """True when the file starts with the FLAC marker, or with an ID3v2 tag and then the marker (False when it cannot
    be read: the WAV reader reports that)."""
    try:
        f = open(path, 'rb')
    except OSError:
        return False
    with f:
        head = f.read(10)
        if head[0:4] == FLAC_MAGIC:
            return True
        skip = id3v2_size(head)
        if not skip:
            return False
        f.seek(skip)
        return f.read(4) == FLAC_MAGIC


class FlacFile(object):
    """FLAC metadata reader: an optional leading ID3v2 tag, the marker, then the metadata blocks.  STREAMINFO (which
    must come first) gives the stream parameters; every other block (PADDING, APPLICATION, SEEKTABLE, VORBIS_COMMENT,
    CUESHEET, PICTURE) is skipped.  `frame_offset` is where the first audio frame starts; the frames are decoded on the
    GPU (sb_flac_decode_file / sb_flac_decode_frames)."""

    def __init__(self, path):
        with open(path, 'rb') as f:
            self.data = f.read()
        self._parse(self.data, path)

    @classmethod
    def from_bytes(cls, data, name):
        """The metadata of `data` (a Matroska track's CodecPrivate: the marker and the metadata blocks, no frames);
        messages name `name`."""
        self = object.__new__(cls)
        self.data = bytes(data)
        self._parse(self.data, name)
        return self

    def _parse(self, d, path):
        self.path = path
        at = id3v2_size(d[:10])
        if d[at:at + 4] != FLAC_MAGIC:
            raise SushiError('{0}: not a FLAC file'.format(path))
        at += 4
        self.blocks = []
        have_info = False
        while True:
            if at + 4 > len(d):
                raise SushiError('{0}: FLAC metadata block header at byte {1} is truncated'.format(path, at))
            last, kind = d[at] >> 7, d[at] & 0x7F
            size = int.from_bytes(d[at + 1:at + 4], 'big')
            body = d[at + 4:at + 4 + size]
            if len(body) < size or kind == 127:
                raise SushiError('{0}: invalid FLAC metadata block at byte {1}'.format(path, at))
            if (kind == 0) != (not self.blocks):
                raise SushiError('{0}: STREAMINFO must be the first and only STREAMINFO metadata block'.format(path))
            if kind == 0:
                if size < 34:
                    raise SushiError('{0}: STREAMINFO of {1} bytes'.format(path, size))
                self.min_block, self.max_block = struct.unpack('>HH', body[0:4])
                packed = int.from_bytes(body[10:18], 'big')
                self.framerate = packed >> 44
                self.channels_count = ((packed >> 41) & 7) + 1
                self.bits_per_sample = ((packed >> 36) & 31) + 1
                self.total_samples = packed & ((1 << 36) - 1)
                have_info = True
            self.blocks.append(FLAC_BLOCK_NAMES.get(kind, 'reserved {0}'.format(kind)))
            at += 4 + size
            if last:
                break
        if not have_info:
            raise SushiError('{0}: FLAC file without STREAMINFO'.format(path))
        if self.framerate < 1:
            raise SushiError('{0}: FLAC STREAMINFO sample rate is 0'.format(path))
        self.frame_offset = at

    def check_depth(self):
        """SushiError unless the samples have 16 or 24 bits, the depths the GPU decoder takes."""
        if self.bits_per_sample not in (16, 24):
            raise SushiError('FLAC with {0} bits per sample is not supported (16 or 24)'.format(self.bits_per_sample))

    def select_audio(self, track=None):
        """The file's audio; its bit depth is refused here."""
        self.check_depth()

        def check(frames):
            # after the frames passed their checks, which name a damaged frame more precisely than the total does
            if self.total_samples and self.total_samples != frames:
                raise SushiError('{0}: FLAC STREAMINFO says {1} samples, the frames hold {2}'.format(
                    self.path, self.total_samples, frames))
        return Audio('FLAC', path=self.path, decode=lambda device: decode_file(device, self), check=check,
                     **swr.audio_format(self.bits_per_sample, swr.FLAC))


def decode_file(device, flac):
    """sb_flac_decode_file on a FlacFile's bytes."""
    buf = np.frombuffer(flac.data, dtype=np.uint8)
    return _native.decode(device, 'sb_flac_decode_file', buf.ctypes.data_as(ctypes.c_void_p), len(flac.data),
                          flac.frame_offset, flac.channels_count, flac.bits_per_sample, flac.framerate)


def track_decoder(config, name):
    """decode(device, table) of a container's FLAC track (sb_flac_decode_frames on its FrameTable; the frame numbers
    and a stale STREAMINFO total are not checked).  `config` holds the track's metadata blocks, read here, with the bit
    depth refused; messages name `name`."""
    info = FlacFile.from_bytes(config, name)
    info.check_depth()
    return lambda device, table: _native.decode_frames(
        device, 'sb_flac_decode_frames', table.data, table.offset, table.block, info.channels_count,
        info.bits_per_sample, info.framerate)
