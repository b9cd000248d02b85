"""TTA (True Audio) streams on the host: a raw .tta file's header, seek table and tags, and a Matroska A_TTA1 track's
frames, turned into the frame table sb_tta_decode_frames decodes on the GPU.

Format-1 TTA of 16 or 24 bits per sample and 1 to 8 channels is decoded.  Encrypted streams (format 2), other formats,
8-bit streams and more than 8 channels are refused by name before any sample is produced.  Everything the header and
the seek table can show about damage is refused here too, naming the frame and its byte offset where there is one; the
bitstream and each frame's CRC are checked on the GPU.

A frame table is the frames' bytes back to back, each frame's offset in them, the file offset errors name (the
frame's own in a .tta file, its block's in a Matroska file), and the config sb_tta_decode_frames takes: channels, bits,
rate, frame length (256 * rate / 245) and the last frame's length (0 for a whole frame)."""
import ctypes
import struct
import zlib

import numpy as np

from . import _native, swr, wavpack
from .common import Audio, SushiError
from .flac import id3v2_size

TTA_EXTENSIONS = ('.tta',)
MAX_RATE = 1000000                  # FFmpeg's tta demuxer refuses a higher rate
_HEADER = struct.Struct('<4sHHHIII')


def is_tta(path):
    """True for a file that starts with `TTA1`, or with an ID3v2 tag and then `TTA1`."""
    try:
        with open(path, 'rb') as f:
            head = f.read(10)
            skip = id3v2_size(head)
            if skip:
                f.seek(skip)
                head = f.read(4)
    except (OSError, TypeError):
        return False
    return head[:4] == b'TTA1'


def frame_length(rate):
    """Samples per frame at `rate`: FFmpeg's 256 * rate / 245."""
    return 256 * rate // 245


def _refusal(fmt, channels, bits):
    """What makes a stream undecodable here (None when it is fine)."""
    if fmt == 2:
        return 'encrypted TTA (format 2)'
    if fmt != 1:
        return 'TTA format {0}'.format(fmt)
    if bits not in (16, 24):
        return 'TTA at {0} bits'.format(bits)
    if not 1 <= channels <= 8:
        return 'TTA with {0} channels'.format(channels)
    return None


def _refuse(name, why):
    raise SushiError('{0} is {1}, which cannot be decoded here (16- or 24-bit TTA of 1 to 8 channels can): convert it '
                     'to FLAC or WAV first'.format(name, why))


def _config(channels, bits, rate, total, name):
    if not 1 <= rate <= MAX_RATE:
        raise SushiError('{0}: TTA sample rate {1} is not supported (1 to {2})'.format(name, rate, MAX_RATE))
    fl = frame_length(rate)
    if fl < 1:
        raise SushiError('{0}: TTA sample rate {1} gives frames of 0 samples'.format(name, rate))
    return np.array([channels, bits, rate, fl, total % fl], np.int32)


class TTAFile(object):
    """A raw .tta file: its bytes, the frames' bytes (`audio`, a view of them), their offsets in it, their file offsets
    (`where`), where the audio ends (`end`) and the decoder config.  An ID3v2 tag in front is skipped; an APEv2 or ID3v1 tag at the end ends the audio."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.data = data = f.read()
        at = id3v2_size(data[:10])
        if len(data) < at + 22 or data[at:at + 4] != b'TTA1':
            raise SushiError('{0}: not a TTA file'.format(path))
        _, fmt, channels, bits, rate, total, crc = _HEADER.unpack_from(data, at)
        why = _refusal(fmt, channels, bits)
        if why:
            _refuse(path, why)
        if zlib.crc32(data[at:at + 18]) != crc:
            raise SushiError('{0}: TTA header CRC mismatch'.format(path))
        if total == 0:
            raise SushiError('{0}: TTA header says 0 samples'.format(path))
        self.channels, self.bits, self.rate, self.samples = channels, bits, rate, total
        self.config = _config(channels, bits, rate, total, path)
        fl = int(self.config[3])
        n = total // fl + (1 if total % fl else 0)
        table = at + 22
        first = table + 4 * n + 4
        if first > len(data):
            raise SushiError('{0}: TTA seek table of {1} frames runs past the end of the file'.format(path, n))
        sizes = np.frombuffer(data, '<u4', n, table).astype(np.int64)
        if zlib.crc32(data[table:first - 4]) != struct.unpack_from('<I', data, first - 4)[0]:
            raise SushiError('{0}: TTA seek table CRC mismatch'.format(path))
        starts = first + np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        ends = starts + sizes
        end = wavpack.tag_start(data)
        label = '{0}: TTA'.format(path)
        small = np.nonzero(sizes < 4)[0]
        if len(small):
            f = int(small[0])
            raise SushiError('{0} frame {1} at byte offset {2}: frame of {3} bytes is shorter than its CRC'.format(
                label, f, int(starts[f]), int(sizes[f])))
        past = np.nonzero(ends > end)[0]
        if len(past):
            f = int(past[0])
            raise SushiError('{0} frame {1} at byte offset {2}: frame runs past the end of the audio at byte {3} (the '
                             'file is cut short, or its seek table is damaged)'.format(label, f, int(starts[f]), end))
        if ends[-1] != end:
            raise SushiError('{0}: seek table sizes end at byte {1}, the audio at byte {2}'.format(label, int(ends[-1]),
                                                                                                 end))
        self.end = end
        self.audio = memoryview(data)[first:end]
        self.offsets = starts - first
        self.where = starts

    def select_audio(self, track=None):
        return Audio('TTA', path=self.path, decode=self._decode, **swr.audio_format(self.bits, swr.TTA))

    def _decode(self, device):
        # the file's bytes as read, up to the end of the audio: frames at their file offsets, no copy
        buf = np.frombuffer(self.data, dtype=np.uint8)
        where = self.where.ctypes.data_as(_native.c_i64p)
        return _native.decode(device, 'sb_tta_decode_frames', buf.ctypes.data_as(ctypes.c_void_p), self.end, where,
                              where, len(self.where), self.config.ctypes.data_as(_native.c_i32p))


def check_track(track):
    """An A_TTA1 track's refusals, before any frame is read: FFmpeg builds its TTA header from the track (format 1,
    Channels, BitDepth, SamplingFrequency), so a missing BitDepth leaves its decoder unable to open."""
    if not track.bit_depth:
        raise SushiError('Audio track {0} is TTA without BitDepth, which cannot be decoded here (FFmpeg cannot open '
                         'it either)'.format(track.id))
    why = _refusal(1, track.channels, track.bit_depth)
    if why:
        _refuse('Audio track {0}'.format(track.id), why)
    rate = int(track.sampling_frequency)
    if not 1 <= rate <= 0x7FFFFF or frame_length(rate) < 1:
        raise SushiError('Audio track {0} is TTA at {1:g} Hz, which cannot be decoded here'.format(
            track.id, track.sampling_frequency))


def matroska_config(track, timestamp_scale, duration):
    """The decoder config of an A_TTA1 track.  FFmpeg's Matroska demuxer has no TTA header to read: it takes the sample
    total from the Segment's Duration (in TimestampScale units), av_rescale(Duration * TimestampScale, rate, 10^9),
    and 0 without one; only the total modulo the frame length, the last frame's length, reaches the decoder."""
    rate = int(track.sampling_frequency)
    total = 0
    if duration:
        ns = int(duration * timestamp_scale)            # the double product, truncated to int64
        total = ((ns * rate + 500000000) // 1000000000) & 0xFFFFFFFF
    return _config(track.channels, track.bit_depth, rate, total, 'Audio track {0}'.format(track.id))


def track_decoder(track, timestamp_scale, duration):
    """decode(device, table) of an A_TTA1 track (sb_tta_decode_frames on its FrameTable, with matroska_config)."""
    config = matroska_config(track, timestamp_scale, duration)
    return lambda device, table: _native.decode_frames(device, 'sb_tta_decode_frames', table.data, table.offset,
                                                       table.block, config.ctypes.data_as(_native.c_i32p))
