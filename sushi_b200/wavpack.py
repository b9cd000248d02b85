"""WavPack streams on the host: a raw .wv file's block chain and a Matroska A_WAVPACK4 track's frames, turned into the
block table sb_wavpack_decode_blocks decodes on the GPU.

Lossless integer WavPack 4 / 5 (stream versions 0x402 to 0x410) of 2 or 3 bytes per sample and 1 to 8 channels is
decoded.  Hybrid (lossy) streams, float data, DSD, 1- and 4-byte samples and extended-precision streams (ID_WVX_BITSTREAM,
or ID_INT32_INFO with sent bits) are refused by name before any sample is produced; the flags are checked in every
block, the sub-blocks in the first frame (the GPU decoder refuses them in any block).  Everything the header chain can
show about damage is refused here too, naming the block and its byte offset; the sub-blocks and the bitstream are
checked on the GPU.

A block table has one row of 8 int64 per block: the offset and size of its sub-blocks in the uploaded bytes, block
samples, flags, CRC, the track sample where it starts, its first output channel, and the file offset errors name."""
import ctypes
import struct

import numpy as np

from . import _native, swr
from .common import Audio, SushiError

WV_EXTENSIONS = ('.wv',)
VERSIONS = (0x402, 0x410)
RATES = (6000, 8000, 9600, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 64000, 88200, 96000, 192000)
MONO, HYBRID, FLOAT, INITIAL, FINAL, DSD = 0x4, 0x8, 0x80, 0x800, 0x1000, 0x80000000
BLOCK_LIMIT = 1 << 20                      # FFmpeg's WV_BLOCK_LIMIT
MAX_BLOCK_SAMPLES = 150000                 # FFmpeg's WV_MAX_SAMPLES
ID_WVX, ID_INT32, ID_CHANNELS, ID_RATE = 0x0C, 0x09, 0x0D, 0x27
_HEADER = struct.Struct('<4sIHBBIIIII')


def is_wavpack(path):
    """True for a file that starts with a plausible WavPack block header (`wvpk`, a size of at least 24 bytes)."""
    try:
        with open(path, 'rb') as f:
            head = f.read(32)
    except (OSError, TypeError):
        return False
    return len(head) == 32 and head[:4] == b'wvpk' and struct.unpack_from('<I', head, 4)[0] >= 24


def refusal(flags):
    """What a block's flags make undecodable here (None when they are fine)."""
    if flags & HYBRID:
        return 'hybrid'
    if flags & DSD:
        return 'DSD'
    if flags & FLOAT:
        return 'float'
    if flags & 3 in (0, 3):
        return '{0}-byte samples'.format((flags & 3) + 1)
    return None


def _subblocks(data, at, end):
    """(id & 0x3f, payload offset, payload size) of each sub-block in data[at:end], stopping at a damaged one (the GPU
    decoder names it)."""
    while end - at >= 2:
        sid, words = data[at], data[at + 1]
        h = 2
        if sid & 0x80:
            if end - at < 4:
                return
            words |= (data[at + 2] | (data[at + 3] << 8)) << 8
            h = 4
        size = 2 * words - (1 if sid & 0x40 else 0)
        if size < 0 or at + h + 2 * words > end:
            return
        yield sid & 0x3F, at + h, size
        at += h + 2 * words


class Stream(object):
    """What the first frame says about a stream: rate, channels, bytes per sample; refusals raised by name."""

    def __init__(self, data, rows, name, declared=None):
        first = rows[:np.argmax(rows[:, 3] & FINAL != 0) + 1] if len(rows) else rows
        for r in rows:
            why = refusal(int(r[3]))
            if why:
                raise SushiError('{0} is WavPack ({1}), which cannot be decoded here (lossless integer WavPack of 2 or '
                                 '3 bytes per sample can): convert it to FLAC or WAV first'.format(name, why))
        self.bytes_per_sample = (int(first[0, 3]) & 3) + 1
        self.channels = int(sum(1 if f & MONO else 2 for f in first[:, 3]))
        rate_index = (int(first[0, 3]) >> 23) & 0xF
        self.rate = RATES[rate_index] if rate_index < 15 else 0
        self.declared_channels = None
        for k, r in enumerate(first):
            for sid, at, size in _subblocks(data, int(r[0]), int(r[0] + r[1])):
                if sid == ID_WVX or (sid == ID_INT32 and size == 4 and data[at]):
                    raise SushiError('{0} is WavPack (extended precision), which cannot be decoded here (lossless '
                                     'integer WavPack of 2 or 3 bytes per sample can): convert it to FLAC or WAV '
                                     'first'.format(name))
                if k == 0 and sid == ID_RATE and size == 3 and rate_index == 15:
                    self.rate = data[at] | (data[at + 1] << 8) | (data[at + 2] << 16)
                if k == 0 and sid == ID_CHANNELS and size >= 2 and self.declared_channels is None:
                    self.declared_channels = data[at]
        if not self.rate:
            raise SushiError('{0}: WavPack stream with a custom sample rate but no ID_SAMPLE_RATE'.format(name))
        if len(first) > 1 and declared is not None:
            self.declared_channels = declared
        if self.declared_channels is not None and len(first) > 1 and self.declared_channels != self.channels:
            raise SushiError('{0}: WavPack stream of {1} channels whose first frame codes {2}'.format(
                name, self.declared_channels, self.channels))
        if not 1 <= self.channels <= 8:
            raise SushiError('{0}: WavPack with {1} channels is not supported (1 to 8)'.format(name, self.channels))
        self.bits_per_sample = 8 * self.bytes_per_sample


def _frames(rows, where, label):
    """Each block's first channel and frame number from the INITIAL / FINAL flags, refusing a broken sequence or a
    frame whose blocks disagree on block_samples.  rows[:, 2] block samples, rows[:, 3] flags."""
    n = len(rows)
    channel = np.zeros(n, np.int64)
    frame = np.zeros(n, np.int64)
    f = -1
    inside = False
    ch = 0
    for i in range(n):
        flags = int(rows[i, 3])
        if not inside:
            if not flags & INITIAL:
                raise SushiError('{0} block {1} at byte offset {2}: frame does not start with an INITIAL block'.format(
                    label, i, int(where[i])))
            f += 1
            ch = 0
            inside = True
        elif flags & INITIAL:
            raise SushiError('{0} block {1} at byte offset {2}: INITIAL block before the FINAL block of its '
                             'frame'.format(label, i, int(where[i])))
        elif rows[i, 2] != rows[i - 1, 2]:
            raise SushiError('{0} block {1} at byte offset {2}: block_samples differ within a frame'.format(
                label, i, int(where[i])))
        channel[i], frame[i] = ch, f
        ch += 1 if flags & MONO else 2
        if flags & FINAL:
            inside = False
    if inside:
        raise SushiError('{0} block {1} at byte offset {2}: frame without a FINAL block'.format(
            label, n - 1, int(where[n - 1])))
    return channel, frame


def _finish(rows, where, label, channels):
    """Channel offsets and sample positions of every block; each frame must code `channels` channels."""
    channel, frame = _frames(rows, where, label)
    bad = np.nonzero((rows[:, 2] < 1) | (rows[:, 2] > MAX_BLOCK_SAMPLES))[0]
    if len(bad):
        i = int(bad[0])
        raise SushiError('{0} block {1} at byte offset {2}: block_samples {3} is not supported (1 to {4})'.format(
            label, i, int(where[i]), int(rows[i, 2]), MAX_BLOCK_SAMPLES))
    width = np.where(rows[:, 3] & MONO, 1, 2)
    per_frame = np.bincount(frame, weights=width).astype(np.int64)
    wrong = np.nonzero(per_frame != channels)[0]
    if len(wrong):
        i = int(np.argmax(frame == wrong[0]))
        raise SushiError('{0} block {1} at byte offset {2}: frame codes {3} channels, the stream has {4}'.format(
            label, i, int(where[i]), int(per_frame[wrong[0]]), channels))
    starts = np.nonzero(channel == 0)[0]
    counts = rows[starts, 2]
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    table = np.empty((len(rows), 8), np.int64)
    table[:, :5] = rows[:, :5]
    table[:, 5] = first[frame]
    table[:, 6] = channel
    table[:, 7] = where
    return table, first, counts


def tag_start(data):
    """Where the block chain ends: before a trailing ID3v1 tag and an APEv2 tag (found by its footer), as FFmpeg's wv
    demuxer stops at them."""
    end = len(data)
    if end >= 128 and data[end - 128:end - 125] == b'TAG':
        end -= 128
    if end >= 32 and data[end - 32:end - 24] == b'APETAGEX':
        size, _, flags = struct.unpack_from('<III', data, end - 20)
        start = end - size - (32 if flags & 0x80000000 else 0)
        if 0 <= start <= end - 32:
            end = start
    return end


class WavPackFile(object):
    """A raw .wv file: its bytes, the block table and the Stream of its first frame."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.data = data = f.read()
        end = tag_start(data)
        rows, where = [], []
        at, i = 0, 0
        label = '{0}: WavPack'.format(path)
        while at < end:
            if end - at < 32 or data[at:at + 4] != b'wvpk':
                raise SushiError('{0} block {1} at byte offset {2}: not a WavPack block header'.format(label, i, at))
            _, ck, version, _, _, total, index, count, flags, crc = _HEADER.unpack_from(data, at)
            if not VERSIONS[0] <= version <= VERSIONS[1]:
                raise SushiError('{0} block {1} at byte offset {2}: stream version 0x{3:03x} is not supported (0x402 to '
                                 '0x410)'.format(label, i, at, version))
            if ck < 24 or ck > BLOCK_LIMIT:
                raise SushiError('{0} block {1} at byte offset {2}: block size {3} is not supported'.format(
                    label, i, at, ck))
            if at + 8 + ck > end:
                raise SushiError('{0} block {1} at byte offset {2}: block runs past the end of the file (the file is '
                                 'cut short)'.format(label, i, at))
            if count:                              # blocks without samples carry only metadata; FFmpeg outputs none
                rows.append((at + 32, ck - 24, count, flags, crc, index, total))
                where.append(at)
                i += 1
            at += 8 + ck
        if not rows:
            raise SushiError('{0}: WavPack file without audio blocks'.format(path))
        rows = np.array(rows, np.int64)
        self.where = np.array(where, np.int64)
        self.stream = Stream(data, rows, path)
        table, first, counts = _finish(rows, self.where, label, self.stream.channels)
        # block_index continues the previous frame, as a STREAMINFO total does for FLAC
        starts = np.nonzero(table[:, 6] == 0)[0]
        index = rows[starts, 5]
        gap = np.nonzero(index[1:] != index[:-1] + counts[:-1])[0]
        if len(gap):
            b = int(starts[gap[0] + 1])
            raise SushiError('{0} block {1} at byte offset {2}: block_index {3} does not continue the previous frame '
                             '(expected {4})'.format(label, b, int(self.where[b]), int(rows[b, 5]),
                                                     int(index[gap[0]] + counts[gap[0]])))
        self.samples = int(counts.sum())
        total = int(rows[0, 6])
        if total != 0xFFFFFFFF and total != self.samples:
            raise SushiError('{0}: WavPack header says {1} samples, the blocks hold {2}'.format(path, total, self.samples))
        self.table = table

    def select_audio(self, track=None):
        return Audio('WavPack', path=self.path,
                     decode=lambda device: decode(device, self.data, self.table, self.stream),
                     **swr.audio_format(self.stream.bits_per_sample, swr.PLAIN))


def decode(device, data, table, stream):
    """sb_wavpack_decode_blocks on the blocks of `table` (a block table, above) in `data`."""
    buf = np.frombuffer(data, dtype=np.uint8)
    table = np.ascontiguousarray(table, np.int64)
    return _native.decode(device, 'sb_wavpack_decode_blocks', buf.ctypes.data_as(ctypes.c_void_p), len(data),
                          table.ctypes.data_as(_native.c_i64p), len(table), stream.channels, stream.rate)


def track_decoder(track):
    """decode(device, table) of an A_WAVPACK4 track: matroska_table on its FrameTable (the stream version from
    CodecPrivate, and the channel count a multi-block frame must code), then decode."""
    return lambda device, table: decode(device, table.data, *matroska_table(table, track.codec_private, track.id,
                                                                             track.channels))


def matroska_table(table, codec_private, track_id, declared_channels):
    """(block table, Stream) of an A_WAVPACK4 track's FrameTable: each frame is block_samples, then per block flags and
    CRC, and a size unless the block is both INITIAL and FINAL (the layout FFmpeg's Matroska demuxer rebuilds headers
    from).  The stream version is CodecPrivate's first 2 bytes."""
    name = 'Audio track {0}'.format(track_id)
    label = 'WavPack'
    data = table.data
    n = len(table)
    off, size = table.offset, table.size
    # single-block (mono or stereo) frames: every row at once
    if n and np.all(size >= 12):
        buf = np.frombuffer(data, np.uint8)
        idx = off[:, None] + np.arange(12)
        head = buf[idx].copy().view('<u4').reshape(n, 3).astype(np.int64)
        single = np.all(head[:, 1] & (INITIAL | FINAL) == (INITIAL | FINAL))
    else:
        single = False
    if single:
        rows = np.empty((n, 5), np.int64)
        rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3], rows[:, 4] = off + 12, size - 12, head[:, 0], head[:, 1], head[:, 2]
        where = table.block.copy()
    else:
        rows, where = [], []
        for i in range(n):
            at, end = int(off[i]), int(off[i] + size[i])
            if end - at < 4:
                raise SushiError('{0} frame {1} at byte offset {2}: frame too short'.format(label, i, int(table.block[i])))
            count = struct.unpack_from('<I', data, at)[0]
            at += 4
            while end - at >= 8:
                flags, crc = struct.unpack_from('<II', data, at)
                at += 8
                if flags & (INITIAL | FINAL) == (INITIAL | FINAL):
                    length = end - at
                else:
                    if end - at < 4:
                        break
                    length = struct.unpack_from('<I', data, at)[0]
                    at += 4
                if length > end - at:
                    raise SushiError('{0} frame {1} at byte offset {2}: block runs past its frame'.format(
                        label, i, int(table.block[i])))
                rows.append((at, length, count, flags, crc))
                where.append(int(table.block[i]))
                at += length
            if at != end:
                raise SushiError('{0} frame {1} at byte offset {2}: bytes after the last block of the frame'.format(
                    label, i, int(table.block[i])))
        rows = np.array(rows, np.int64).reshape(-1, 5)
        where = np.array(where, np.int64)
    stream = Stream(data, rows, name, declared_channels)
    out, _, _ = _finish(rows, where, label, stream.channels)
    return out, stream


def check_version(codec_private, track_id):
    """The A_WAVPACK4 CodecPrivate's stream version, refused outside 0x402-0x410 before any frame is read."""
    if len(codec_private) < 2:
        raise SushiError('Audio track {0} is A_WAVPACK4 without the 2-byte CodecPrivate'.format(track_id))
    version = struct.unpack_from('<H', codec_private)[0]
    if not VERSIONS[0] <= version <= VERSIONS[1]:
        raise SushiError('Audio track {0} is WavPack stream version 0x{1:03x}, which cannot be decoded here (0x402 to '
                         '0x410 can)'.format(track_id, version))
    return version
