"""RIFF/WAVE files on the host, and the NumPy arithmetic of the reference's loader (wav.py:15-156): the header walk,
the int16/int24 decode and channel averaging, OpenCV's nearest-neighbour index map and the median-clip normalisation.
WavStream's loader='host' runs these; its GPU loader gives bit-identical .data (sb_load_pcm, sb_normalise)."""
import io
import logging
import math
import os
import struct

import numpy as np

from .common import Audio, SushiError

WAVE_FORMAT_PCM = 0x0001
WAVE_FORMAT_EXTENSIBLE = 0xFFFE


class DownmixedWavFile(object):
    """RIFF/WAVE reader + int16/int24 decode + channel averaging (wav.py:15-101).

    Header walking stays on the host (survey row a10); decode/downmix of the PCM
    payload is done by ``readframes`` on the host for the streaming loader and by
    the GPU loader kernels for whole-file loads.
    """

    def __init__(self, path):
        self._file = open(path, 'rb')
        self.channels_count = self.framerate = self.sample_width = self.frame_size = None
        self.frames_count = None
        try:
            head = self._file.read(12)
            if len(head) < 12 or head[0:4] != b'RIFF':
                raise SushiError('File does not start with RIFF id')
            if head[8:12] != b'WAVE':
                raise SushiError('Not a WAVE file')
            file_size = os.path.getsize(path)
            have_fmt = have_data = False
            while True:
                hdr = self._file.read(8)
                if len(hdr) < 8:
                    break
                name, size = hdr[0:4], struct.unpack('<L', hdr[4:8])[0]
                if name == b'fmt ':
                    self._read_fmt_chunk(self._file.read(size + (size & 1)))
                    have_fmt = True
                    continue
                if name == b'data':
                    if file_size > 0xFFFFFFFF:
                        # >4 GiB "broken" wav: trust the file size, not the 32-bit chunk size (wav.py:42-44)
                        self.frames_count = (file_size - self._file.tell()) // self.frame_size
                    else:
                        self.frames_count = size // self.frame_size
                    self.data_offset = self._file.tell()
                    have_data = True
                    break
                self._file.seek(size + (size & 1), os.SEEK_CUR)
            if not have_fmt or not have_data:
                raise SushiError('Invalid WAV file')
        except Exception:
            self.close()
            raise

    @classmethod
    def from_bytes(cls, data, channels, framerate, sample_width, frames=None):
        """A reader over in-memory interleaved little-endian PCM, as if it were a WAV file's data chunk (of `frames`
        frames by its header; default: the frames `data` holds)."""
        self = cls.__new__(cls)
        self._file = io.BytesIO(data)
        self.channels_count, self.framerate, self.sample_width = channels, framerate, sample_width
        self.frame_size = channels * sample_width
        self.frames_count = len(data) // self.frame_size if frames is None else frames
        return self

    def __del__(self):
        self.close()

    def close(self):
        f = getattr(self, '_file', None)
        if f:
            f.close()
            self._file = None

    def _read_fmt_chunk(self, payload):
        tag, self.channels_count, self.framerate, _, _ = struct.unpack('<HHLLH', payload[:14])
        if tag not in (WAVE_FORMAT_PCM, WAVE_FORMAT_EXTENSIBLE):
            raise SushiError('unknown format: {0}'.format(tag))
        bits = struct.unpack('<H', payload[14:16])[0]
        self.sample_width = (bits + 7) // 8
        self.frame_size = self.channels_count * self.sample_width

    def read_raw(self, count):
        return self._file.read(count * self.frame_size)

    def readframes(self, count):
        """Decode `count` frames to mono float32 (wav.py:64-91)."""
        if not count:
            return np.zeros(0, np.float32)
        return decode_downmix(self.read_raw(count), self.sample_width, self.channels_count)

    def select_audio(self, track=None):
        """The PCM the reference's chunk loop reads (wav.py:125-137): whole seconds from the start of the data chunk, so
        the last read can run past the chunk or stop short at the end of a truncated file; the frame count is the
        header's."""
        def pcm():
            reads = math.ceil(self.frames_count / float(self.framerate))
            return (self.read_raw(reads * self.framerate), self.frames_count, self.channels_count, self.sample_width,
                    self.framerate, False)
        return Audio(None, pcm=pcm)


def decode_downmix(raw, sample_width, channels):
    """bytes -> float32 mono; int24 keeps the top 16 bits (wav.py:68-74); channels are
    summed left to right in float32, then divided (wav.py:88-90)."""
    if sample_width == 2:
        pcm = np.frombuffer(raw, dtype='<i2', count=len(raw) // 2)
    elif sample_width == 3:
        b = np.frombuffer(raw, dtype=np.uint8, count=(len(raw) // 3) * 3).reshape(-1, 3)
        pcm = (b[:, 1].astype(np.uint16) | (b[:, 2].astype(np.uint16) << 8)).view(np.int16)
    else:
        raise SushiError('Unsupported sample width: {0}'.format(sample_width))
    samples = pcm.astype(np.float32)
    if channels == 1:
        return samples
    frames = len(samples) // channels
    if frames * channels != len(samples):
        logging.error("Length of audio channels didn't match. This might result in broken output")
    acc = samples[0::channels][:frames].copy()
    for ch in range(1, channels):
        acc += samples[ch::channels][:frames]
    acc /= np.float32(channels)
    return acc


def nearest_index_map(n_in, n_out):
    """Source index of every output sample of cv2.resize(..., INTER_NEAREST) on a
    (1, n_in) row resized to (1, n_out): floor(x * (1 / (n_out / n_in))) in fp64,
    clamped to n_in-1 (OpenCV resizeNN; pinned against cv2 in tests)."""
    inv = 1.0 / (float(n_out) / float(n_in))
    idx = np.floor(np.arange(n_out, dtype=np.float64) * inv).astype(np.int64)
    np.minimum(idx, n_in - 1, out=idx)
    return idx


def normalise_host(data, sample_type):
    """Median-clip normalisation of a padded float32 (1,N) array, in place semantics of
    wav.py:145-156 (float32 arithmetic throughout, medians over the padded array)."""
    flat = data.reshape(-1)
    max_value = np.float32(np.median(flat[flat >= 0])) * np.float32(3)
    min_value = np.float32(np.median(flat[flat <= 0])) * np.float32(3)
    np.clip(data, min_value, max_value, out=data)
    data -= min_value
    data /= (max_value - min_value)
    if sample_type == 'uint8':
        data *= np.float32(255.0)
        data += np.float32(0.5)
        data = data.astype(np.uint8)
    return data, float(min_value), float(max_value)
