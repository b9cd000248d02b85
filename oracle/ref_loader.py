"""CPU restatement of the reference loader -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Follows /root/reference/wav.py:15-162: RIFF walk (18-54), fmt chunk (93-101), PCM decode and
downmix (64-91), 1-second chunk loop with cv2.resize(INTER_NEAREST) (125-137), edge padding
(140-141), median-clip normalisation (145-151), uint8 quantisation (153-156).
Python-3 edits only: bytes literals, np.frombuffer, integer division, range/functools.reduce.
"""
import math
import os
import struct
from functools import reduce

import cv2
import numpy as np

WAVE_FORMAT_PCM = 0x0001
WAVE_FORMAT_EXTENSIBLE = 0xFFFE


def parse_header(f, path):
    """-> dict(channels, framerate, sample_width, frame_size, frames_count); file left at the PCM payload."""
    riff_id, _, wave_id = struct.unpack('<4sL4s', f.read(12))
    if riff_id != b'RIFF':
        raise ValueError('File does not start with RIFF id')
    if wave_id != b'WAVE':
        raise ValueError('Not a WAVE file')
    info = {}
    file_size = os.path.getsize(path)
    while True:
        hdr = f.read(8)
        if len(hdr) < 8:
            break
        name, size = struct.unpack('<4sL', hdr)
        if name == b'fmt ':
            body = f.read(size + (size & 1))
            tag, ch, rate, _, _ = struct.unpack('<HHLLH', body[:14])
            if tag not in (WAVE_FORMAT_PCM, WAVE_FORMAT_EXTENSIBLE):
                raise ValueError('unknown format: {0}'.format(tag))
            width = (struct.unpack('<H', body[14:16])[0] + 7) // 8
            info.update(channels=ch, framerate=rate, sample_width=width, frame_size=ch * width)
        elif name == b'data':
            if file_size > 0xFFFFFFFF:
                info['frames_count'] = (file_size - f.tell()) // info['frame_size']
            else:
                info['frames_count'] = size // info['frame_size']
            return info
        else:
            f.seek(size + (size & 1), os.SEEK_CUR)
    raise ValueError('Invalid WAV file')


def _py2_round(x):
    """The reference runs under Python 2, whose round() goes half away from zero (wav.py:127)."""
    return math.floor(x + 0.5) if x >= 0 else -math.floor(-x + 0.5)


def readframes(raw, sample_width, channels):          # wav.py:64-91
    if sample_width == 2:
        unpacked = np.frombuffer(raw, dtype=np.int16)
    elif sample_width == 3:
        raw_bytes = np.frombuffer(raw, dtype=np.int8)
        unpacked = np.zeros(len(raw) // 3, np.int16)
        unpacked.view(dtype='int8')[0::2] = raw_bytes[1::3]
        unpacked.view(dtype='int8')[1::2] = raw_bytes[2::3]
    else:
        raise ValueError('Unsupported sample width: {0}'.format(sample_width))
    unpacked = unpacked.astype('float32')
    if channels == 1:
        return unpacked
    min_length = len(unpacked) // channels
    chans = (unpacked[i::channels] for i in range(channels))
    data = reduce(lambda a, b: a[:min_length] + b[:min_length], chans)
    data /= float(channels)
    return data


def pad_stream(read_raw, frames_count, framerate, sample_width, channels, sample_rate=12000, skip_empty=False):
    """wav.py:108-141: the chunk loop and the edge padding, before normalisation.
    Returns (padded float32 data (1,N), sample_count, padding_size).  skip_empty=True is NOT the reference: a read
    that resamples to no sample, where cv2.resize raises, contributes none (the product's documented rule)."""
    total_seconds = frames_count / float(framerate)
    downsample_rate = sample_rate / float(framerate)
    sample_count = math.ceil(total_seconds * sample_rate)
    # np.empty in the reference (wav.py:119); zero-filled here so the rare gap is deterministic
    data = np.zeros((1, int(10 * 2 * framerate + sample_count)), np.float32)
    padding_size = 10 * framerate
    seconds_read = 0
    samples_read = padding_size
    while seconds_read < total_seconds:
        chunk = readframes(read_raw(int(1 * framerate)), sample_width, channels)
        new_length = int(_py2_round(len(chunk) * downsample_rate))
        if skip_empty and new_length == 0:
            seconds_read += 1
            continue
        dst_view = data[0][samples_read:samples_read + new_length]
        if downsample_rate != 1:
            chunk = chunk.reshape((1, len(chunk)))
            chunk = cv2.resize(chunk, (new_length, 1), interpolation=cv2.INTER_NEAREST)[0]
        np.copyto(dst_view, chunk, casting='no')
        samples_read += new_length
        seconds_read += 1
    data[0][0:padding_size].fill(data[0][padding_size])
    data[0][-padding_size:].fill(data[0][-padding_size - 1])
    return data, sample_count, padding_size


def normalise(data, sample_type='uint8'):
    """wav.py:145-156 on a padded array (overwritten).  Returns (data, min_value, max_value)."""
    max_value = np.median(data[data >= 0], overwrite_input=True) * 3
    min_value = np.median(data[data <= 0], overwrite_input=True) * 3
    np.clip(data, min_value, max_value, out=data)
    data -= min_value
    data /= (max_value - min_value)
    if sample_type == 'uint8':
        data *= 255.0
        data += 0.5
        data = data.astype('uint8')
    return data, min_value, max_value


def load_stream(read_raw, frames_count, framerate, sample_width, channels, sample_rate=12000, sample_type='uint8'):
    """wav.py:108-156 with `read_raw(nframes) -> bytes` standing in for the open file.
    Returns (data (1,N), sample_count, padding_size)."""
    data, sample_count, padding_size = pad_stream(read_raw, frames_count, framerate, sample_width, channels, sample_rate)
    data, _, _ = normalise(data, sample_type)
    return data, sample_count, padding_size


def load_wav_padded(path, sample_rate=12000):
    """(padded float32 data before normalisation, sample_count, padding_size) of a WAV file."""
    with open(path, 'rb') as f:
        info = parse_header(f, path)
        return pad_stream(lambda n: f.read(n * info['frame_size']), info['frames_count'], info['framerate'],
                          info['sample_width'], info['channels'], sample_rate)


def load_wav(path, sample_rate=12000, sample_type='uint8'):
    with open(path, 'rb') as f:
        info = parse_header(f, path)
        return load_stream(lambda n: f.read(n * info['frame_size']), info['frames_count'], info['framerate'],
                           info['sample_width'], info['channels'], sample_rate, sample_type)
