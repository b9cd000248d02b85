"""A seeded TTA writer for the tests: format-1 streams whose PCM is known, refused variants and damaged copies.

The writer runs the decoder's arithmetic backwards (FFmpeg's `tta` decoder): the inter-channel decorrelation and the
fixed predictor are inverted over whole frames with NumPy, the 8-tap adaptive filter runs sample by sample with the
same taps, steps and 32-bit wrap-around, and the residuals are coded with the adaptive Rice code (two parameters and
sums per channel, the same update rule), least significant bit first.  Every frame restarts the state and ends with
the CRC-32 of its bitstream; the file has the 22-byte TTA1 header and the seek table of frame sizes, each with its
CRC-32.  Every case records which features it used (Rice parameters reached, branches, unary run lengths, rates,
channel counts, lengths against the frame length, tags), and `assert_coverage` checks that the cases together use all
of FEATURES.

A case's `pcm` is (frames, channels) int64 at its bit depth in FFmpeg's channel order; `pcm16` the int16 the loader
keeps (the top 16 bits of FFmpeg's S32 sample for 24-bit streams)."""
import functools
import struct
import zlib

import numpy as np

M32 = 0xFFFFFFFF
RATES = (7919, 8000, 11025, 12001, 16000, 22050, 32000, 44100, 48000, 88200, 96000, 192000)
FEATURES = ({'bits_16', 'bits_24', 'full_scale_16', 'full_scale_24', 'quiet_16', 'quiet_24', 'extreme_differences',
             'k0_zero', 'k1_zero', 'k_max', 'depth_0', 'depth_1', 'long_unary', 'exact_multiple', 'multiple_plus_one',
             'multiple_minus_one', 'one_frame', 'id3v2', 'apev2', 'id3v1'} |
            {'channels_%d' % c for c in (1, 2, 3, 6, 8)} | {'rate_%d' % r for r in RATES})
K_MAX = 25                                   # FFmpeg's decoder refuses a Rice parameter above this


def frame_length(rate):
    return 256 * rate // 245


def shift_1(i):
    return 1 << i if i < 31 else 0x80000000


def shift_16(i):
    return shift_1(i + 4)


def i32(v):
    v &= M32
    return v - (1 << 32) if v >> 31 else v


def to16(pcm, bits):
    return (pcm >> (bits - 16)).astype(np.int16) if bits > 16 else pcm.astype(np.int16)


def _trunc_half(a):
    """C's a / 2 (toward zero) on int64 arrays"""
    return np.where(a < 0, -((-a) // 2), a // 2)


def decorrelated(x):
    """The values the decoder's channels hold before decorrelation, for output samples x (n, channels)"""
    if x.shape[1] == 1:
        return x.copy()
    v = np.empty_like(x)
    v[:, :-1] = x[:, 1:] - x[:, :-1]
    v[:, -1] = x[:, -1] - _trunc_half(v[:, -2])
    return v


def filter_residuals(f, shift):
    """The residuals whose filtered values are f (one channel of one frame, Python ints): the filter of FFmpeg's
    tta_filter_process_c, run forwards with the output known."""
    q0 = q1 = q2 = q3 = q4 = q5 = q6 = q7 = 0
    x0 = x1 = x2 = x3 = x4 = x5 = x6 = x7 = 0
    l0 = l1 = l2 = l3 = l4 = l5 = l6 = l7 = 0
    err = 0
    rnd = 1 << (shift - 1)
    out = []
    for v in f:
        if err < 0:
            q0 -= x0; q1 -= x1; q2 -= x2; q3 -= x3; q4 -= x4; q5 -= x5; q6 -= x6; q7 -= x7
        elif err > 0:
            q0 += x0; q1 += x1; q2 += x2; q3 += x3; q4 += x4; q5 += x5; q6 += x6; q7 += x7
        s = (rnd + l0 * q0 + l1 * q1 + l2 * q2 + l3 * q3 + l4 * q4 + l5 * q5 + l6 * q6 + l7 * q7) & M32
        s = s - (1 << 32) if s >> 31 else s
        n4, n5, n6, n7 = (l4 >> 30) | 1, ((l5 >> 30) | 2) & ~1, ((l6 >> 30) | 2) & ~1, ((l7 >> 30) | 4) & ~3
        err = v - (s >> shift)
        out.append(err)
        d6 = v - l7
        d5 = d6 - l6
        d4 = d5 - l5
        l0, l1, l2, l3, l4, l5, l6, l7 = l1, l2, l3, l4, d4, d5, d6, v
        x0, x1, x2, x3, x4, x5, x6, x7 = x1, x2, x3, x4, n4, n5, n6, n7
    return out


def rice_codes(values, used):
    """(unary, k, low bits) per zigzag value of one channel of one frame, the Rice state adapting as the decoder's"""
    k0 = k1 = 10
    s0 = s1 = shift_16(10)
    n = len(values)
    un = np.empty(n, np.int64)
    kk = np.empty(n, np.int64)
    low = np.empty(n, np.int64)
    for i, v in enumerate(values):
        k = k0
        s0 = (s0 + v - (s0 >> 4)) & M32
        if k0 > 0 and s0 < shift_16(k0):
            k0 -= 1
        elif s0 > shift_16(k0 + 1):
            k0 += 1
        if v >= shift_1(k):
            v -= shift_1(k)
            k = k1
            s1 = (s1 + v - (s1 >> 4)) & M32
            if k1 > 0 and s1 < shift_16(k1):
                k1 -= 1
            elif s1 > shift_16(k1 + 1):
                k1 += 1
            u = 1 + (v >> k)
            used['depth_1'] = True
            if k1 == 0:
                used['k1_zero'] = True
        else:
            u = 0
            used['depth_0'] = True
        if k0 == 0:
            used['k0_zero'] = True
        assert k <= K_MAX, 'Rice parameter %d: FFmpeg refuses it' % k
        used['k_top'] = max(used.get('k_top', 0), k)
        used['u_top'] = max(used.get('u_top', 0), u)
        un[i], kk[i], low[i] = u, k, v & ((1 << k) - 1)
    return un, kk, low


def pack(un, kk, low):
    """The LSB-first bitstream of the codes (u ones, a zero, k low bits each), padded to a byte"""
    lengths = un + 1 + kk
    start = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    total = int(lengths.sum())
    mark = np.zeros(total + 1, np.int64)
    np.add.at(mark, start, 1)
    np.add.at(mark, start + un, -1)
    bits = np.cumsum(mark)[:total].astype(np.uint8)
    base = start + un + 1
    for j in range(int(kk.max()) if len(kk) else 0):
        sel = kk > j
        bits[base[sel] + j] = (low[sel] >> j) & 1
    return np.packbits(bits, bitorder='little').tobytes()


def encode_frame(x, bits, used):
    """One frame's bytes (bitstream and CRC) for samples x (n, channels) int64"""
    n, channels = x.shape
    v = decorrelated(x)
    pred = np.zeros_like(v)
    pred[1:] = (v[:-1] * 31) >> (4 if bits == 8 else 5)
    f = v - pred
    shift = {8: 10, 16: 9, 24: 10}[bits]
    codes = []
    for c in range(channels):
        res = np.array(filter_residuals(f[:, c].tolist(), shift), np.int64)
        assert np.all(np.abs(res) < (1 << 30)), 'residual out of range'
        zz = np.where(res > 0, 2 * res - 1, -2 * res)
        codes.append(rice_codes(zz.tolist(), used))
    un = np.stack([c[0] for c in codes], 1).reshape(-1)
    kk = np.stack([c[1] for c in codes], 1).reshape(-1)
    low = np.stack([c[2] for c in codes], 1).reshape(-1)
    body = pack(un, kk, low)
    return body + struct.pack('<I', zlib.crc32(body))


def header(channels, bits, rate, total, fmt=1):
    h = b'TTA1' + struct.pack('<HHHII', fmt, channels, bits, rate, total)
    return h + struct.pack('<I', zlib.crc32(h))


def seek_table(frames):
    t = b''.join(struct.pack('<I', len(f)) for f in frames)
    return t + struct.pack('<I', zlib.crc32(t))


class TtaCase(object):
    """A stream: pcm (n, channels) at `bits`, its frames, and what surrounds them in a .tta file"""

    def __init__(self, name, pcm, rate, bits, frames, used, head=b'', tail=b'', fmt=1):
        self.name, self.pcm, self.rate, self.bits, self.frames = name, pcm, rate, bits, frames
        self.channels = pcm.shape[1]
        self.used, self.head, self.tail, self.fmt = used, head, tail, fmt

    @property
    def pcm16(self):
        return to16(self.pcm, self.bits)

    @property
    def frame_length(self):
        return frame_length(self.rate)

    def tta(self):
        return (self.head + header(self.channels, self.bits, self.rate, len(self.pcm), self.fmt) +
                seek_table(self.frames) + b''.join(self.frames) + self.tail)

    def frame_offsets(self):
        """file offset of each frame in tta()"""
        at = len(self.head) + 22 + 4 * len(self.frames) + 4
        return list(np.concatenate([[0], np.cumsum([len(f) for f in self.frames])[:-1]]).astype(np.int64) + at)

    def __repr__(self):
        return 'TtaCase(%s)' % self.name


def signal(rng, n, channels, bits, kind):
    """n samples of `kind`: 'tone' (sines and noise at half scale), 'noise' (full scale), 'quiet' (near silence with
    spikes to +-2^15, each coded as a long unary run), 'extreme' (channels at opposite extremes, flipping)"""
    top = (1 << (bits - 1)) - 1
    t = np.arange(n)
    if kind == 'noise':
        return rng.integers(-top - 1, top + 1, (n, channels))
    if kind == 'quiet':
        x = rng.integers(-1, 2, (n, channels)) * (rng.random((n, channels)) < 0.1)
        for c in range(channels):
            at = rng.integers(0, n, 3)
            x[at, c] = rng.choice([min(top, 32767), -min(top, 32767) - 1], 3)
        return x
    if kind == 'extreme':
        flip = ((t // 97) % 2)[:, None]
        sign = np.where((np.arange(channels)[None, :] + flip) % 2 == 0, 1, -1)
        x = np.where(sign > 0, top, -top - 1) + 0 * t[:, None]
        x += (sign * -rng.integers(0, 4, (n, channels)))
        return x
    out = np.empty((n, channels), np.int64)
    for c in range(channels):
        f1, f2 = 0.003 + 0.011 * c, 0.0007 + 0.003 * c
        out[:, c] = (0.3 * top * np.sin(f1 * t) + 0.15 * top * np.sin(f2 * t + c) +
                     rng.normal(0, top / 300, n)).astype(np.int64)
    return np.clip(out, -top - 1, top)


def make_case(name, seed, rate=44100, channels=2, bits=16, total=None, kind='tone', head=b'', tail=b'', pcm=None):
    """A stream of `total` samples (default: two frames and a bit) of `kind`"""
    fl = frame_length(rate)
    rng = np.random.default_rng([20261016, seed])
    if pcm is None:
        total = 2 * fl + fl // 3 if total is None else total
        pcm = signal(rng, total, channels, bits, kind)
    total = len(pcm)
    used = {}
    frames = [encode_frame(pcm[a:a + fl], bits, used) for a in range(0, total, fl)]
    k_top, u_top = used.pop('k_top', 0), used.pop('u_top', 0)
    used = set(used)
    used |= {'bits_%d' % bits, 'channels_%d' % channels, 'rate_%d' % rate}
    if k_top >= 24:
        used.add('k_max')
    if u_top >= 1000:
        used.add('long_unary')
    rem = total % fl
    used.add({0: 'exact_multiple', 1: 'multiple_plus_one', fl - 1: 'multiple_minus_one'}.get(rem, 'other_length'))
    if len(frames) == 1:
        used.add('one_frame')
    if kind == 'noise':
        used.add('full_scale_%d' % bits)
    if kind == 'quiet':
        used.add('quiet_%d' % bits)
    if kind == 'extreme':
        used.add('extreme_differences')
    case = TtaCase(name, pcm.astype(np.int64), rate, bits, frames, used, head, tail)
    case.k_top, case.u_top = k_top, u_top
    return case


def apetag():
    """An APEv2 tag with a header, one item and a footer"""
    item = struct.pack('<II', 5, 0) + b'Title\0' + b'Sushi'
    size = len(item) + 32

    def part(flags):
        return b'APETAGEX' + struct.pack('<IIII', 2000, size, 1, flags) + bytes(8)
    return part(0xA0000000) + item + part(0x80000000)


def id3v1():
    return b'TAG' + b'Sushi'.ljust(30, b'\0') + bytes(30 + 30 + 4 + 30) + b'\xff'


def id3v2():
    body = b'TIT2' + struct.pack('>I', 6) + b'\0\0' + b'\0Sushi' + bytes(40)
    n = len(body)
    return b'ID3\x04\x00\x00' + bytes([(n >> 21) & 127, (n >> 14) & 127, (n >> 7) & 127, n & 127]) + body


@functools.lru_cache(maxsize=None)
def _all_cases():
    c = []
    fl = frame_length
    c.append(make_case('mono16', 1, rate=44100, channels=1))
    c.append(make_case('stereo16_exact', 2, rate=44100, total=2 * fl(44100)))
    c.append(make_case('stereo16_minus_one', 3, rate=48000, total=2 * fl(48000) - 1))
    c.append(make_case('stereo24_noise', 4, rate=48000, bits=24, total=fl(48000) + 1, kind='noise'))
    c.append(make_case('stereo16_noise', 5, rate=8000, total=fl(8000) + 1, kind='noise'))
    c.append(make_case('three24', 6, rate=8000, channels=3, bits=24, total=fl(8000) + 1))
    c.append(make_case('six16', 7, rate=11025, channels=6, total=fl(11025) - 1))
    c.append(make_case('eight24_extreme', 8, rate=8000, channels=8, bits=24, total=fl(8000), kind='extreme'))
    c.append(make_case('eight16_extreme', 9, rate=7919, channels=8, total=fl(7919) + 1, kind='extreme'))
    c.append(make_case('quiet16', 10, rate=22050, channels=1, total=fl(22050) + 5000, kind='quiet'))
    c.append(make_case('quiet24', 11, rate=16000, bits=24, total=fl(16000) + 1, kind='quiet'))
    c.append(make_case('one_frame', 12, rate=44100, total=1000))
    for k, rate in enumerate((12001, 32000, 88200, 96000, 192000)):
        c.append(make_case('rate%d' % rate, 20 + k, rate=rate, channels=1, total=fl(rate) + (1 if k % 2 else -1)))
    c.append(make_case('id3v2_front', 13, rate=8000, channels=1, total=3000, head=id3v2()))
    c[-1].used.add('id3v2')
    c.append(make_case('apev2_end', 14, rate=8000, total=fl(8000) + 700, tail=apetag()))
    c[-1].used.add('apev2')
    c.append(make_case('id3v1_end', 15, rate=8000, channels=1, total=fl(8000) + 300, tail=id3v1()))
    c[-1].used.add('id3v1')
    c.append(make_case('apev2_id3v1_end', 16, rate=8000, channels=2, bits=24, total=2000, tail=apetag() + id3v1()))
    c[-1].used |= {'apev2', 'id3v1'}
    return tuple(c)


def all_cases():
    """Every .tta case, covering FEATURES together"""
    return list(_all_cases())


def assert_coverage(cases):
    used = set().union(*[c.used for c in cases])
    missing = FEATURES - used
    assert not missing, sorted(missing)


def _rewrite_seek(data, at, n, sizes):
    """data with the seek table at `at` (n frames) holding `sizes`, its CRC fixed"""
    t = b''.join(struct.pack('<I', s) for s in sizes)
    return data[:at] + t + struct.pack('<I', zlib.crc32(t)) + data[at + 4 * n + 4:]


def _with_frame(case, f, frame):
    """case's .tta bytes with frame f replaced (sizes and CRCs fixed)"""
    frames = list(case.frames)
    frames[f] = frame
    return (case.head + header(case.channels, case.bits, case.rate, len(case.pcm)) + seek_table(frames) +
            b''.join(frames) + case.tail)


def _recrc(body):
    return body + struct.pack('<I', zlib.crc32(body))


@functools.lru_cache(maxsize=None)
def _damaged():
    base = make_case('base', 30, rate=8000, total=2 * frame_length(8000) + 3000)
    data = base.tta()
    offs = base.frame_offsets()
    n = len(base.frames)
    seek = 22 + 0
    out = []

    def add(name, d, frame, regex, kernel):
        out.append((name, d, frame, regex, kernel))

    def flip(d, at):
        return d[:at] + bytes([d[at] ^ 0x40]) + d[at + 1:]
    add('header_crc', flip(data, 19), None, 'TTA header CRC mismatch', False)
    add('seek_crc', flip(data, seek + 4 * n + 1), None, 'TTA seek table CRC mismatch', False)
    add('frame_crc', flip(data, offs[1] + len(base.frames[1]) - 2), 1, 'CRC mismatch', True)
    f1 = base.frames[1][:-4]
    add('bitstream_past', _with_frame(base, 1, _recrc(f1[:len(f1) // 2])), 1, 'reads past the frame', True)
    add('not_on_crc', _with_frame(base, 1, _recrc(f1 + b'\0')), 1, 'does not end on its CRC', True)
    sizes = [len(f) for f in base.frames]
    add('sizes_past', _rewrite_seek(data, seek, n, [sizes[0] + 1000] + sizes[1:]), n - 1,
        'runs past the end of the audio', False)
    add('sizes_short', _rewrite_seek(data, seek, n, sizes[:-1] + [sizes[-1] - 10]), None, 'seek table sizes end at byte',
        False)
    add('cut_last_frame', data[:-7], n - 1, 'runs past the end of the audio', False)
    add('seek_table_past_file', data[:seek + 3], None, 'seek table of 3 frames runs past the end of the file', False)
    for name, fmt, channels, bits, regex in (('encrypted', 2, 2, 16, r'is encrypted TTA \(format 2\)'),
                                             ('format3', 3, 2, 16, r'is TTA format 3'),
                                             ('8-bit', 1, 2, 8, r'is TTA at 8 bits'),
                                             ('9-channels', 1, 9, 16, r'is TTA with 9 channels')):
        pcm = signal(np.random.default_rng([7, channels, bits]), 2000, channels, bits, 'tone')
        c = make_case(name, 31, rate=8000, channels=channels, bits=bits, pcm=pcm)
        c.fmt = fmt
        add(name, c.tta(), None, regex, False)
    early = early_case()
    add('early_end', early.tta(), 0, "frame ends at the last frame's sample count", True)
    return base, tuple(out)


def damaged_cases():
    """(base case, [(name, bytes, frame index or None, regex of the refusal, refused by the GPU decoder)])"""
    base, out = _damaged()
    return base, list(out)


def early_case():
    """A silent mono stream one sample short of two frames: after frame 0's (frame length - 1)th sample only its last
    code, padding and CRC are left, so FFmpeg's decoder ends that frame there (the short-last-frame test it makes in
    every frame)."""
    fl = frame_length(8000)
    return make_case('early', 32, rate=8000, channels=1, pcm=np.zeros((2 * fl - 1, 1), np.int64))


def long_stream(bits=24, minutes=90, rate=48000, seed=40, kind='tone'):
    """A stereo case of one whole frame and a short one, and the .tta bytes of `minutes` minutes: the whole frame
    repeated, then the short one: (case, data, repeats)."""
    fl = frame_length(rate)
    case = make_case('long', seed, rate=rate, bits=bits, total=fl + 1000, kind=kind)
    reps = minutes * 60 * rate // fl
    frames = [case.frames[0]] * reps + [case.frames[1]]
    total = reps * fl + 1000
    data = header(2, bits, rate, total) + seek_table(frames) + b''.join(frames)
    return case, data, reps


def long_pcm16(case, reps):
    fl = case.frame_length
    p = case.pcm16
    return np.concatenate([np.tile(p[:fl], (reps, 1)), p[fl:]])
