"""Seeded Monkey's Audio 3.99 streams for the tests: the frames come from tests/ape_writer.cpp (compiled here with g++,
the encoder mirror of each decoder stage), and this module lays out the file around them: an optional ID3v2 tag, the
descriptor, the header, the seek table, the frames as 32-bit little-endian words counted from the first frame, and an
optional APEv2 / ID3v1 tag.

`all_cases()` are the good streams, `damaged_cases()` copies FFmpeg or the decoder must refuse, `long_stream()` a
stream of one full-size frame repeated, and `assert_coverage()` checks that the cases reach every corner the decoder
has.  Test infrastructure only."""
import ctypes
import os
import struct
import subprocess
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, 'tests', 'ape_writer.cpp')
LIB = os.path.join(ROOT, 'tests', 'emu', '_build', 'libape_writer.so')
LEVELS = (1000, 2000, 3000, 4000, 5000)
# Monkey's Audio's frame sizes, as its compressor sets them for version 3.99 and later: 73728 blocks, 4 times that at
# extra high and 16 times at insane
FULL = {1000: 73728, 2000: 73728, 3000: 73728, 4000: 73728 * 4, 5000: 73728 * 16}
MODES = {'coded': 0, 'pseudo': 1, 'silence': 2}

_lib = None


def writer():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SOURCE):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            tmp = LIB + '.%d' % os.getpid()
            subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-shared', '-fPIC', SOURCE, '-o', tmp])
            os.replace(tmp, LIB)
        lib = ctypes.CDLL(LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        lib.ape_encode_frame.argtypes = [vp, i64, i32, i32, i32, i32, i32, i32, vp, i64, vp]
        lib.ape_encode_frame.restype = i64
        _lib = lib
    return _lib


def encode_frame(pcm, channels, bits, level, mode='coded', flags_word=False, escape_every=0):
    """(frame bytes, stats dict) of one frame of interleaved int32 pcm (blocks, channels)"""
    pcm = np.ascontiguousarray(pcm, np.int32)
    cap = pcm.size * 8 + 4096
    out = np.zeros(cap, np.uint8)
    stats = np.zeros(8, np.int64)
    n = writer().ape_encode_frame(pcm.ctypes.data_as(ctypes.c_void_p), len(pcm), channels, bits, level,
                                  MODES[mode], int(flags_word), escape_every, out.ctypes.data_as(ctypes.c_void_p), cap,
                                  stats.ctypes.data_as(ctypes.c_void_p))
    assert n > 0
    keys = ('escapes', 'max_overflow', 'max_pivot', 'saturated', 'big_pivots', 'min_pivot')
    return out[:n].tobytes(), dict(zip(keys, (int(v) for v in stats[:6])))


def id3v2(size=40):
    body = b'\0' * size
    return b'ID3\x03\x00\x00' + bytes([(size >> 21) & 127, (size >> 14) & 127, (size >> 7) & 127, size & 127]) + body


def apev2():
    item = struct.pack('<II', 5, 0) + b'Title\0' + b'hello'
    footer = b'APETAGEX' + struct.pack('<IIII', 2000, len(item) + 32, 1, 0) + b'\0' * 8
    header = b'APETAGEX' + struct.pack('<IIII', 2000, len(item) + 32, 1, 0xA0000000) + b'\0' * 8
    return header + item + footer


def id3v1():
    return b'TAG' + b'\0' * 125


def layout(frames, channels, bits, rate, level, blocks_per_frame, final_blocks, head=b'', tail=b'', version=3990,
           seek=None, total_frames=None):
    """The file bytes of `frames` (each frame's own bytes).  seek: the seek table's entries in place of the true ones;
    total_frames: the header's frame count in place of len(frames)."""
    n = len(frames)
    total_frames = n if total_frames is None else total_frames
    table_len = 4 * (len(seek) if seek is not None else n)
    first = 52 + 24 + table_len
    starts, at = [], first
    for fr in frames:
        starts.append(at)
        at += len(fr)
    blob = b''.join(frames)
    blob += b'\0' * (-len(blob) % 4)
    blob = np.frombuffer(blob, '>u4').astype('<u4').tobytes()
    entries = seek if seek is not None else starts
    desc = b'MAC ' + struct.pack('<HHIIIIIII', version, 0, 52, 24, table_len, 0, len(blob), 0, 0) + b'\0' * 16
    hdr = struct.pack('<HHIIIHHI', level, 0, blocks_per_frame, final_blocks, total_frames, bits, channels, rate)
    table = struct.pack('<%dI' % len(entries), *entries)
    return head + desc + hdr + table + blob + tail, [len(head) + s for s in starts]


class Case(object):
    """One stream: pcm (samples, channels) int64 at `bits` bits, coded at `level` in frames of `bpf` blocks."""

    def __init__(self, name, pcm, channels, bits, rate, level, bpf, modes=None, head=b'', tail=b'', flags_word=False,
                 escape_every=0):
        self.name, self.pcm, self.channels, self.bits, self.rate, self.level, self.bpf = (
            name, pcm, channels, bits, rate, level, bpf)
        self.head, self.tail, self.flags_word, self.escape_every = head, tail, flags_word, escape_every
        n = (len(pcm) + bpf - 1) // bpf
        self.modes = modes or ['coded'] * n
        assert len(self.modes) == n
        self._built = None

    @property
    def pcm16(self):
        return (self.pcm if self.bits == 16 else self.pcm >> 8).astype(np.int16)

    def frames(self):
        if self._built is None:
            out, stats = [], []
            for i, mode in enumerate(self.modes):
                block = self.pcm[i * self.bpf:(i + 1) * self.bpf]
                data, st = encode_frame(block, self.channels, self.bits, self.level, mode, self.flags_word,
                                        self.escape_every)
                out.append(data)
                stats.append(st)
            self._built = out, stats
        return self._built

    @property
    def final_blocks(self):
        return len(self.pcm) - (len(self.modes) - 1) * self.bpf

    def ape(self, **kw):
        data, _ = layout(self.frames()[0], self.channels, self.bits, self.rate, self.level, self.bpf, self.final_blocks,
                         self.head, self.tail, **kw)
        return data

    def frame_offsets(self):
        return layout(self.frames()[0], self.channels, self.bits, self.rate, self.level, self.bpf, self.final_blocks,
                      self.head, self.tail)[1]


def _signal(rng, n, channels, bits, kind):
    top = (1 << (bits - 1)) - 1
    t = np.arange(n)
    if kind == 'tone':
        x = np.stack([np.sin(t * (0.01 + 0.013 * c)) * 0.6 * top for c in range(channels)], 1)
        x += rng.normal(0, top / 300, (n, channels))
    elif kind == 'noise':
        x = rng.normal(0, top / 3, (n, channels))
    elif kind == 'full':                                  # full-scale jumps: large residuals, extreme k, escapes
        x = rng.choice([-top - 1, top, 0, top // 2], (n, channels)).astype(np.float64)
    elif kind == 'quiet':                                 # digital near-silence: k down to 0
        x = np.zeros((n, channels))
        x[rng.integers(0, n, max(1, n // 5000))] = 1
    else:
        raise ValueError(kind)
    return np.clip(np.round(x), -top - 1, top).astype(np.int64)


def make_case(name, channels, bits, level, total, bpf, rate=44100, kind='tone', seed=1, modes=None, **kw):
    rng = np.random.default_rng(seed)
    pcm = _signal(rng, total, channels, bits, kind)
    n = (total + bpf - 1) // bpf
    modes = modes or ['coded'] * n
    for i, m in enumerate(modes):
        if m == 'silence':
            pcm[i * bpf:(i + 1) * bpf] = 0
        elif m == 'pseudo':
            pcm[i * bpf:(i + 1) * bpf, 1] = pcm[i * bpf:(i + 1) * bpf, 0]
    return Case(name, pcm, channels, bits, rate, level, bpf, modes, **kw)


_cases = None


def all_cases():
    global _cases
    if _cases is not None:
        return _cases
    cs = []
    for level in LEVELS:
        for channels in (1, 2):
            for bits in (16, 24):
                cs.append(make_case('l%d_%dch_%d' % (level // 1000, channels, bits), channels, bits, level, 3 * 4096 - 1,
                                    4096, seed=level + channels + bits))
    # full-size frames at every level (the last one cut short), stereo 16-bit, one at 24 bits
    for level in LEVELS:
        bpf = FULL[level]
        cs.append(make_case('full%d' % (level // 1000), 2, 16, level, bpf + 777, bpf, rate=48000, seed=level))
    cs.append(make_case('full5_24', 2, 24, 5000, FULL[5000] + 1, FULL[5000], rate=96000, kind='noise', seed=9))
    # totals at, one above and one below a frame multiple; odd and high rates
    cs.append(make_case('at_multiple', 2, 16, 2000, 3 * 1000, 1000, rate=7919, seed=21))
    cs.append(make_case('one_above', 2, 16, 3000, 3 * 1000 + 1, 1000, rate=192000, seed=22))
    cs.append(make_case('one_below', 1, 24, 4000, 3 * 1000 - 1, 1000, rate=11025, seed=23))
    cs.append(make_case('one_block', 2, 16, 5000, 1, 1000, rate=8000, seed=24))
    # special frames
    cs.append(make_case('specials_stereo', 2, 16, 3000, 5 * 2000, 2000, seed=31,
                        modes=['coded', 'silence', 'pseudo', 'coded', 'pseudo']))
    cs.append(make_case('specials_mono', 1, 16, 2000, 3 * 2000, 2000, seed=32, modes=['silence', 'coded', 'silence']))
    cs.append(make_case('specials_24', 2, 24, 5000, 3 * 2000, 2000, seed=33, modes=['pseudo', 'silence', 'coded']))
    cs.append(make_case('flags_word', 2, 16, 1000, 2 * 2000, 2000, seed=34, flags_word=True))
    # entropy extremes: full-scale jumps (extreme k, large pivots, escapes), quiet (k to 0), forced escapes
    cs.append(make_case('jumps24', 2, 24, 1000, 6000, 3000, kind='full', seed=41))
    cs.append(make_case('jumps16', 1, 16, 5000, 6000, 3000, kind='full', seed=42))
    cs.append(make_case('quiet', 2, 16, 3000, 20000, 10000, kind='quiet', seed=43))
    cs.append(make_case('escapes', 2, 16, 2000, 4000, 2000, seed=44, escape_every=7))
    # NN inputs that saturate int16
    cs.append(make_case('noise16', 2, 16, 5000, 8000, 4000, kind='noise', seed=45))
    # 24-bit stereo samples at +2^23 and -2^23: the widest FFmpeg decodes in its default predictor mode (+2^23 reaches
    # its S32 output as -2^31, so the top 16 bits are -32768)
    edge = make_case('edge24', 2, 24, 4000, 4000, 2000, seed=53)
    edge.pcm[100, 0] = 1 << 23
    edge.pcm[2100, 1] = -(1 << 23)
    edge.pcm[3000] = [1 << 23, -(1 << 23)]
    cs.append(edge)
    # tags at both ends
    cs.append(make_case('tags', 2, 16, 4000, 5000, 2000, seed=51, head=id3v2(), tail=apev2() + id3v1()))
    cs.append(make_case('id3v1_only', 1, 16, 1000, 3000, 2000, seed=52, tail=id3v1()))
    _cases = cs
    return cs


def assert_coverage(cases):
    seen = {(c.level, c.channels, c.bits) for c in cases}
    for level in LEVELS:
        for channels in (1, 2):
            for bits in (16, 24):
                assert (level, channels, bits) in seen
    stats = [s for c in cases for s in c.frames()[1]]
    assert any(s['escapes'] for s in stats) and max(s['max_overflow'] for s in stats) >= 63
    assert max(s['max_pivot'] for s in stats) >= 1 << 23 and min(s['min_pivot'] for s in stats) == 1
    assert any(s['big_pivots'] for s in stats)
    assert any(s['saturated'] for c in cases if c.level > 1000 for s in c.frames()[1])
    modes = {(c.channels, m) for c in cases for m in c.modes}
    assert {(1, 'silence'), (2, 'silence'), (2, 'pseudo'), (1, 'coded'), (2, 'coded')} <= modes
    assert any(c.flags_word for c in cases)
    assert any(c.head for c in cases) and any(c.tail for c in cases)
    rates = {c.rate for c in cases}
    assert min(rates) < 8000 and max(rates) >= 192000 and any(r % 2 for r in rates)
    assert any(len(c.pcm) % c.bpf == 0 for c in cases) and any(len(c.pcm) % c.bpf == 1 for c in cases)
    assert any(len(c.pcm) % c.bpf == c.bpf - 1 for c in cases)
    assert {c.bpf for c in cases} >= set(FULL.values()) and min(c.bpf for c in cases) <= 1000
    skips = {(o - c.frame_offsets()[0]) % 4 for c in cases for o in c.frame_offsets()}
    assert skips == {0, 1, 2, 3}


def damaged_cases():
    """(base case, [(name, file bytes, frame, regex, found on the GPU)]): frame is the refused frame, or None for a
    refusal of the whole file."""
    base = make_case('damage_base', 2, 16, 3000, 4 * 2000, 2000, seed=61)
    good = base.ape()
    offs = base.frame_offsets()
    frames = base.frames()[0]
    out = []

    def patched(at, value):
        b = bytearray(good)
        b[at] ^= value
        return bytes(b)

    def word_byte(frame, i):
        # file position of byte i of frame `frame` (the file holds 32-bit words counted from the first frame)
        rel = offs[frame] - offs[0] + i
        return offs[0] + (rel & ~3) + 3 - (rel & 3)

    out.append(('version', patched(4, 0x10), None, r'file version 3\.97 \(3974\)', False))
    out.append(('bits8', good[:52 + 16] + struct.pack('<H', 8) + good[52 + 18:], None, '8 bits', False))
    out.append(('bits32', good[:52 + 16] + struct.pack('<H', 32) + good[52 + 18:], None, '32 bits', False))
    out.append(('channels3', good[:52 + 18] + struct.pack('<H', 3) + good[52 + 20:], None, '3 channels', False))
    out.append(('level6000', struct.pack('<H', 6000).join([good[:52], good[54:]]), None, 'compression level 6000',
                False))
    out.append(('level1500', struct.pack('<H', 1500).join([good[:52], good[54:]]), None, 'compression level 1500',
                False))
    out.append(('rate_2g', good[:52 + 20] + struct.pack('<I', 1 << 31) + good[52 + 24:], None,
                'APE sample rate 2147483648 is not supported', False))
    out.append(('blocks_huge', good[:52 + 4] + struct.pack('<II', 1 << 30, 1) + good[52 + 12:], None,
                'APE frames of 1073741824 blocks are not supported', False))
    out.append(('seek_short', base.ape(seek=[offs[0] - len(base.head), offs[1], offs[2]]), None,
                'seek table of 3 entries is cut short: the header gives 4 frames', False))
    bad = list(o - len(base.head) for o in offs)
    bad[2] = bad[1] - 4
    out.append(('seek_backwards', base.ape(seek=bad), None, 'seek table is inconsistent: frame 2 at byte offset .* '
                'does not follow frame 1', False))
    bad = list(o - len(base.head) for o in offs)
    bad[3] = len(good) + 100
    out.append(('seek_past_end', base.ape(seek=bad), None, 'seek table is inconsistent: frame 3 at byte offset .* '
                'starts past the end of the audio', False))
    out.append(('crc', patched(word_byte(1, 3), 0x01), 1, 'CRC mismatch', True))
    out.append(('flags', _set_flags(base, 2, 0x10), 2, 'invalid frame flags', True))
    out.append(('payload', patched(word_byte(1, 40), 0x55), 1, 'range decoder runs past the frame', True))
    # the last frame cut: the range decoder runs past it
    cut = good[:offs[3] + 12]
    cut += b'\0' * (-len(cut) % 4)
    out.append(('cut_last', cut, 3, 'range decoder runs past the frame', True))
    # a 24-bit stereo sample one past 2^23 in frame 1 (FFmpeg's test for its 64-bit predictor mode is |sample| > 2^23)
    out.append(('interim24', interim_case().ape(), 1, 'outside 24 bits', True))
    return base, out


def interim_case():
    """24-bit stereo, 3 frames; frame 1 holds a left sample of 2^23 + 1, past what 24 bits hold"""
    case = make_case('interim24', 2, 24, 3000, 3 * 2000, 2000, seed=62)
    case.pcm[2500, 0] = (1 << 23) + 1
    return case


def wrap24(pcm):
    """24-bit samples as FFmpeg's S32P holds them (the sample times 256, in 32 bits), shifted back down"""
    return ((np.asarray(pcm, np.int64) + (1 << 23)) & ((1 << 24) - 1)) - (1 << 23)


def _set_flags(case, frame, flags):
    frames = list(case.frames()[0])
    fr = bytearray(frames[frame])
    word = struct.unpack('>I', bytes(fr[:4]))[0]
    if word & 0x80000000:
        fr[4:8] = struct.pack('>I', struct.unpack('>I', bytes(fr[4:8]))[0] | flags)
    else:
        fr[0:4] = struct.pack('>I', word | 0x80000000)
        fr[4:4] = struct.pack('>I', flags)
    frames[frame] = bytes(fr)
    return layout(frames, case.channels, case.bits, case.rate, case.level, case.bpf, case.final_blocks, case.head,
                  case.tail)[0]


def long_stream(bits=16, minutes=90, level=5000, rate=48000):
    """(case of one full-size frame, file bytes of that frame repeated for `minutes`, repeats)"""
    bpf = FULL[level]
    case = make_case('long%d' % bits, 2, bits, level, bpf, bpf, rate=rate, kind='tone', seed=77)
    frame = case.frames()[0][0]
    frame += b'\0' * (-len(frame) % 4)
    reps = max(1, minutes * 60 * rate // bpf)
    swapped = np.frombuffer(frame, '>u4').astype('<u4').tobytes()
    first = 52 + 24 + 4 * reps
    seek = [first + i * len(frame) for i in range(reps)]
    head, _ = layout([], 2, bits, rate, level, bpf, bpf, seek=seek, total_frames=reps)
    return case, head + swapped * reps, reps


def long_pcm16(case, reps):
    return np.tile(case.pcm16, (reps, 1))


def crc_of(data):
    return zlib.crc32(data)
