"""Seeded TAK streams for the tests: each frame's data comes from tests/tak_writer.cpp (compiled here with g++, the
encoder mirror of each decoder stage), and this module lays out the file around them: an optional ID3v2 tag, the
`tBaK` marker, the metadata blocks (STREAMINFO with its CRC-24, and optionally SEEKTABLE, ENCODER, MD5, PADDING and
LAST_FRAME), the frames (header with its CRC-24, data, data CRC-24), and an optional APEv2 / ID3v1 tag.

`all_cases()` are the good streams, `damaged_cases()` copies FFmpeg or the decoder must refuse, `long_stream()` a
stream of one full-size frame repeated, and `assert_coverage()` checks that the cases reach every corner the decoder
has.  Test infrastructure only."""
import ctypes
import os
import struct
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, 'tests', 'tak_writer.cpp')
LIB = os.path.join(ROOT, 'tests', 'emu', '_build', 'libtak_writer.so')
# the writer's option and stats slots (tak_writer.cpp's O_* and S_*)
OPTIONS = ('dmode', 'ch_lpc', 'max_shift', 'order', 'nsub', 'escape_every', 'mc', 'filtered', 'cont', 'partition',
           'pred', 'dshift')
DEFAULTS = dict(dmode=-1, ch_lpc=-1, max_shift=-1, order=-1, nsub=0, escape_every=0, mc=1, filtered=80, cont=-1,
                partition=-1, pred=1, dshift=4)
STATS = ('orders', 'sub_lpc', 'ch_lpc', 'nsub', 'cont', 'paths', 'partitioned', 'deltas', 'dmodes', 'mc_index',
         'chained', 'shifts', 'clips', 'wraps', 'zero_segments', 'fresh', 'dvals', 'fir_orders')
ORDERS = (4, 8, 12, 16, 24, 32, 48, 64, 80, 96, 128, 160, 192, 224, 256)
FRAME_TYPES = (3, 4, 6, 8, 4096, 8192, 16384, 512, 1024, 2048)   # quarter-32nds of a second (0-3), or samples
# FFmpeg's tak_channel_layouts: TAK speaker code -> channel mask bit
SPEAKERS = {1: 0x1, 2: 0x2, 3: 0x4, 4: 0x8, 5: 0x10, 6: 0x20, 7: 0x40, 8: 0x80, 9: 0x100, 10: 0x200, 11: 0x400}
METADATA = {'end': 0, 'streaminfo': 1, 'seektable': 2, 'wavedata': 3, 'encoder': 4, 'padding': 5, 'md5': 6,
            'last_frame': 7}

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
        vp = ctypes.c_void_p
        lib.tak_encode_data.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_uint64, vp, vp, ctypes.c_int64, vp]
        lib.tak_encode_data.restype = ctypes.c_int64
        _lib = lib
    return _lib


# ---- CRC-24 (FFmpeg's AV_CRC_24_IEEE from 0xCE04B7; stored little-endian) ----

def _crc_table():
    t = []
    for i in range(256):
        r = i << 16
        for _ in range(8):
            r = ((r << 1) ^ (0x864CFB if r & 0x800000 else 0)) & 0xFFFFFF
        t.append(r)
    return t


_TABLE = _crc_table()


def crc24(data, r=0xB704CE):
    t = _TABLE
    for b in data:
        r = ((r << 8) & 0xFFFFFF) ^ t[(r >> 16) ^ b]
    return r


def with_crc(data):
    return data + struct.pack('<I', crc24(data))[:3]


# ---- bit packing (FFmpeg's little-endian reader: first bit lowest) ----

class Bits(object):
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, width):
        self.v |= (value & ((1 << width) - 1)) << self.n
        self.n += width
        return self

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, 'little')


def put_info(b, codec, frame_type, samples, rate, bits, channels, speakers=None, data_type=0):
    b.put(codec, 6).put(0, 4).put(frame_type, 4).put(samples, 35).put(data_type, 3).put(rate - 6000, 18)
    b.put(bits - 8, 5).put(channels - 1, 4)
    if speakers is None:
        b.put(0, 1)
    else:
        b.put(1, 1).put(0, 5).put(1, 1)
        for s in speakers:
            b.put(s, 6)
    return b


def streaminfo(codec, frame_type, samples, rate, bits, channels, speakers=None, data_type=0):
    return put_info(Bits(), codec, frame_type, samples, rate, bits, channels, speakers, data_type).bytes()


def frame_header(number, info=None, last=None, metadata=False):
    """a frame header with its CRC: info, the put_info arguments of a frame carrying stream info; last, the samples of
    the last frame"""
    b = Bits().put(0xA0FF, 16).put((1 if last else 0) | (2 if info else 0) | (4 if metadata else 0), 3).put(number, 21)
    if last:
        b.put(last - 1, 14).put(0, 2)
    if info:
        put_info(b, *info)
        b.put(0, 6)
    return with_crc(b.bytes())


def block(kind, payload, crc=True):
    body = with_crc(payload) if crc else payload
    return bytes([METADATA[kind]]) + struct.pack('<I', len(body))[:3] + body


def id3v2(size=40):
    body = b'\0' * size
    return b'ID3\x03\x00\x00' + bytes([(size >> 21) & 127, (size >> 14) & 127, (size >> 7) & 127, size & 127]) + body


def apev2():
    item = struct.pack('<II', 5, 0) + b'Title\0' + b'hello'
    footer = b'APETAGEX' + struct.pack('<IIII', 2000, len(item) + 32, 1, 0x80000000) + b'\0' * 8
    header = b'APETAGEX' + struct.pack('<IIII', 2000, len(item) + 32, 1, 0xA0000000) + b'\0' * 8
    return header + item + footer


def id3v1():
    return b'TAG' + b'\0' * 125


def frame_samples(rate, frame_type):
    """FFmpeg's tak_get_nb_samples, 0 where it refuses"""
    q = FRAME_TYPES[frame_type]
    if frame_type <= 3:
        n, top = rate * q >> 5, 16384
    else:
        n, top = q, rate * 8 >> 5
    return n if 0 < n <= top else 0


def encode_data(pcm, bits, rate, codec, seed, **opts):
    """(data bytes, stats) of one frame of pcm (n, channels)"""
    o = dict(DEFAULTS, **opts)
    n, channels = pcm.shape
    planar = np.ascontiguousarray(pcm.T, np.int32)
    cap = n * channels * 16 + 65536
    out = np.zeros(cap, np.uint8)
    stats = np.zeros(len(STATS), np.int64)
    opt = np.array([o[k] for k in OPTIONS], np.int32)
    size = writer().tak_encode_data(planar.ctypes.data_as(ctypes.c_void_p), n, channels, bits, rate, codec, seed,
                                    opt.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), cap,
                                    stats.ctypes.data_as(ctypes.c_void_p))
    assert size > 0
    return out[:size].tobytes(), dict(zip(STATS, (int(v) for v in stats)))


class Case(object):
    """One stream: pcm (samples, channels) int64 at `bits` bits, in frames of frame size type `frame_type`.
    opts: the writer's options, for every frame (or per frame by a list of dicts in `frame_opts`).  info_every: every
    how many frames carry stream info (frame 0 always does).  blocks: optional metadata blocks in order ('seektable',
    'encoder', 'md5', 'padding', 'last_frame').  speakers: TAK speaker codes of the layout, None for none."""

    def __init__(self, name, pcm, bits, rate, frame_type, codec=None, speakers=None, info_every=0, blocks=(),
                 head=b'', tail=b'', seed=1, frame_opts=None, **opts):
        self.name, self.pcm, self.bits, self.rate, self.frame_type = name, pcm, bits, rate, frame_type
        self.channels = pcm.shape[1]
        self.codec = codec or (2 if self.channels <= 2 else 4)
        self.speakers, self.info_every, self.blocks = speakers, info_every, tuple(blocks)
        self.head, self.tail, self.seed, self.opts, self.frame_opts = head, tail, seed, opts, frame_opts
        self.nb = frame_samples(rate, frame_type)
        assert self.nb > 0, (rate, frame_type)
        self._built = None

    @property
    def mask(self):
        return 0 if self.speakers is None else sum(SPEAKERS[s] for s in self.speakers)

    @property
    def pcm16(self):
        return (self.pcm if self.bits == 16 else self.pcm >> 8).astype(np.int16)

    def info(self):
        return (self.codec, self.frame_type, len(self.pcm), self.rate, self.bits, self.channels, self.speakers)

    def frames(self):
        """([frame bytes], [stats])"""
        if self._built is None:
            out, stats = [], []
            n = (len(self.pcm) + self.nb - 1) // self.nb
            for i in range(n):
                block_pcm = self.pcm[i * self.nb:(i + 1) * self.nb]
                opts = dict(self.opts, **(self.frame_opts[i % len(self.frame_opts)] if self.frame_opts else {}))
                data, st = encode_data(block_pcm, self.bits, self.rate, self.codec, self.seed * 1000003 + i, **opts)
                info = self.info() if i == 0 or (self.info_every and i % self.info_every == 0) else None
                head = frame_header(i, info, len(block_pcm) if i == n - 1 else None)
                out.append(head + with_crc(data))
                stats.append(st)
            self._built = out, stats
        return self._built

    def metadata(self, frames):
        si = streaminfo(*self.info()[:2], len(self.pcm), self.rate, self.bits, self.channels, self.speakers)
        out = [block('streaminfo', si)]
        for kind in self.blocks:
            if kind == 'seektable':
                out.append(block('seektable', b'\x01\x00' + b'\0' * 20, crc=False))
            elif kind == 'encoder':
                out.append(block('encoder', struct.pack('<I', 0x020301)[:3] + b'\x00'))
            elif kind == 'md5':
                out.append(block('md5', bytes(range(16))))
            elif kind == 'padding':
                out.append(block('padding', b'\0' * 37, crc=False))
            elif kind == 'last_frame':
                pos = sum(len(f) for f in frames[:-1])
                b = Bits().put(pos, 40).put(len(frames[-1]), 24)
                out.append(block('last_frame', b.bytes()))
        out.append(bytes([0, 0, 0, 0]))
        return b''.join(out)

    def layout(self, frames=None):
        """(file bytes, [frame offsets], audio start)"""
        frames = self.frames()[0] if frames is None else frames
        head = self.head + b'tBaK' + self.metadata(frames)
        offs, at = [], len(head)
        for f in frames:
            offs.append(at)
            at += len(f)
        return head + b''.join(frames) + self.tail, offs, len(head)

    def tak(self):
        return self.layout()[0]

    def frame_offsets(self):
        return self.layout()[1]


def _signal(rng, n, channels, bits, kind, shift=0):
    top = (1 << (bits - 1)) - 1
    t = np.arange(n)
    if kind == 'tone':
        x = np.stack([np.sin(t * (0.01 + 0.013 * c)) * 0.6 * top for c in range(channels)], 1)
        x += rng.normal(0, top / 300, (n, channels))
    elif kind == 'corr':                                  # channels close to each other: what decorrelation is for
        base = np.sin(t * 0.007) * 0.5 * top + rng.normal(0, top / 200, n)
        x = np.stack([base * (1 - 0.1 * c) + rng.normal(0, top / 500, n) for c in range(channels)], 1)
    elif kind == 'noise':
        x = rng.normal(0, top / 3, (n, channels))
    elif kind == 'full':                                  # full-scale jumps: the clip, int16 history wrap, escapes
        x = rng.choice([-top - 1, top, 0, top // 2, -top], (n, channels)).astype(np.float64)
    elif kind == 'quiet':
        x = np.zeros((n, channels))
        x[rng.integers(0, n, max(1, n // 500))] = 1
    else:
        raise ValueError(kind)
    x = np.clip(np.round(x), -top - 1, top).astype(np.int64)
    return x >> shift << shift


def make_case(name, channels, bits, total, rate=44100, frame_type=None, kind='tone', seed=1, shift=0, **kw):
    rng = np.random.default_rng(seed)
    if frame_type is None:
        frame_type = next(t for t in (7, 8, 9, 4) if frame_samples(rate, t))
    return Case(name, _signal(rng, total, channels, bits, kind, shift), bits, rate, frame_type, seed=seed, **kw)


_cases = None


def all_cases():
    global _cases
    if _cases is not None:
        return _cases
    cs = []
    # every predictor order, alone, fresh and continued, at both widths
    for i, order in enumerate(ORDERS):
        cs.append(make_case('order%d' % order, 1 + i % 2, 16 if i % 3 else 24, 3 * 2048 + 100, rate=44100,
                            frame_type=9, seed=100 + i, order=i, filtered=100, nsub=1 + i % 4, pred=2 if i % 2 else 1))
    # every stereo dmode, with the filtered ones on both orders and dval flags
    for dmode in range(8):
        cs.append(make_case('dmode%d' % dmode, 2, 16 if dmode % 2 else 24, 4 * 1024 + 7, rate=48000, frame_type=8,
                            kind='corr', seed=200 + dmode, dmode=dmode))
    # channel lpc modes, subframe counts, continuation forced and never
    for lpc in range(4):
        cs.append(make_case('chlpc%d' % lpc, 2, 16, 3 * 4096, rate=44100, frame_type=4, seed=300 + lpc, ch_lpc=lpc,
                            nsub=8, cont=1 if lpc % 2 else 0))
    # sample shifts: every shift of each width through channels whose samples are multiples of 2^shift
    for bits, shifts in ((16, range(16)), (24, range(0, 17, 2))):
        for s in shifts:
            cs.append(make_case('shift%d_%d' % (bits, s), 1, bits, 600, rate=22050, frame_type=7, kind='noise',
                                seed=400 + s + bits, shift=s, max_shift=s))
    # multichannel: identity lists, random pair lists and chained pairs, up to 6 channels (FFmpeg's limit), layouts
    cs.append(make_case('mc6_plain', 6, 16, 3 * 2048, rate=48000, frame_type=9, kind='corr', seed=501, mc=0,
                        speakers=[1, 2, 3, 4, 5, 6]))
    cs.append(make_case('mc6_pairs', 6, 24, 5 * 2048 + 3, rate=48000, frame_type=9, kind='corr', seed=502, mc=1))
    cs.append(make_case('mc6_chained', 6, 16, 6 * 2048, rate=96000, frame_type=9, kind='corr', seed=503, mc=2,
                        speakers=[1, 2, 3, 4, 10, 11]))
    cs.append(make_case('mc3', 3, 16, 4 * 1024, rate=32000, frame_type=8, kind='corr', seed=504, mc=2, codec=4))
    cs.append(make_case('mc_mono', 1, 16, 2000, rate=16000, frame_type=7, seed=505, codec=4))
    # rates and frame size types
    for ft, rate in ((0, 44100), (1, 48000), (2, 48000), (3, 44100), (4, 192000), (5, 192000), (6, 192000),
                     (7, 6000), (8, 7919), (9, 11025)):
        cs.append(make_case('ft%d_%d' % (ft, rate), 2, 16 if ft % 2 else 24, 2 * frame_samples(rate, ft) + 333,
                            rate=rate, frame_type=ft, seed=600 + ft))
    # totals at, one above and one below a frame multiple, and a stream shorter than one frame; frames of under 16
    cs.append(make_case('at_multiple', 2, 16, 3 * 1024, rate=44100, frame_type=8, seed=701))
    cs.append(make_case('one_above', 2, 16, 3 * 1024 + 1, rate=44100, frame_type=8, seed=702))
    cs.append(make_case('one_below', 1, 24, 3 * 1024 - 1, rate=44100, frame_type=8, seed=703))
    cs.append(make_case('short_last', 2, 24, 2 * 512 + 15, rate=44100, frame_type=7, seed=704))
    cs.append(make_case('tiny', 2, 16, 9, rate=44100, frame_type=7, seed=705))
    # entropy extremes: full-scale jumps with wild predictors (the 14-bit clip, int16 history wrap, big escapes),
    # digital near-silence (mode 0), forced escapes
    cs.append(make_case('jumps16', 2, 16, 3 * 2048, rate=48000, frame_type=9, kind='full', seed=801, pred=2, dshift=0,
                        filtered=100))
    cs.append(make_case('jumps24', 2, 24, 3 * 2048, rate=48000, frame_type=9, kind='full', seed=802, pred=2, dshift=0,
                        filtered=100))
    cs.append(make_case('quiet', 2, 16, 4 * 2048, rate=44100, frame_type=9, kind='quiet', seed=803))
    cs.append(make_case('escapes', 2, 16, 3 * 2048, rate=44100, frame_type=9, kind='noise', seed=804, escape_every=5))
    cs.append(make_case('partitioned', 1, 16, 3 * 4096, rate=44100, frame_type=4, kind='noise', seed=805,
                        partition=1, filtered=0))
    # 24-bit samples at +-(2^23 - 1)
    edge = make_case('edge24', 2, 24, 3 * 1024, rate=48000, frame_type=8, seed=901)
    edge.pcm[100, 0] = (1 << 23) - 1
    edge.pcm[1500, 1] = -(1 << 23) + 1
    edge.pcm[2000] = [(1 << 23) - 1, -(1 << 23) + 1]
    cs.append(edge)
    # frames carrying stream info, metadata blocks, LAST_FRAME present and absent, tags at both ends
    cs.append(make_case('info_every', 2, 16, 6 * 1024, rate=44100, frame_type=8, seed=1001, info_every=2,
                        blocks=('seektable', 'encoder', 'md5', 'padding', 'last_frame')))
    cs.append(make_case('tags', 2, 16, 4 * 1024, rate=44100, frame_type=8, seed=1002, head=id3v2(),
                        tail=apev2() + id3v1(), blocks=('last_frame',)))
    cs.append(make_case('tags_no_last', 1, 16, 3 * 1024, rate=44100, frame_type=8, seed=1003, tail=apev2() + id3v1()))
    _cases = cs
    return cs


def stats_of(cases):
    return [s for c in cases for s in c.frames()[1]]


def assert_coverage(cases):
    stats = stats_of(cases)

    def union(key):
        v = 0
        for s in stats:
            v |= s[key]
        return v

    assert union('orders') == (1 << 15) - 1, bin(union('orders'))
    assert union('sub_lpc') == 0b111 and union('ch_lpc') == 0b1111
    assert union('nsub') & 0x1FE == 0x1FE, bin(union('nsub'))
    assert sum(s['cont'] for s in stats) and sum(s['fresh'] for s in stats)
    assert union('paths') == 0x7F, bin(union('paths'))
    assert sum(s['partitioned'] for s in stats) and union('deltas') == 0x7F, bin(union('deltas'))
    assert sum(s['zero_segments'] for s in stats)
    assert union('dmodes') == 0xFF and union('mc_index') == 0xF and sum(s['chained'] for s in stats)
    assert union('dvals') == 3 and union('fir_orders') == 24
    for bits, top in ((16, 15), (24, 16)):
        seen = 0
        for c in cases:
            if c.bits == bits:
                for s in c.frames()[1]:
                    seen |= s['shifts']
        assert seen == (1 << (top + 1)) - 1 if bits == 16 else seen & 0x15555 == 0x15555, (bits, bin(seen))
    assert sum(s['clips'] for s in stats) and sum(s['wraps'] for s in stats)
    assert {c.frame_type for c in cases} == set(range(10))
    assert {1, 2, 3, 6} <= {c.channels for c in cases} and {16, 24} <= {c.bits for c in cases}
    assert {6000, 44100, 48000, 192000} <= {c.rate for c in cases} and any(c.rate % 2 for c in cases)
    assert any(len(c.pcm) % c.nb == 0 for c in cases) and any(len(c.pcm) % c.nb == 1 for c in cases)
    assert any(len(c.pcm) % c.nb == c.nb - 1 for c in cases) and any(len(c.pcm) < 16 for c in cases)
    assert any(c.info_every for c in cases)
    kinds = {k for c in cases for k in c.blocks}
    assert kinds == {'seektable', 'encoder', 'md5', 'padding', 'last_frame'}
    assert any('last_frame' not in c.blocks for c in cases)
    assert any(c.head for c in cases) and any(c.tail for c in cases)
    assert any(c.bits == 24 and np.abs(c.pcm).max() == (1 << 23) - 1 for c in cases)


# ---- damaged and refused copies ----

def _channel_bits(b, bits, first=0, shift=0, lpc=0, nsub_v=None, sub=None):
    """one channel as FFmpeg reads it, hand-made: sample shift, first sample, lpc mode, subframes (nsub_v: the boundary
    values of a second subframe and more), then `sub`(b) for the subframes (default: unfiltered, all-zero residuals)"""
    b.put(0, 1) if not shift else b.put(1, 1).put(shift - 1, 4)
    if shift >= bits:
        return b
    b.put(first, bits - shift).put(lpc, 2)
    vs = nsub_v or []
    b.put(len(vs), 3)
    for v in vs:
        b.put(v, 6)
    if sub:
        return sub(b)
    for _ in range(len(vs) + 1):
        b.put(0, 1).put(0, 1).put(0, 6)
    return b


def _frame(number, data_bits, info=None, last=None, metadata=False):
    return frame_header(number, info, last, metadata) + with_crc(data_bits.bytes())


def damaged_cases():
    """(base case, [(name, file bytes, frame, regex, found on the GPU)]): frame is the refused frame, or None for a
    refusal of the whole file."""
    base = make_case('damage_base', 2, 16, 4 * 1024, rate=44100, frame_type=8, seed=61, mc=0)
    frames = list(base.frames()[0])
    good, offs, start = base.layout()
    out = []

    def with_frames(fs, case=base):
        return case.layout(fs)[0]

    def info_with(**kw):
        v = dict(zip(('codec', 'frame_type', 'samples', 'rate', 'bits', 'channels', 'speakers'), base.info()))
        v.update(kw)
        return v

    def head_with(**kw):
        v = info_with(**kw)
        si = streaminfo(v['codec'], v['frame_type'], v['samples'], v['rate'], v['bits'], v['channels'], v['speakers'],
                        v.get('data_type', 0))
        return b'tBaK' + block('streaminfo', si) + b'\0\0\0\0'

    body = good[start:]

    def host(name, head, regex):
        out.append((name, head + body, None, regex, False))

    host('bits8', head_with(bits=8), 'TAK at 8 bits')
    host('channels7', head_with(codec=4, channels=7), 'TAK with 7 channels')
    host('stereo_codec_3ch', head_with(channels=3), r'TAK with 3 channels \(mono/stereo codec\)')
    host('data_type1', head_with(data_type=1), 'TAK of data type 1')
    host('codec3', head_with(codec=3), 'TAK of codec type 3')
    host('frame_type12', head_with(frame_type=12), 'TAK of frame size type 12')
    host('frame_type6_6k', head_with(frame_type=6, rate=6000), 'TAK of frame size type 6, invalid at 6000 Hz')
    host('no_streaminfo', b'tBaK' + block('padding', b'\0' * 8, crc=False) + b'\0\0\0\0', 'has no STREAMINFO')
    corrupt = bytearray(head_with())
    corrupt[10] ^= 0x40
    host('streaminfo_crc', bytes(corrupt), r'STREAMINFO is corrupt \(CRC mismatch\)')
    lf = Bits().put(10 ** 6, 40).put(100, 24).bytes()
    host('last_frame_past_end', head_with()[:-4] + block('last_frame', lf) + b'\0\0\0\0',
         'LAST_FRAME ends at byte offset .* past the end of the file')

    def gpu(name, fs, frame, regex, data=None):
        out.append((name, data if data is not None else with_frames(fs), frame, regex, True))

    crc = bytearray(frames[1])
    crc[-1] ^= 0x01
    gpu('data_crc', frames[:1] + [bytes(crc)] + frames[2:], 1, 'data CRC mismatch')
    gpu('trailing', frames[:1] + [frames[1] + b'\x00\x11'] + frames[2:], 1, 'bytes left after the data CRC')
    # the last frame's data cut by one byte (its CRC with it): the last bits are read past the frame
    gpu('cut_last', None, 3, 'data runs past the frame', data=good[:offs[3] + len(frames[3]) - 4])
    def crafted(number, data, last=None):
        fs = list(frames)
        fs[number] = _frame(number, data, last=last)
        return fs

    gpu('shift', crafted(1, _channel_bits(Bits(), 16, shift=16)), 1, 'sample shift at or above the bit depth')
    gpu('subframes', crafted(2, _channel_bits(Bits(), 16, nsub_v=[0])), 2, 'invalid subframe layout')
    gpu('order', crafted(2, _channel_bits(_channel_bits(Bits(), 16), 16, nsub_v=[1],
                                          sub=lambda b: b.put(1, 1).put(14, 4))), 2, 'invalid filter order')
    gpu('coding', crafted(1, _channel_bits(Bits(), 16, sub=lambda b: b.put(0, 1).put(0, 1).put(51, 6))), 1,
        'invalid residual coding')
    short = 200
    tail = _channel_bits(_channel_bits(Bits(), 16), 16).put(0, 1).put(7, 3)
    fs = list(frames[:3]) + [_frame(3, tail, last=short)]
    case = make_case('damage_short', 2, 16, 3 * 1024 + short, rate=44100, frame_type=8, seed=61, mc=0)
    gpu('short_decor', fs, 3, 'filtered decorrelation on fewer than 256 samples', data=case.layout(fs)[0])
    mc = make_case('damage_mc', 3, 16, 3 * 1024, rate=44100, frame_type=8, seed=62, mc=0)
    mfs = list(mc.frames()[0])
    bad = Bits().put(1, 1).put(2, 4).put(0, 4).put(1, 1).put(0, 2).put(1, 4)
    mfs[1] = _frame(1, bad)
    gpu('mcdparams', mfs, 1, 'invalid multichannel decorrelation parameters', data=mc.layout(mfs)[0])
    meta = list(frames)
    meta[2] = frame_header(2, metadata=True) + frames[2][8:]
    gpu('metadata', meta, 2, 'frame metadata is not supported')
    contra = list(frames)
    v = info_with(rate=48000)
    contra[2] = frame_header(2, (v['codec'], v['frame_type'], v['samples'], 48000, 16, 2, None)) + frames[2][8:]
    gpu('contradicts', contra, 2, 'frame header contradicts the stream info')
    gap = list(frames)
    gap[2] = frame_header(5) + frames[2][8:]
    gpu('number_gap', gap, 2, 'frame number out of sequence')
    noinfo = list(frames)
    hsize = len(frame_header(0, base.info()))
    noinfo[0] = frame_header(0) + frames[0][hsize:]
    gpu('no_info_first', noinfo, 0, 'the first frame carries no stream info')
    total = head_with(samples=len(base.pcm) + 1)
    out.append(('total', total + body, None, 'the frames hold 4096 samples per channel, the stream info 4097', True))
    return base, out


def long_stream(bits=16, minutes=90, rate=48000, order=14):
    """(case of one full-size frame at the largest filter order, file bytes of that frame repeated for `minutes`,
    repeats): frame 0 carries the stream info, the others reuse the data with their own numbers."""
    ft = 3                                                    # 250 ms frames
    nb = frame_samples(rate, ft)
    reps = max(1, minutes * 60 * rate // nb)
    case = make_case('long%d' % bits, 2, bits, nb, rate=rate, frame_type=ft, kind='tone', seed=77, order=order,
                     filtered=100, nsub=2, cont=1, dmode=3)
    data = encode_data(case.pcm, bits, rate, 2, 77, order=order, filtered=100, nsub=2, cont=1, dmode=3)[0]
    tail = with_crc(data)
    info = case.info()[:2] + (nb * reps,) + case.info()[3:]
    parts = [frame_header(0, info) + tail]
    for i in range(1, reps):
        parts.append(frame_header(i, last=nb if i == reps - 1 else None) + tail)
    if reps == 1:
        parts[0] = frame_header(0, info, last=nb) + tail
    head = b'tBaK' + block('streaminfo', streaminfo(*info)) + b'\0\0\0\0'
    return case, head + b''.join(parts), reps


def long_pcm16(case, reps):
    return np.tile(case.pcm16, (reps, 1))
