"""Seeded writer of MPEG-1/2 audio layer II (MP2) streams for the tests, in NumPy.  The streams are valid layer II
bitstreams with random bit allocations, SCFSI, scalefactors and sample codes: what they decode to is FFmpeg's decode
of them (tests/ref_mp2.py), not anything the writer meant, so randomness is enough.  `assert_coverage` checks that
the cases reach every rate and mode, every joint-stereo bound, every allocation table and quantiser class (grouped and
plain), every SCFSI, the scalefactor range, padding, CRC present and absent, bitrate switches, ancillary bytes,
clipping and silence.

Containers: `TsFile` writes a DVB-style 188-byte transport stream (no HDMV registration) with PES packets that split
frames, optionally starting mid-frame or cut at the end; `mkv_file` a Matroska file with an A_MPEG/L2 track laced
every way tests/mkv_cases.py writes, whole frames to a block or (`mkv_straddling`) cut anywhere.  `damaged_cases` gives broken copies."""
import numpy as np

KBPS = [[0, 32, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, 384],
        [0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160]]
RATES = [44100, 48000, 32000]
STEPS = [3, 5, 7, 9, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 16383, 32767, 65535]
QBITS = [-5, -7, 3, -10, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
_A4 = [0, 2, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
_B4 = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 16]
_C3 = [0, 1, 2, 3, 4, 5, 16]
_D2 = [0, 1, 16]
_E4 = [0, 1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15]
_F3 = [0, 1, 3, 4, 5, 6, 7]
_G4 = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14]
_H2 = [0, 1, 3]
# per table: the quantiser classes of allocations 1.. of each subband (11172-3 B.2a-d, 13818-3 B.1)
TABLES = [[_A4] * 3 + [_B4] * 8 + [_C3] * 12 + [_D2] * 4,
          [_A4] * 3 + [_B4] * 8 + [_C3] * 12 + [_D2] * 7,
          [_E4] * 2 + [_F3] * 6,
          [_E4] * 2 + [_F3] * 10,
          [_G4] * 4 + [_F3] * 7 + [_H2] * 19]
NBAL = {15: 4, 7: 3, 3: 2}


def select_table(kbps, channels, rate, lsf):
    if lsf:
        return 4
    ch = kbps // channels
    if (rate == 48000 and ch >= 56) or 56 <= ch <= 80:
        return 0
    if rate != 48000 and ch >= 96:
        return 1
    if rate != 32000 and ch <= 48:
        return 2
    return 3


class Bits(object):
    def __init__(self):
        self.bits = []

    def put(self, v, n):
        self.bits.extend((int(v) >> (n - 1 - i)) & 1 for i in range(n))

    def __len__(self):
        return len(self.bits)


def crc16(bits, crc=0xFFFF):
    for b in bits:
        top = (crc >> 15) & 1
        crc = (crc << 1) & 0xFFFF
        if top ^ b:
            crc ^= 0x8005
    return crc


def frame_size(lsf, rate_index, bitrate_index, padding):
    return KBPS[lsf][bitrate_index] * 144000 // (RATES[rate_index] >> lsf) + padding


class FrameSpec(object):
    """What one frame was written with (for the coverage checks)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def frame(rng, lsf=0, rate_index=1, bitrate_index=10, mode=0, mode_ext=0, crc=False, padding=0, emphasis=0,
          density=0.6, loud=False, silent=False, ancillary=True):
    """(bytes, FrameSpec): one layer II frame with random allocations (each nonzero with probability `density`, then
    dropped at random until the frame holds them), SCFSI, scalefactors (the loudest indices when `loud`) and codes"""
    channels = 1 if mode == 3 else 2
    rate = RATES[rate_index] >> lsf
    kbps = KBPS[lsf][bitrate_index]
    table = select_table(kbps, channels, rate, lsf)
    classes = TABLES[table]
    sblimit = len(classes)
    bound = min((mode_ext + 1) * 4, sblimit) if mode == 1 else sblimit
    size = frame_size(lsf, rate_index, bitrate_index, padding)
    alloc = np.zeros((2, 32), np.int64)
    if not silent:
        for i in range(sblimit):
            for c in range(channels if i < bound else 1):
                if rng.random() < density:
                    alloc[c, i] = rng.integers(1, len(classes[i]) + 1)
            if i >= bound:
                alloc[1, i] = alloc[0, i]
    scfsi = rng.integers(0, 4, (2, 32))
    sf = rng.integers(0, 4 if loud else 63, (2, 32, 3))

    def need():
        n = 32 + 16 * crc
        for i in range(sblimit):
            nb = NBAL[len(classes[i])]
            n += nb * (channels if i < bound else 1)
        for i in range(sblimit):
            for c in range(channels):
                if alloc[c, i]:
                    n += 2 + 6 * {0: 3, 1: 2, 2: 1, 3: 2}[int(scfsi[c, i])]
                    if c == 0 or i < bound:
                        q = classes[i][alloc[c, i] - 1]
                        n += 12 * (-QBITS[q] if QBITS[q] < 0 else 3 * QBITS[q])
        return n

    while need() > size * 8:
        nz = np.argwhere(alloc[:, :sblimit] > 0)
        c, i = nz[rng.integers(len(nz))]
        if i >= bound:
            alloc[:, i] = 0
        else:
            alloc[c, i] = 0
    h = (0xFFF << 20) | ((0 if lsf else 1) << 19) | (2 << 17) | ((0 if crc else 1) << 16) | (bitrate_index << 12) | \
        (rate_index << 10) | (padding << 9) | (mode << 6) | (mode_ext << 4) | emphasis
    head = Bits()
    head.put(h, 32)
    side = Bits()
    for i in range(sblimit):
        nb = NBAL[len(classes[i])]
        for c in range(channels if i < bound else 1):
            side.put(alloc[c, i], nb)
    for i in range(sblimit):
        for c in range(channels):
            if alloc[c, i]:
                side.put(scfsi[c, i], 2)
    body = Bits()
    for i in range(sblimit):
        for c in range(channels):
            if alloc[c, i]:
                s = scfsi[c, i]
                for k in {0: (0, 1, 2), 1: (0, 2), 2: (0,), 3: (0, 2)}[int(s)]:
                    body.put(sf[c, i, k], 6)
    codes = []
    for part in range(3):
        for g in range(4):
            for i in range(sblimit):
                for c in range(channels if i < bound else 1):
                    if alloc[c, i]:
                        q = classes[i][alloc[c, i] - 1]
                        if QBITS[q] < 0:
                            body.put(rng.integers(0, STEPS[q] ** 3), -QBITS[q])
                        else:
                            for _ in range(3):
                                body.put(rng.integers(0, STEPS[q]), QBITS[q])
                        codes.append(q)
    bits = head.bits[:]
    if crc:
        bits += [(crc16(head.bits[16:] + side.bits) >> (15 - i)) & 1 for i in range(16)]
    bits += side.bits + body.bits
    assert len(bits) <= size * 8
    data = np.packbits(np.array(bits + [0] * (-len(bits) % 8), np.uint8)).tobytes()
    tail = size - len(data)
    fill = rng.integers(0, 256, tail, dtype=np.uint8).tobytes() if ancillary else bytes(tail)
    spec = FrameSpec(lsf=lsf, rate=rate, mode=mode, mode_ext=mode_ext, bound=bound, table=table, crc=crc,
                     padding=padding, bitrate_index=bitrate_index, classes=set(codes),
                     scfsi={int(scfsi[c, i]) for c in range(channels) for i in range(sblimit) if alloc[c, i]},
                     sf={int(sf[c, i, k]) for c in range(channels) for i in range(sblimit) if alloc[c, i]
                         for k in range(3)},
                     ancillary=tail if ancillary else 0, loud=loud, silent=silent)
    return data + fill, spec


class Case(object):
    def __init__(self, name, frames, specs):
        self.name, self.frames, self.specs = name, frames, specs
        s = specs[0]
        self.channels = 1 if s.mode == 3 else 2
        self.rate = s.rate

    @property
    def data(self):
        return b''.join(self.frames)

    def __repr__(self):
        return self.name


def stream(name, seed, n, **kw):
    """n frames; keyword values that are lists are cycled frame by frame (bitrate switches, modes, ...)"""
    rng = np.random.default_rng([seed])
    frames, specs = [], []
    for k in range(n):
        args = {a: (v[k % len(v)] if isinstance(v, list) else v) for a, v in kw.items()}
        d, s = frame(rng, **args)
        frames.append(d)
        specs.append(s)
    return Case(name, frames, specs)


def all_cases():
    cases = []
    seed = 100
    for lsf in (0, 1):
        for ri in range(3):
            for mode in range(4):
                exts = range(4) if mode == 1 else [0]
                for ext in exts:
                    seed += 1
                    # bitrates that reach every table: 48 kHz and 44.1 / 32 kHz at per-channel rates on both sides
                    brs = [4, 7, 10, 13] if mode != 3 else [1, 4, 8, 11]
                    cases.append(stream('mp2_{0}_{1}_m{2}e{3}'.format('lsf' if lsf else 'mpeg1', RATES[ri] >> lsf,
                                                                       mode, ext),
                                        seed, 6, lsf=lsf, rate_index=ri, bitrate_index=brs, mode=mode, mode_ext=ext,
                                        crc=[False, True], padding=[0, 1, 0], emphasis=[0, 1, 3]))
    # every bitrate at every rate, mono and stereo: the bitrate switches frame by frame
    for ri in range(3):
        for mode in (0, 3):
            cases.append(stream('mp2_bitrates_{0}_{1}'.format(RATES[ri], 'mono' if mode == 3 else 'stereo'),
                                20 + ri * 4 + mode, 14, rate_index=ri, mode=mode, bitrate_index=list(range(1, 15))))
    cases.append(stream('mp2_dense', 9, 8, bitrate_index=14, mode=[0, 2], density=1.0))
    cases.append(stream('mp2_loud_clips', 10, 6, bitrate_index=14, mode=0, density=1.0, loud=True))
    cases.append(stream('mp2_silence', 11, 5, mode=1, silent=[True, True, False], mode_ext=2))
    cases.append(stream('mp2_no_ancillary', 12, 4, ancillary=False, crc=True))
    return cases


def assert_coverage(cases):
    specs = [s for c in cases for s in c.specs]
    assert {(s.lsf, s.rate, s.mode) for s in specs} == {(l, r >> l, m) for l in (0, 1) for r in RATES
                                                        for m in range(4)}
    assert {(s.bound, s.table) for s in specs if s.mode == 1} >= {(4, 0), (8, 0), (12, 0), (16, 0), (8, 2), (12, 3),
                                                                 (4, 4), (16, 4)}
    assert {s.table for s in specs} == set(range(5))
    assert set().union(*(s.classes for s in specs)) == set(range(17))
    assert set().union(*(s.scfsi for s in specs)) == {0, 1, 2, 3}
    used = set().union(*(s.sf for s in specs))
    assert {0, 1, 2, 3, 62} <= used and len(used) >= 60
    assert {s.padding for s in specs} == {0, 1} and {s.crc for s in specs} == {False, True}
    assert any(len({s.bitrate_index for s in c.specs}) > 1 for c in cases)
    assert any(s.ancillary for s in specs) and any(s.loud for s in specs) and any(s.silent for s in specs)


# ---- containers ----

def mkv_file(name, case, pieces=None):
    """A Matroska file with the case as an A_MPEG/L2 track, blocks laced by LAYOUT in turn.  pieces: the byte lengths
    the stream is cut into, one per Matroska frame (default: one MP2 frame each), so that frames straddle blocks."""
    from tests import mkv_cases as mc
    from tests import mkv_tta_cases as mtc
    spec = mc.TrackSpec('audio', 'A_MPEG/L2', b'', True, 'mp2', 'eng', 0, case.rate, case.channels, None,
                        pcm=np.zeros((1, case.channels), np.int64), pcm_bits=16)
    data = case.data
    if pieces is None:
        pieces = [len(f) for f in case.frames]
    at = 0
    for k, n in enumerate(pieces):
        spec.frames.append((data[at:at + n], k * 1152, None))
        at += n
    assert at == len(data)
    a = mc._timed(spec, 1000.0 / case.rate)
    ab = mc._blocks_for(0, a, lambda j: mtc.LAYOUT[j % len(mtc.LAYOUT)][:3] + (None,))
    ts, clusters = mc.arrange([a], 2000, [ab])
    return mc.build(name, [a], clusters, ts)


class TsFile(object):
    """A DVB-style transport stream (188-byte packets, no HDMV registration) carrying `es` as MPEG audio PES packets
    (stream id 0xC0) of random lengths that split frames; `data` the file, `es` the elementary stream in it."""

    def __init__(self, name, es, rng, stream_type=0x03, cut_end=0):
        from tests import ts_cases as tsc
        self.name, self.es = name, es
        s = tsc.Stream(0x101, stream_type, 'mp2')
        at = 0
        payloads = []
        while at < len(es):
            n = int(rng.integers(300, 4000))
            payloads.append(es[at:at + n])
            s.pes.append(tsc.pes(0xC0, es[at:at + n], 9000 + at))
            s.pes_frames.append(None)
            at += n
        t = tsc.TsCase(name, 188, False, [s], rng)
        self.data = t.data[:len(t.data) - cut_end * 188] if cut_end else t.data
        # the elementary stream the file holds: each PES's payload up to the packets that survive the cut (14 bytes
        # of PES header first)
        kept = [0] * len(payloads)
        for off, pid, tag, n, _ in t.packets:
            if tag is not None and tag[0] == 0x101 and off + 188 <= len(self.data):
                kept[tag[1]] += n
        self.es = b''.join(p[:max(0, k - 14)] for p, k in zip(payloads, kept))

    def write(self, directory):
        path = str(directory / (self.name + '.ts'))
        with open(path, 'wb') as f:
            f.write(self.data)
        return path


def ts_files(cases=None):
    """[(TsFile, Case)]: whole streams, one starting mid-frame (its first 300 bytes gone), one whose file ends
    mid-frame, and one of stream type 0x04"""
    by = {c.name: c for c in (cases or all_cases())}
    out = []
    rng = np.random.default_rng([77])
    for k, name in enumerate(('mp2_mpeg1_48000_m1e1', 'mp2_lsf_22050_m3e0', 'mp2_mpeg1_44100_m2e0', 'mp2_dense')):
        c = by[name]
        out.append((TsFile('ts_' + name, c.data, rng, stream_type=0x03 if k % 2 == 0 else 0x04), c))
    c = by['mp2_bitrates_48000_stereo']
    out.append((TsFile('ts_mid_frame_start', c.data[300:], rng), c))
    out.append((TsFile('ts_cut_end', c.data, rng, cut_end=3), c))
    return out


def mkv_files(cases=None):
    """[(MkvCase, Case)]: one MP2 frame per Matroska frame, and frames cut across blocks"""
    by = {c.name: c for c in (cases or all_cases())}
    out = []
    for name in ('mp2_mpeg1_32000_m0e0', 'mp2_lsf_24000_m1e3', 'mp2_loud_clips'):
        out.append((mkv_file('mka_' + name, by[name]), by[name]))
    c = by['mp2_bitrates_44100_stereo']
    sizes = [len(f) for f in c.frames]
    out.append((mkv_file('mka_mp2_three_per_block', c, [sum(sizes[k:k + 3]) for k in range(0, len(sizes), 3)]), c))
    return out


def mkv_straddling(cases=None):
    """A Matroska track whose blocks cut the stream anywhere, so frames straddle blocks: FFmpeg decodes each block as
    a packet (and refuses those that do not start with a header); the decoder refuses the track"""
    c = {x.name: x for x in (cases or all_cases())}['mp2_bitrates_44100_stereo']
    rng = np.random.default_rng([78])
    pieces = []
    left = len(c.data)
    while left:
        n = min(left, int(rng.integers(100, 1500)))
        pieces.append(n)
        left -= n
    return mkv_file('mka_mp2_straddling', c, pieces), c


def long_stream(minutes=90.0, distinct=120, seed=5):
    """(frames, stream bytes): 48 kHz stereo at 192 kbit/s, `distinct` random frames cycled to `minutes`"""
    c = stream('mp2_long', seed, distinct, bitrate_index=10, mode=[0, 1, 2], mode_ext=[0, 3], crc=[False, True])
    n = int(minutes * 60 * 48000 // 1152)
    frames = [c.frames[k % distinct] for k in range(n)]
    return frames, b''.join(frames)


# ---- damaged copies ----

def damaged_cases():
    """[(name, stream bytes, frame, offset, regex)]: copies of one stream that the decoder refuses, naming the frame
    and its byte offset in the stream"""
    base = stream('mp2_damage_base', 90, 6, crc=True, bitrate_index=[10, 12])
    offs = np.cumsum([0] + [len(f) for f in base.frames])
    out = []

    def frames_with(k, new):
        fr = list(base.frames)
        fr[k] = new
        return b''.join(fr)

    f2 = bytearray(base.frames[2])
    f2[1] &= 0x0F                                              # sync broken: 0xFF 0x0? no longer a header
    out.append(('broken_sync', frames_with(2, bytes(f2)), 2, int(offs[2]), 'no frame sync'))
    f3 = bytearray(base.frames[3])
    f3[6] ^= 0x40                                              # an allocation bit: the CRC disagrees
    out.append(('crc', frames_with(3, bytes(f3)), 3, int(offs[3]), 'CRC-16 mismatch'))
    l3 = stream('l3', 91, 1, crc=True)
    f1 = bytearray(l3.frames[0])
    f1[1] = (f1[1] & ~0x06) | 0x02                             # layer III
    out.append(('layer_change', frames_with(1, bytes(f1)), 1, int(offs[1]), r'layer III \(MP3\)'))
    other = stream('r', 92, 1, rate_index=0, crc=True, bitrate_index=10)
    out.append(('rate_change', frames_with(4, other.frames[0]), 4, int(offs[4]), 'sample rate changes mid-stream'))
    mono = stream('m', 93, 1, mode=3, crc=True, bitrate_index=10)
    out.append(('channel_change', frames_with(5, mono.frames[0]), 5, int(offs[5]), 'channel count changes'))
    f4 = bytearray(base.frames[4])
    f4[2] = (f4[2] & 0x0F) | 0x00                              # free format
    out.append(('free_format', frames_with(4, bytes(f4)), 4, int(offs[4]), 'free-format bitrate'))
    f5 = bytearray(base.frames[5])
    f5[3] = (f5[3] & ~3) | 2                                   # reserved emphasis
    out.append(('reserved_emphasis', frames_with(5, bytes(f5)), 5, int(offs[5]), 'reserved emphasis'))
    # the last frame claims the lowest bitrate and is cut to that length: its samples run past its end
    f5 = bytearray(base.frames[5])
    f5[1] |= 1                                                 # no CRC, so the bit count is what refuses it
    f5[2] = (f5[2] & 0x0D) | 0x10
    short = bytes(f5[:frame_size(0, 1, 1, 0)])
    out.append(('samples_past_end', b''.join(base.frames[:5]) + short, 5, int(offs[5]), 'run past its end'))
    return base, out
