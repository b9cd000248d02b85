"""A seeded WavPack writer for the tests: lossless integer streams whose PCM is known, and damaged copies.

The writer mirrors the decoder's arithmetic to find residuals: each decorrelation pass runs backwards, with the same
wrap-around, weight adaptation and history as FFmpeg's `wavpack` decoder, then the residuals are coded with the adaptive
Golomb code (three medians per channel, zero runs, the held one / zero bit, large-value escapes).  Every block carries
its own state in its metadata sub-blocks (terms, weights, sample history, medians), as WavPack's encoder writes it.
Every case records which coding features it used, and `assert_coverage` checks that the cases together use every one
the decoder handles (see FEATURES).

A case's `pcm` is (frames, channels) int64 at the container width (16 or 24 bits) in FFmpeg's channel order (blocks in
order within a frame); `pcm16` the int16 the loader keeps (the top 16 bits)."""
import math
import struct

import numpy as np

M32 = 0xFFFFFFFF
EXP2 = [int(math.floor(256 * 2 ** (i / 256) + 0.5)) - 256 for i in range(256)]
RATES = (6000, 8000, 9600, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 64000, 88200, 96000, 192000)
MONO, HYBRID, JOINT, CROSS, FLOAT, INITIAL, FINAL, FALSE_STEREO, DSD = (0x4, 0x8, 0x10, 0x20, 0x80, 0x800, 0x1000,
                                                                       0x40000000, 0x80000000)
ID_TERMS, ID_WEIGHTS, ID_SAMPLES, ID_ENTROPY, ID_INT32, ID_BITS, ID_WVX, ID_CHANNELS = 2, 3, 4, 5, 9, 10, 12, 13
ID_RIFF_HEADER, ID_RIFF_TRAILER, ID_CONFIG, ID_MD5, ID_RATE = 0x21, 0x22, 0x25, 0x26, 0x27
TERMS = [1, 2, 3, 4, 5, 6, 7, 8, 17, 18, -1, -2, -3]
FEATURES = {'channels_1', 'channels_2', 'channels_3', 'channels_6', 'channels_8', 'bits_16', 'bits_20', 'bits_24',
            'table_rate', 'custom_rate', 'joint', 'false_stereo', 'mono_in_multichannel', 'shift', 'int32_zeros',
            'int32_ones', 'int32_dups', 'riff_header', 'riff_trailer', 'config', 'md5', 'unknown_subblock',
            'odd_subblock', 'large_subblock', 'zero_run', 'holding_one', 'escape', 'apetag', 'id3v1'} | \
           {'term_%d' % t for t in TERMS} | {'delta_%d' % d for d in range(8)} | {'terms_%d' % n for n in range(17)}


def i32(v):
    v &= M32
    return v - (1 << 32) if v >> 31 else v


def sx(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def wp_exp2(code):
    code = sx(code, 16)
    neg = code < 0
    if neg:
        code = -code
    res = EXP2[code & 0xFF] | 0x100
    code >>= 8
    res = res << (code - 9) if code > 9 else res >> (9 - code)
    return -res if neg else res


def restore_weight(b):
    w = sx(b, 8) * 8
    return w + ((w + 64) >> 7) if w > 0 else w


def apply_weight(w, a, wide):
    if wide:
        return i32((w * a + 512) >> 10)
    return i32(w * a + 512) >> 10


def clip_update(w, delta, s, x):
    if s and x:
        if (s ^ x) < 0:
            return max(w - delta, -1024)
        return min(w + delta, 1024)
    return w


class Bits(object):
    """LSB-first bit writer"""

    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, n, v):
        if n:
            self.acc |= (v & ((1 << n) - 1)) << self.n
            self.n += n

    def ones(self, n):
        self.put(n, (1 << n) - 1)

    def bytes(self):
        return self.acc.to_bytes((self.n + 7) // 8, 'little')


def _unary_escape(bits, k):
    """k as a zero-run count or escape: k < 2 as k ones and a zero, else bit length ones, a zero, the low bits"""
    if k < 2:
        bits.ones(k)
        bits.put(1, 0)
    else:
        bl = k.bit_length()
        assert bl < 32
        bits.ones(bl)
        bits.put(1, 0)
        bits.put(bl - 1, k)


def _get_med(m, n):
    return (m[n] >> 4) + 1


def _dec_med(m, n):
    m[n] = i32(m[n] - ((m[n] + (128 >> n) - 2) // (128 >> n)) * 2)


def _inc_med(m, n):
    m[n] = i32(m[n] + ((m[n] + (128 >> n)) // (128 >> n)) * 5)


class Entropy(object):
    """The adaptive Golomb coder of one block, mirroring the decoder's state call for call."""

    def __init__(self, meds, used):
        self.med = [list(meds[0]), list(meds[1])]
        self.used = used

    def _split(self, ch, v):
        """(t, low, add) for value v on channel ch, updating the medians as the decoder will"""
        m = self.med[ch]
        r = v if v >= 0 else ~v
        g0, g1, g2 = _get_med(m, 0), _get_med(m, 1), _get_med(m, 2)
        if r < g0:
            _dec_med(m, 0)
            return 0, 0, g0 - 1
        if r - g0 < g1:
            _inc_med(m, 0)
            _dec_med(m, 1)
            return 1, g0, g1 - 1
        t = 2 + (r - g0 - g1) // g2
        _inc_med(m, 0)
        _inc_med(m, 1)
        (_dec_med if t == 2 else _inc_med)(m, 2)
        return t, g0 + g1 + (t - 2) * g2, g2 - 1

    def _t_of(self, ch, v):
        m = self.med[ch]
        r = v if v >= 0 else ~v
        g0, g1, g2 = _get_med(m, 0), _get_med(m, 1), _get_med(m, 2)
        if r < g0:
            return 0
        if r - g0 < g1:
            return 1
        return 2 + (r - g0 - g1) // g2

    def code(self, values, chans):
        """Code values[i] of channel chans[i] in decode order; returns the bitstream bytes."""
        b = Bits()
        one = zero = 0
        zeroes = 0
        n = len(values)
        i = 0
        while i < n:
            v, ch = values[i], chans[i]
            if self.med[0][0] < 2 and self.med[1][0] < 2 and not zero and not one:
                if zeroes:
                    zeroes -= 1
                    if zeroes:
                        assert v == 0
                        i += 1
                        continue
                else:
                    k = 0
                    while i + k < n and values[i + k] == 0:
                        k += 1
                    _unary_escape(b, k)
                    zeroes = k
                    if k:
                        self.used.add('zero_run')
                        self.med = [[0, 0, 0], [0, 0, 0]]
                        i += 1
                        continue
            if zero:
                assert self._t_of(ch, v) == 0
                zero = 0
                t, low, add = self._split(ch, v)
            else:
                t, low, add = self._split(ch, v)
                nxt = 1 if i + 1 < n and self._t_of(chans[i + 1], values[i + 1]) > 0 else 0
                u = 2 * (t - 1) + nxt if one else 2 * t + nxt
                if one:
                    self.used.add('holding_one')
                if u < 16:
                    b.ones(u)
                    b.put(1, 0)
                else:
                    self.used.add('escape')
                    b.ones(16)
                    b.put(1, 0)
                    _unary_escape(b, u - 16)
                one, zero = nxt, 1 - nxt
            r = v if v >= 0 else ~v
            code = r - low
            assert 0 <= code <= add < 0x2000000, (code, add)
            if add:
                p = add.bit_length() - 1
                e = (1 << (p + 1)) - add - 1
                if code < e:
                    b.put(p, code)
                else:
                    b.put(p, (code + e) >> 1)
                    b.put(1, (code + e) & 1)
            b.put(1, 1 if v < 0 else 0)
            i += 1
        b.put(1, 0)                                   # at least one bit after the last sign bit
        return b.bytes()


class Term(object):
    def __init__(self, value, delta, wa, wb, ha, hb):
        self.value, self.delta = value, delta
        self.wa, self.wb = restore_weight(wa), restore_weight(wb)
        self.wa_byte, self.wb_byte = wa, wb
        self.ha = [wp_exp2(c) for c in ha] + [0] * (8 - len(ha))
        self.hb = [wp_exp2(c) for c in hb] + [0] * (8 - len(hb))
        self.ha_codes, self.hb_codes = ha, hb


def _history_len(value):
    return 2 if value > 8 else (1 if value < 0 else value)


def residuals(x, terms, stereo, wide):
    """The residuals (decode order, interleaved when stereo) for which the decoder's passes give back x (n, 1 or 2)."""
    n = len(x)
    out = []
    pos = 0
    for s in range(n):
        if stereo:
            L, R = int(x[s, 0]), int(x[s, 1])
            for tm in reversed(terms):
                t = tm.value
                if t > 0:
                    if t > 8:
                        a0, a1, b0, b1 = tm.ha[0], tm.ha[1], tm.hb[0], tm.hb[1]
                        A = i32(2 * a0 - a1) if t & 1 else i32(3 * a0 - a1) >> 1
                        B = i32(2 * b0 - b1) if t & 1 else i32(3 * b0 - b1) >> 1
                        tm.ha[1], tm.hb[1] = a0, b0
                        j = 0
                    else:
                        A, B = tm.ha[pos], tm.hb[pos]
                        j = (pos + t) & 7
                    Lin = i32(L - apply_weight(tm.wa, A, wide))
                    Rin = i32(R - apply_weight(tm.wb, B, wide))
                    if A and Lin:
                        tm.wa += tm.delta if (Lin ^ A) >= 0 else -tm.delta
                    if B and Rin:
                        tm.wb += tm.delta if (Rin ^ B) >= 0 else -tm.delta
                    tm.ha[j], tm.hb[j] = L, R
                    L, R = Lin, Rin
                elif t == -1:
                    a0 = tm.ha[0]
                    Lin = i32(L - apply_weight(tm.wa, a0, wide))
                    tm.wa = clip_update(tm.wa, tm.delta, a0, Lin)
                    Rin = i32(R - apply_weight(tm.wb, L, wide))
                    tm.wb = clip_update(tm.wb, tm.delta, L, Rin)
                    tm.ha[0] = R
                    L, R = Lin, Rin
                else:
                    b0 = tm.hb[0]
                    Rin = i32(R - apply_weight(tm.wb, b0, wide))
                    tm.wb = clip_update(tm.wb, tm.delta, b0, Rin)
                    other = R
                    if t == -3:
                        other = tm.ha[0]
                        tm.ha[0] = R
                    Lin = i32(L - apply_weight(tm.wa, other, wide))
                    tm.wa = clip_update(tm.wa, tm.delta, other, Lin)
                    tm.hb[0] = L
                    L, R = Lin, Rin
            out += [L, R]
        else:
            S = int(x[s, 0])
            for tm in reversed(terms):
                t = tm.value
                if t > 8:
                    a0, a1 = tm.ha[0], tm.ha[1]
                    A = i32(2 * a0 - a1) if t & 1 else i32(3 * a0 - a1) >> 1
                    tm.ha[1] = a0
                    j = 0
                else:
                    A = tm.ha[pos]
                    j = (pos + t) & 7
                T = i32(S - apply_weight(tm.wa, A, wide))
                if A and T:
                    tm.wa += tm.delta if (T ^ A) >= 0 else -tm.delta
                tm.ha[j] = S
                S = T
            out.append(S)
        pos = (pos + 1) & 7
    return out


def subblock(sid, payload):
    """A metadata sub-block: id (odd / long flags set as needed), size in words, payload padded to even"""
    odd = len(payload) & 1
    words = (len(payload) + 1) // 2
    flags = (0x40 if odd else 0) | (0x80 if words > 255 else 0)
    head = struct.pack('<BB', sid | flags, words & 0xFF) + (struct.pack('<H', words >> 8) if words > 255 else b'')
    return head + payload + (b'\0' if odd else b'')


def store(x, int32, shift, width):
    """FFmpeg's sample for stored value x: ID_INT32_INFO (kind, bits), then the header's shift, wrapped to width bits"""
    kind, bits = int32 or (None, 0)
    a = o = 0
    if kind == 'ones':
        a = o = 1
    elif kind == 'dups':
        a = 1
    bit = (x & a) | o
    return sx((((x + bit) << bits) - bit) << shift, width)


class Stream(object):
    """What one case's blocks share"""

    def __init__(self, bytes_per_sample=2, shift=0, rate=48000, int32=None, joint=False, version=0x407):
        self.bps, self.shift, self.rate, self.int32, self.joint, self.version = (bytes_per_sample, shift, rate, int32,
                                                                                 joint, version)


def encode_block(x, st, rng, used, nterms, stereo_mode, extra=(), history=True, meds=None):
    """One block of samples x (n, 1) or (n, 2) stored values: (flags, crc, sub-block bytes).  stereo_mode is 'mono',
    'stereo' or 'false' (one channel coded, the other equal to it)."""
    n = len(x)
    stereo_in = stereo_mode == 'stereo'
    wide = st.bps == 3
    flags = (st.bps - 1) | (st.shift << 13)
    if stereo_mode == 'mono':
        flags |= MONO
    elif stereo_mode == 'false':
        flags |= FALSE_STEREO
    rate_index = RATES.index(st.rate) if st.rate in RATES else 15
    flags |= rate_index << 23
    # joint stereo: the passes see (L - R, R + ((L - R) >> 1)) of the stored pair
    v = np.asarray(x, np.int64)
    if stereo_in and st.joint:
        flags |= JOINT
        lp = [i32(int(a) - int(b)) for a, b in v]
        v = np.array([[lp[k], i32(int(v[k, 1]) + (lp[k] >> 1))] for k in range(n)], np.int64) if n else v
    if stereo_in:
        pool = TERMS
    else:
        pool = TERMS[:10]
        v = v[:, :1]
    terms = []
    for _ in range(nterms):
        value = int(rng.choice(pool))
        delta = int(rng.integers(0, 8))
        hl = _history_len(value)
        ha = [int(rng.integers(0, 0x0900)) * (1 if rng.random() < 0.7 else -1) & 0xFFFF for _ in range(hl)]
        hb = [int(rng.integers(0, 0x0900)) * (1 if rng.random() < 0.7 else -1) & 0xFFFF for _ in range(hl)]
        if not history:
            ha = hb = []
        terms.append(Term(value, delta, int(rng.integers(-40, 120)) & 0xFF, int(rng.integers(-40, 120)) & 0xFF,
                          ha, hb if (stereo_in or value < 0) else []))
        used.add('term_%d' % value)
        used.add('delta_%d' % delta)
        if value < 0:
            flags |= CROSS
    used.add('terms_%d' % nterms)
    # sub-blocks, in the decoder's storage order (the last pass applied first)
    tbytes = bytes(((t.value + 5) & 0x1F) | (t.delta << 5) for t in reversed(terms))
    wbytes = b''.join(bytes([t.wa_byte, t.wb_byte] if stereo_in else [t.wa_byte]) for t in reversed(terms))
    hbytes = b''
    if history:
        for t in reversed(terms):
            if t.value > 8:
                codes = t.ha_codes + (t.hb_codes if stereo_in else [])
            elif t.value < 0:
                codes = [t.ha_codes[0], t.hb_codes[0]]
            else:
                codes = [c for j in range(t.value) for c in ([t.ha_codes[j], t.hb_codes[j]] if stereo_in
                                                             else [t.ha_codes[j]])]
            hbytes += b''.join(struct.pack('<H', c) for c in codes)
    else:
        for t in terms:
            t.ha, t.hb = [0] * 8, [0] * 8
    if meds is None:
        meds = [[int(rng.integers(0, 0x0C00)) for _ in range(3)] for _ in range(2)]
    ebytes = b''.join(struct.pack('<H', meds[c][i]) for c in range(1 + stereo_in) for i in range(3))
    ent = Entropy([[wp_exp2(c) for c in meds[0]], [wp_exp2(c) for c in meds[1]] if stereo_in else [0, 0, 0]], used)
    res = residuals(v, terms, stereo_in, wide)
    chans = [k % 2 for k in range(len(res))] if stereo_in else [0] * len(res)
    bits = ent.code(res, chans)
    # the block CRC over the stored values
    crc = M32
    xs = np.asarray(x, np.int64)
    for k in range(n):
        if stereo_in:
            crc = ((crc * 3 + int(xs[k, 0])) * 3 + int(xs[k, 1])) & M32
        else:
            crc = (crc * 3 + int(xs[k, 0])) & M32
    body = b''.join(extra)
    body += subblock(ID_TERMS, tbytes) + subblock(ID_WEIGHTS, wbytes) + subblock(ID_SAMPLES, hbytes)
    body += subblock(ID_ENTROPY, ebytes)
    if st.int32:
        kind, b = st.int32
        body += subblock(ID_INT32, bytes([0, b if kind == 'zeros' else 0, b if kind == 'ones' else 0,
                                          b if kind == 'dups' else 0]))
        used.add('int32_' + kind)
    if rate_index == 15:
        body += subblock(ID_RATE, struct.pack('<I', st.rate)[:3])
    body += subblock(ID_BITS, bits)
    return flags, crc, body


class WvCase(object):
    """A WavPack stream: frames of blocks [(flags, crc, body)], one block_samples per frame."""

    def __init__(self, name, st, channels, frames, counts, pcm, used, layout, chmask=0):
        self.name, self.st, self.channels, self.frames, self.counts = name, st, channels, frames, counts
        self.pcm, self.used, self.layout, self.chmask = pcm, used, layout, chmask
        self.rate, self.bits = st.rate, 8 * st.bps
        self.pcm16 = to16(pcm, self.bits)
        self.tail = b''
        self.total = sum(counts)

    def wv(self, total=None, version=None):
        """The .wv file: every block behind its 32-byte header"""
        out = []
        at = 0
        total = self.total if total is None else total
        for blocks, count in zip(self.frames, self.counts):
            for flags, crc, body in blocks:
                out.append(header(len(body), version or self.st.version, total, at, count, flags, crc) + body)
            at += count
        return b''.join(out) + self.tail

    def mkv_frames(self):
        """The A_WAVPACK4 frames: block_samples, then per block flags, crc (and size unless the only block), payload"""
        out = []
        for blocks, count in zip(self.frames, self.counts):
            f = struct.pack('<I', count)
            for flags, crc, body in blocks:
                single = (flags & (INITIAL | FINAL)) == (INITIAL | FINAL)
                f += struct.pack('<II', flags, crc) + (b'' if single else struct.pack('<I', len(body))) + body
            out.append(f)
        return out


def header(size, version, total, index, count, flags, crc):
    return b'wvpk' + struct.pack('<IHBBIIIII', size + 24, version, 0, 0, total & M32, index, count, flags, crc)


def to16(pcm, bits):
    pcm = np.asarray(pcm, np.int64)
    return (pcm >> (bits - 16)).astype(np.int16) if bits > 16 else pcm.astype(np.int16)


LAYOUTS = {1: ['mono'], 2: ['stereo'], 3: ['stereo', 'mono'], 6: ['stereo', 'mono', 'mono', 'stereo'],
           8: ['stereo', 'mono', 'mono', 'stereo', 'stereo']}
MASKS = {3: 0x7, 6: 0x3F, 8: 0x63F}


def signal(rng, n, channels, amp, silence=False, spike=False):
    """Stored values: sines and noise per channel, with silences and a spike when asked"""
    t = np.arange(n)
    out = np.zeros((n, channels), np.int64)
    for c in range(channels):
        f = rng.uniform(0.003, 0.05)
        s = 0.6 * np.sin(2 * np.pi * f * t + c) + 0.25 * rng.standard_normal(n) * rng.uniform(0.05, 1)
        out[:, c] = np.clip(np.round(s * amp * rng.uniform(0.2, 0.9)), -amp, amp - 1).astype(np.int64)
    if silence and n > 40:
        a = int(rng.integers(0, n // 2))
        out[a:a + n // 3] = 0
    if spike and n > 10:
        out[n // 2, 0] = amp - 1
        out[n // 2 + 1, 0] = -amp
    return out


def make_case(name, seed, channels=2, bps=2, shift=0, rate=48000, int32=None, joint=False, counts=(700, 700, 300),
              nterms=None, layout=None, false_stereo=False, extra_first=(), extra_last=(), silence=True, spike=True,
              version=0x407, amp_bits=None, meds=None, x=None):
    """A case of `counts` frames: the stored values are x (frames, channels) when given, else a seeded signal."""
    rng = np.random.default_rng(seed)
    st = Stream(bps, shift, rate, int32, joint, version)
    used = set()
    layout = layout or LAYOUTS[channels]
    width = 8 * bps
    eff = width - shift - (int32[1] if int32 else 0)
    amp = 1 << ((amp_bits or eff) - 1)
    n = sum(counts)
    x = signal(rng, n, channels, amp, silence, spike) if x is None else np.asarray(x, np.int64)
    if false_stereo:
        x[:, 1] = x[:, 0]
    frames = []
    at = 0
    for fi, count in enumerate(counts):
        blocks = []
        ch = 0
        for bi, mode in enumerate(layout):
            w = 1 if mode == 'mono' else 2
            xb = x[at:at + count, ch:ch + w]
            extra = []
            if bi == 0 and fi == 0:
                extra += list(extra_first)
            if bi == 0 and len(layout) > 1:
                extra.append(subblock(ID_CHANNELS, bytes([channels]) + MASKS[channels].to_bytes(
                    1 if MASKS[channels] < 256 else 2, 'little')))
            if bi == len(layout) - 1 and fi == len(counts) - 1:
                extra += list(extra_last)
            k = nterms if nterms is not None else int(rng.integers(0, 17))
            if isinstance(nterms, (list, tuple)):
                k = nterms[(fi * len(layout) + bi) % len(nterms)]
            smode = mode
            if mode == 'stereo' and false_stereo:
                smode = 'false'
                used.add('false_stereo')
            if smode != 'stereo':
                k = max(k, 1)                         # FFmpeg decodes a mono block without terms as silence
            flags, crc, body = encode_block(xb, st, rng, used, k, smode, extra, meds=meds)
            if bi == 0:
                flags |= INITIAL
            if bi == len(layout) - 1:
                flags |= FINAL
            blocks.append((flags, crc, body))
            ch += w
        frames.append(blocks)
        at += count
    pcm = np.vectorize(lambda v: store(int(v), int32, shift, width), otypes=[np.int64])(x) if n else x
    used.add('channels_%d' % channels)
    used.add('bits_%d' % (width - shift if shift and bps == 3 else width))
    used.add('custom_rate' if rate not in RATES else 'table_rate')
    if joint and 'stereo' in layout and not false_stereo:
        used.add('joint')
    if 'mono' in layout and len(layout) > 1:
        used.add('mono_in_multichannel')
    if shift:
        used.add('shift')
    return WvCase(name, st, channels, frames, list(counts), pcm, used, layout, MASKS.get(channels, 0))


def riff_header(channels, rate, bps, frames, pad=0):
    data = frames * channels * bps
    fmt = struct.pack('<HHIIHH', 1, channels, rate, rate * channels * bps, channels * bps, 8 * bps)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', len(fmt)) + fmt
    if pad:
        body += b'LIST' + struct.pack('<I', pad) + bytes((i * 7) & 0xFF for i in range(pad))
    return b'RIFF' + struct.pack('<I', len(body) + 8 + data) + body + b'data' + struct.pack('<I', data)


def apetag():
    """An APEv2 tag with a header, one item and a footer"""
    item = struct.pack('<II', 5, 0) + b'Title\0' + b'Sushi'
    size = len(item) + 32

    def part(flags):
        return b'APETAGEX' + struct.pack('<IIII', 2000, size, 1, flags) + bytes(8)
    return part(0xA0000000) + item + part(0x80000000)


def id3v1():
    return b'TAG' + b'Sushi'.ljust(30, b'\0') + bytes(30 + 30 + 4 + 30) + b'\xff'


def all_cases():
    """Every .wv case, covering FEATURES together"""
    c = []
    c.append(make_case('mono16', 1, channels=1, nterms=[1, 3, 8]))
    c.append(make_case('stereo16_joint', 2, joint=True, nterms=[16, 0, 1]))
    c.append(make_case('stereo16_cross', 3, nterms=[12, 16, 9], counts=(900, 600)))
    c.append(make_case('stereo24', 4, bps=3, nterms=[16, 7, 2], joint=True))
    c.append(make_case('stereo20_shift', 5, bps=3, shift=4, nterms=[4, 10, 13], rate=44100))
    c.append(make_case('mono24_custom_rate', 6, channels=1, bps=3, rate=37800, nterms=[6, 11, 14]))
    c.append(make_case('false_stereo16', 7, false_stereo=True, nterms=[2, 15, 3]))
    c.append(make_case('three24', 8, channels=3, bps=3, nterms=[5, 0, 16, 4, 12, 7]))
    c.append(make_case('six16', 9, channels=6, joint=True, counts=(500, 400)))
    c.append(make_case('eight24', 10, channels=8, bps=3, counts=(400, 350)))
    c.append(make_case('int32_zeros16', 11, int32=('zeros', 3), nterms=[3, 4, 5]))
    c.append(make_case('int32_ones24', 12, bps=3, int32=('ones', 5), nterms=[8, 2, 16]))
    c.append(make_case('int32_dups16', 13, channels=1, int32=('dups', 2), nterms=[1, 2, 9]))
    c.append(make_case('shift16', 14, shift=2, nterms=[6, 6, 6], rate=96000))
    riff = riff_header(2, 48000, 2, 1700, pad=700)
    c.append(make_case('riff_config_md5', 15, nterms=[10, 3, 6], meds=[[0, 0, 0], [0, 0, 0]],
                       extra_first=[subblock(ID_RIFF_HEADER, riff), subblock(ID_CONFIG, b'\x01\x02\x03'),
                                    subblock(0x3A, b'unknown optional sub-block')],
                       extra_last=[subblock(ID_RIFF_TRAILER, b'LIST' + struct.pack('<I', 4) + b'INFO'),
                                   subblock(ID_MD5, bytes(range(16)))]))
    c[-1].used |= {'riff_header', 'riff_trailer', 'config', 'md5', 'unknown_subblock', 'odd_subblock',
                   'large_subblock'}
    c.append(make_case('tagged_ape', 16, channels=1, nterms=[2, 7, 16], counts=(500, 200), version=0x410))
    c[-1].tail = apetag()
    c[-1].used.add('apetag')
    c.append(make_case('tagged_id3', 17, nterms=[1, 13, 3], counts=(500, 200), version=0x402))
    c[-1].tail = id3v1()
    c[-1].used.add('id3v1')
    return c


def assert_coverage(cases):
    used = set().union(*[c.used for c in cases])
    missing = FEATURES - used
    assert not missing, sorted(missing)


def long_stream(bits=24, minutes=90, block=24000, n_unique=4, seed=40):
    """A stereo 48 kHz case of n_unique blocks, and the .wv bytes of `minutes` minutes of them repeated (block_index
    rewritten): (case, data, repeats)."""
    case = make_case('long', seed, bps=bits // 8, counts=(block,) * n_unique, nterms=[2, 5, 8, 3], joint=True,
                     silence=False, spike=False, amp_bits=bits - 2)
    reps = minutes * 60 * 48000 // (block * n_unique)
    total = reps * n_unique * block
    out = []
    at = 0
    for _ in range(reps):
        for blocks, count in zip(case.frames, case.counts):
            for flags, crc, body in blocks:
                out.append(header(len(body), 0x407, total, at, count, flags, crc) + body)
            at += count
    return case, b''.join(out), reps


def _rewrite(data, at, fmt, value):
    b = bytearray(data)
    struct.pack_into(fmt, b, at, value)
    return bytes(b)


def _block_offsets(data):
    at, out = 0, []
    while at + 32 <= len(data) and data[at:at + 4] == b'wvpk':
        out.append(at)
        at += 8 + struct.unpack_from('<I', data, at + 4)[0]
    return out


def _sub(body, sid):
    """(offset, header bytes, payload size) of the first sub-block of `body` with id & 0x3f == sid"""
    at = 0
    while at < len(body):
        i, w = body[at], body[at + 1]
        h = 2
        if i & 0x80:
            w |= struct.unpack_from('<H', body, at + 2)[0] << 8
            h = 4
        if i & 0x3F == sid:
            return at, h, 2 * w - (1 if i & 0x40 else 0)
        at += h + 2 * w
    raise KeyError(sid)


def wv_bytes(frames, counts, version=0x407, total=None):
    """The .wv file of frames [[(flags, crc, body)]]"""
    out, at = [], 0
    total = sum(counts) if total is None else total
    for blocks, count in zip(frames, counts):
        for flags, crc, body in blocks:
            out.append(header(len(body), version, total, at, count, flags, crc) + body)
        at += count
    return b''.join(out)


def damaged_cases():
    """(base case, [(name, .wv bytes, block, message regex, in_kernel)]): one per refusal.  `block` is the index of the
    block the message names (None: a file-level refusal); in_kernel marks the refusals the GPU decoder makes (the rest
    are the host reader's)."""
    base = make_case('damage_base', 30, counts=(400, 400, 400), nterms=[3, 5, 2])
    good = base.wv()
    offs = _block_offsets(good)
    out = []

    def add(name, data, block, regex, kernel):
        out.append((name, data, block, regex, kernel))

    def edit(bi, fn):
        frames = [[list(b) for b in f] for f in base.frames]
        fn(frames[bi][0])
        return wv_bytes([[tuple(b) for b in f] for f in frames], base.counts)

    def body_edit(bi, fn):
        def apply(b):
            b[2] = fn(b[2])
        return edit(bi, apply)

    def flag_all(fn):
        frames = [[(fn(f), c, b) for f, c, b in blocks] for blocks in base.frames]
        return wv_bytes(frames, base.counts)

    def set_byte(body, at, v):
        return body[:at] + bytes([v]) + body[at + 1:]

    add('bad_version', _rewrite(good, offs[1] + 8, '<H', 0x401), 1, 'version 0x401', False)
    add('size_past_file', _rewrite(good, offs[2] + 4, '<I', len(good)), 2, 'runs past the end of the file', False)
    add('subblock_overrun', body_edit(1, lambda b: b + b'\x21\x40'), 1, 'sub-block runs past its block', True)
    add('no_bitstream', body_edit(1, lambda b: set_byte(b, _sub(b, ID_BITS)[0], 0x30 | (b[_sub(b, ID_BITS)[0]] & 0xC0))),
        1, 'no ID_WV_BITSTREAM', True)
    add('bad_term', body_edit(0, lambda b: set_byte(b, _sub(b, ID_TERMS)[0] + 2, (b[2] & 0xE0) | (12 + 5))), 0,
        'invalid decorrelation term', True)
    add('too_many_terms', body_edit(0, lambda b: subblock(ID_TERMS, bytes([6] * 17)) + b[sum(_sub(b, ID_TERMS)[1:]) + (
        _sub(b, ID_TERMS)[2] & 1):]), 0, 'more than 16 decorrelation terms', True)

    def short_bits(b):
        at, h, size = _sub(b, ID_BITS)
        return b[:at] + subblock(ID_BITS, b[at + h:at + h + 6])
    add('bitstream_overrun', body_edit(2, short_bits), 2, 'bitstream reads past its sub-block', True)

    def bad_crc(b):
        b[1] ^= 1
    add('crc', edit(1, bad_crc), 1, 'CRC mismatch', True)
    add('index_gap', _rewrite(good, offs[2] + 16, '<I', 801), 2, 'block_index 801', False)
    add('cut_last_block', good[:-7], 2, 'cut short', False)
    add('total_mismatch', base.wv(total=1300), None, 'header says 1300 samples', False)
    add('trailing_junk', good + b'junk' * 10, 3, 'not a WavPack block header', False)

    def not_initial(b):
        b[0] &= ~INITIAL
    add('not_initial', edit(1, not_initial), 1, 'INITIAL', False)
    for kind, flag in (('hybrid', HYBRID), ('float', FLOAT), ('DSD', DSD)):
        add(kind.lower(), flag_all(lambda f, flag=flag: f | flag), 0, 'WavPack \\(' + kind, False)
    for width, low in (('1-byte', 0), ('4-byte', 3)):
        add(width, flag_all(lambda f, low=low: (f & ~3) | low), 0, width, False)
    sent = make_case('sent_bits', 32, counts=(300,), nterms=[2], int32=('zeros', 1))
    b = sent.frames[0][0][2]
    at, h, size = _sub(b, ID_INT32)
    add('int32_sent_bits', wv_bytes([[(sent.frames[0][0][0], sent.frames[0][0][1], set_byte(b, at + h, 4))]],
                                    sent.counts), 0, 'extended precision', False)
    add('wvx', body_edit(0, lambda b: subblock(ID_WVX, bytes(8)) + b), 0, 'extended precision', False)
    mono = make_case('mono_no_terms', 33, channels=1, counts=(300, 300), nterms=[1])
    frames = [list(f) for f in mono.frames]
    rng = np.random.default_rng(33)
    flags, crc, body = encode_block(signal(rng, 300, 1, 1 << 14), mono.st, rng, set(), 0, 'mono')
    frames[1] = [(flags | INITIAL | FINAL, crc, body)]
    add('mono_no_terms', wv_bytes(frames, mono.counts), 1, 'mono block without decorrelation terms', True)
    return base, out
