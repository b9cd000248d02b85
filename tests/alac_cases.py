"""A seeded ALAC (Apple Lossless) writer for the tests: streams whose PCM is known, and damaged copies.

The writer mirrors the decoder's arithmetic to find residuals (the adaptive LPC runs the same wrap-around steps as
FFmpeg's `alac` decoder), then codes them with the adaptive Golomb code, its escapes and its zero runs.  Every case
records which coding features it used, and `assert_coverage` checks that the cases together use every one the decoder
handles: channel layouts 1-8 as Apple lays them out, 16/20/24/32 bits with 0/1/2 shifted bytes, escape elements
(32 bits included), has-size frames mid-stream and at the end, LPC orders 0-31, quantisations, pbFactor 0-7,
prediction type 15, mixRes zero and nonzero, Rice parameters up to kb, Golomb escapes, zero runs up to the longest,
full-scale residuals, several (pb, mb, kb) configs and frame lengths, and bytes after END.

A case's `pcm` is (frames, channels) int64 at its bit depth in FFmpeg's channel order; `pcm16` the int16 the loader
keeps (the top 16 bits)."""
import struct

import numpy as np

SCE, CPE, LFE, END = 0, 1, 3, 7
# Apple's element layouts (coded order) for 1-8 channels
LAYOUTS = {1: [SCE], 2: [CPE], 3: [SCE, CPE], 4: [SCE, CPE, SCE], 5: [SCE, CPE, CPE], 6: [SCE, CPE, CPE, LFE],
           7: [SCE, CPE, CPE, SCE, LFE], 8: [SCE, CPE, CPE, CPE, LFE]}
# FFmpeg's output channel of the element at coded channel position ch
OFFSETS = {1: [0], 2: [0, 1], 3: [2, 0, 1], 4: [2, 0, 1, 3], 5: [2, 0, 1, 3, 4], 6: [2, 0, 1, 4, 5, 3],
           7: [2, 0, 1, 4, 5, 6, 3], 8: [2, 6, 7, 0, 1, 4, 5, 3]}
M32 = 0xFFFFFFFF


def i32(v):
    v &= M32
    return v - (1 << 32) if v >> 31 else v


def sx(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def sgn(v):
    return (v > 0) - (v < 0)


def log2(v):
    return v.bit_length() - 1 if v > 0 else 0


class Bits(object):
    def __init__(self):
        self.parts = []
        self.n = 0

    def put(self, n, v):
        if n:
            self.parts.append(format(v & ((1 << n) - 1), '0%db' % n))
            self.n += n

    def bytes(self):
        s = ''.join(self.parts)
        s += '0' * (-len(s) % 8)
        return int(s, 2).to_bytes(len(s) // 8, 'big') if s else b''


class Config(object):
    def __init__(self, frame_length=4096, bit_depth=16, pb=40, mb=10, kb=14, channels=2, rate=48000):
        self.frame_length, self.bit_depth, self.pb, self.mb, self.kb = frame_length, bit_depth, pb, mb, kb
        self.channels, self.rate = channels, rate

    def cookie(self):
        """The 24-byte ALACSpecificConfig (Matroska's CodecPrivate; MP4 wraps it in an `alac` box)."""
        return struct.pack('>IBBBBBBHIII', self.frame_length, 0, self.bit_depth, self.pb, self.mb, self.kb,
                           self.channels, 255, 0, 0, self.rate)

    def array(self):
        return np.array([self.frame_length, self.bit_depth, self.pb, self.mb, self.kb, self.channels, self.rate],
                        np.int32)


def lpc_residuals(u, bps, coefs, order, quant):
    """The residuals for which FFmpeg's lpc_prediction gives back u (its adaptation included)."""
    n = len(u)
    e = [0] * n
    if n == 0:
        return e
    e[0] = u[0]
    if order == 0:
        return list(u)
    if order == 31:
        return [u[0]] + [sx(u[i] - u[i - 1], bps) for i in range(1, n)]
    coefs = list(coefs)
    i = 1
    while i <= order and i < n:
        e[i] = sx(u[i] - u[i - 1], bps)
        i += 1
    half = 1 << (quant - 1)
    while i < n:
        d = u[i - order - 1]
        pred = u[i - order:i]
        acc = i32(sum((pred[j] - d) * coefs[j] for j in range(order)))
        val = (acc + half) >> quant
        ei = sx(u[i] - val - d, bps)
        e[i] = ei
        ev = ei & M32
        es = sgn(i32(ev))
        if es:
            j = 0
            while j < order and i32(ev * es) > 0:
                v = i32(d - pred[j])
                s = sgn(v) * es
                c = coefs[j] - s
                coefs[j] = ((c + 32768) & 0xFFFF) - 32768
                v = i32(v * s)
                ev = (ev - (v >> quant) * (j + 1)) & M32
                j += 1
        i += 1
    return e


class Coder(object):
    """Golomb coding of one channel's residuals, mirroring the decoder's history."""

    def __init__(self, bits, cfg, used):
        self.b, self.cfg, self.used = bits, cfg, used

    def scalar(self, x, k, size, force_escape=False):
        k = min(k, self.cfg.kb)
        m = (1 << k) - 1
        q, r = divmod(x, m)
        if q > 8 or force_escape:
            self.b.put(9, 0x1FF)
            self.b.put(size, x)
            self.used.add('golomb_escape')
            return
        self.used.add('rice_k%d' % k)
        if q:
            self.b.put(q, (1 << q) - 1)
        self.b.put(1, 0)
        if k != 1:
            if r > 0:
                self.b.put(k, r + 1)
            else:
                self.b.put(k - 1, 0)

    def residuals(self, e, bps, mult, escape_every=0):
        cfg = self.cfg
        history = cfg.mb
        sign_mod = 0
        n = len(e)
        i = 0
        while i < n:
            k = min(log2((history >> 9) + 3), cfg.kb)
            if k == cfg.kb:
                self.used.add('rice_at_kb')
            v = e[i]
            x = (2 * v if v >= 0 else -2 * v - 1) & M32
            if x >= 1 << (bps - 1):
                self.used.add('full_scale')
            self.scalar(x - sign_mod, k, bps, force_escape=bool(escape_every) and i % escape_every == 3)
            i += 1
            if x > 0xFFFF:
                history = 0xFFFF
            else:
                history = (history + x * mult - ((history * mult) >> 9)) & M32
            sign_mod = 0
            if history < 128 and i < n:
                k = 7 - log2(history) + ((history + 16) >> 6)
                run = 0
                while i < n and e[i] == 0:
                    i += 1
                    run += 1
                self.scalar(run, k, 16)
                self.used.add('zero_run' if run else 'zero_run_empty')
                if run == n - 1:
                    self.used.add('longest_run')
                sign_mod = 1 if run <= 0xFFFF else 0
                history = 0


class Element(object):
    """How one element is coded."""

    def __init__(self, escape=False, extra=0, shift=2, weight=2, chans=None):
        self.escape, self.extra, self.shift, self.weight = bool(escape), extra, shift, weight
        # per channel: (ptype, quant, rhm, order, coefs)
        self.chans = chans


def encode_frame(cfg, pcm, elems, has_size=False, trailing=b'', escape_every=0, used=None, no_end=False, tags=None,
                 nbits=None):
    """One frame: pcm (n, channels) at cfg.bit_depth in FFmpeg's channel order; elems one Element per layout entry.
    nbits, a list, receives the frame's length in bits before the padding to a byte."""
    used = set() if used is None else used
    n = len(pcm)
    b = Bits()
    layout = LAYOUTS[cfg.channels] if tags is None else tags
    ch = 0
    for t, el in zip(layout, elems):
        nch = 2 if t == CPE else 1
        off = OFFSETS[cfg.channels][ch] if ch < cfg.channels else 0
        data = [[int(v) for v in pcm[:, off + c]] for c in range(nch)] if ch < cfg.channels else \
            [[0] * n for _ in range(nch)]
        ch += nch
        b.put(3, t)
        b.put(4, 0)
        b.put(12, 0)
        b.put(1, int(has_size))
        extra = el.extra * 8
        b.put(2, el.extra)
        b.put(1, int(el.escape))
        if has_size:
            b.put(32, n)
        used.add({SCE: 'sce', CPE: 'cpe', LFE: 'lfe'}.get(t, 'tag%d' % t))
        used.add('depth%d_extra%d' % (cfg.bit_depth, el.extra))
        if el.escape:
            used.add('escape_element')
            used.add('escape_element_%d' % cfg.bit_depth)
            for i in range(n):
                for c in range(nch):
                    b.put(cfg.bit_depth, data[c][i])
            continue
        bps = cfg.bit_depth - extra + nch - 1
        low = [[v & ((1 << extra) - 1) for v in d] for d in data]
        high = [[v >> extra for v in d] for d in data]
        shift, weight = (el.shift, el.weight) if nch == 2 else (0, 0)
        if nch == 2:
            used.add('mixres_nonzero' if weight else 'mixres_zero')
            if weight:
                L, R = high
                bo = [sx(l - r, 32) for l, r in zip(L, R)]
                ao = [sx(r + (i32(bv * weight) >> shift), 32) for r, bv in zip(R, bo)]
                high = [ao, bo]
        b.put(8, shift)
        b.put(8, weight)
        for c in range(nch):
            ptype, quant, rhm, order, coefs = el.chans[c]
            b.put(4, ptype)
            b.put(4, quant)
            b.put(3, rhm)
            b.put(5, order)
            for j in range(order - 1, -1, -1):
                b.put(16, coefs[j])
            used.add('order%d' % order)
            used.add('pb%d' % rhm)
            used.add('quant%d' % quant)
            if ptype == 15:
                used.add('ptype15')
        if extra:
            for i in range(n):
                for c in range(nch):
                    b.put(extra, low[c][i])
        for c in range(nch):
            ptype, quant, rhm, order, coefs = el.chans[c]
            u = [sx(v, bps) for v in high[c]]
            assert u == high[c], 'value outside the element width'
            e = lpc_residuals(u, bps, coefs, order, quant)
            if ptype == 15:
                e = [e[0]] + [sx(e[i] - e[i - 1], bps) for i in range(1, n)]
            Coder(b, cfg, used).residuals(e, bps, rhm * cfg.pb // 4, escape_every)
    if not no_end:
        b.put(3, END)
    if nbits is not None:
        nbits.append(b.n)
    if trailing:
        used.add('trailing_bytes')
    if has_size:
        used.add('has_size')
    return b.bytes() + trailing


def frame_samples(cfg, frame):
    """A frame's sample count: its first element's has-size field, else frameLength."""
    if not (frame[2] >> 4) & 1:
        return cfg.frame_length
    return (int.from_bytes(frame[2:8], 'big') >> 9) & 0xFFFFFFFF


def to16(pcm, depth):
    pcm = np.asarray(pcm, np.int64)
    return pcm.astype(np.int16) if depth == 16 else ((pcm << (32 - depth)) >> 16).astype(np.int16)


class AlacCase(object):
    def __init__(self, name, cfg, frames, pcm, used):
        self.name, self.cfg, self.frames, self.pcm, self.used = name, cfg, frames, pcm, used
        self.pcm16 = to16(pcm, cfg.bit_depth)
        self.data = b''.join(frames)
        self.offsets = np.concatenate([[0], np.cumsum([len(f) for f in frames])[:-1]]).astype(np.int64)
        self.channels, self.rate, self.bits = cfg.channels, cfg.rate, cfg.bit_depth


def signal(rng, n, channels, depth, style):
    """Test audio at `depth` bits: smooth tones with noise, silences (zero runs) and, for 'full', full-scale steps."""
    t = np.arange(n)
    top = (1 << (depth - 1)) - 1
    out = np.zeros((n, channels), np.int64)
    for c in range(channels):
        f = rng.uniform(0.002, 0.05)
        amp = top * rng.uniform(0.05, 0.6)
        x = amp * np.sin(2 * np.pi * f * t + c) + rng.normal(0, top * 0.002 + 1, n)
        x = np.round(x).astype(np.int64)
        if style == 'full':
            x[::7] = top
            x[3::7] = -top - 1
        if style in ('silence', 'mixed'):
            a = int(rng.integers(0, max(1, n // 2)))
            x[a:a + n // 3] = 0
        out[:, c] = np.clip(x, -top - 1, top)
    if style == 'silent_tail':
        out[0] = 1
        out[1:] = 0
    return out


def _chan_params(rng, order=None, ptype=0, quant=None, rhm=None):
    order = int(rng.integers(0, 32)) if order is None else order
    quant = int(rng.integers(9, 15)) if quant is None else quant
    rhm = int(rng.integers(0, 8)) if rhm is None else rhm
    if order in (0, 31):
        coefs = [int(rng.integers(-500, 500)) for _ in range(order)]
    else:
        # a stable-ish predictor: a first-difference start with small random coefficients
        coefs = [int(rng.integers(-300, 300)) for _ in range(order)]
        coefs[-1] += 1 << quant
    return (ptype, quant, rhm, order, coefs)


def make(name, cfg, n_frames, seed, style='mixed', sizes=None, extra=None, escape_frames=(), ptype15=False,
         orders=None, mix=(2, 2), trailing_frames=(), escape_every=0):
    """A stream of n_frames frames; sizes[f] (default frameLength) gives has-size frames where shorter."""
    rng = np.random.default_rng(seed)
    used = set()
    frames, pcms = [], []
    k_order = 0
    for f in range(n_frames):
        n = cfg.frame_length if sizes is None else sizes[f]
        pcm = signal(rng, n, cfg.channels, cfg.bit_depth, style if f % 3 else ('full' if style == 'full' else 'mixed'))
        elems = []
        for t in LAYOUTS[cfg.channels]:
            nch = 2 if t == CPE else 1
            ex = extra[(f + len(elems)) % len(extra)] if extra else 0
            if cfg.bit_depth == 32 and nch == 2 and ex == 0:
                ex = 1                                     # 33-bit stereo elements do not exist (FFmpeg refuses them)
            chans = []
            for c in range(nch):
                order = orders[k_order % len(orders)] if orders else None
                k_order += 1
                chans.append(_chan_params(rng, order=order, ptype=15 if ptype15 and (f + c) % 2 == 0 else 0,
                                          rhm=(f + c + len(elems)) % 8))
            sh, wt = mix if f % 2 == 0 else (0, 0)
            elems.append(Element(escape=f in escape_frames and (nch == 1 or cfg.bit_depth < 32 or ex > 0),
                                 extra=ex, shift=sh, weight=wt, chans=chans))
        frames.append(encode_frame(cfg, pcm, elems, has_size=n != cfg.frame_length or (sizes is not None and f == 1),
                                   trailing=b'\xa5\x00\x17' if f in trailing_frames else b'', used=used,
                                   escape_every=escape_every))
        pcms.append(pcm)
    return AlacCase(name, cfg, frames, np.concatenate(pcms), used)


def all_cases():
    c = []
    c.append(make('mono16', Config(frame_length=256, bit_depth=16, channels=1), 6, 1, orders=list(range(0, 32, 3)),
                  escape_frames=(2,), trailing_frames=(4,)))
    c.append(make('stereo16', Config(frame_length=300, bit_depth=16, channels=2), 8, 2, orders=list(range(1, 32, 3)),
                  sizes=[300, 300, 120, 300, 300, 17, 300, 55], escape_every=50))
    c.append(make('stereo16_pt15', Config(frame_length=200, bit_depth=16, channels=2, pb=28, mb=25, kb=10), 5, 3,
                  ptype15=True, orders=[31, 8, 4, 2, 12, 31, 30, 29, 28, 0], mix=(5, 7)))
    c.append(make('full16', Config(frame_length=128, bit_depth=16, channels=2, kb=6), 4, 4, style='full',
                  orders=[4, 8, 1, 0]))
    c.append(make('orders', Config(frame_length=80, bit_depth=16, channels=1, pb=33, mb=12, kb=13), 32, 6,
                  orders=list(range(32))))
    c.append(make('silence16', Config(frame_length=160, bit_depth=16, channels=1, kb=20), 3, 5, style='silent_tail',
                  orders=[0]))
    for ch in range(3, 9):
        c.append(make('layout%d' % ch, Config(frame_length=96, bit_depth=16, channels=ch, pb=40, mb=10, kb=14), 3,
                      10 + ch, orders=[0, 2, 4, 8, 16, 24, 5, 7, 3]))
    c.append(make('d20', Config(frame_length=128, bit_depth=20, channels=2), 4, 21, extra=[0, 1, 2],
                  orders=[8, 4, 6], escape_frames=(3,)))
    c.append(make('d24', Config(frame_length=128, bit_depth=24, channels=2, kb=16), 5, 22, extra=[0, 1, 2],
                  orders=[8, 2, 12, 20, 0], sizes=[128, 128, 128, 128, 77], escape_frames=(2,), trailing_frames=(1,)))
    c.append(make('d24_mono_pt15', Config(frame_length=100, bit_depth=24, channels=1, pb=12, mb=40, kb=18), 4, 23,
                  extra=[1, 0, 2], ptype15=True, orders=[31, 16, 10, 3]))
    c.append(make('d32', Config(frame_length=96, bit_depth=32, channels=2, kb=24), 4, 24, extra=[1, 2],
                  orders=[8, 4, 31, 0], escape_frames=(1,)))
    c.append(make('d32_mono', Config(frame_length=96, bit_depth=32, channels=1, kb=24), 4, 25, extra=[0, 1, 2],
                  orders=[6, 0, 12, 9], escape_frames=(0, 3), style='full'))
    c.append(make('apple', Config(frame_length=4096, bit_depth=16, channels=2), 3, 26, orders=[8],
                  sizes=[4096, 4096, 1000]))
    return c


def assert_coverage(cases):
    used = set().union(*[c.used for c in cases])
    need = {'sce', 'cpe', 'lfe', 'escape_element', 'escape_element_32', 'has_size', 'ptype15', 'mixres_zero',
            'mixres_nonzero', 'golomb_escape', 'zero_run', 'longest_run', 'full_scale', 'trailing_bytes', 'rice_at_kb'}
    need |= {'order%d' % k for k in range(32)} | {'pb%d' % k for k in range(8)}
    need |= {'depth%d_extra%d' % (d, e) for d in (16,) for e in (0,)}
    need |= {'depth%d_extra%d' % (d, e) for d in (20, 24, 32) for e in (0, 1, 2)}
    missing = need - used
    assert not missing, sorted(missing)
    assert {c.channels for c in cases} == set(range(1, 9))
    assert {c.bits for c in cases} == {16, 20, 24, 32}
    configs = {(c.cfg.pb, c.cfg.mb, c.cfg.kb, c.cfg.frame_length) for c in cases}
    assert len(configs) >= 5
    # has-size frames mid-stream and at the end
    assert any(len(c.frames) > 2 and c.pcm.shape[0] % c.cfg.frame_length for c in cases)


def _damage(case, f, new_frame):
    frames = list(case.frames)
    frames[f] = new_frame
    return frames


def damaged_cases():
    """(name, config, frames, frame index, message regex): copies of a small stream with one frame damaged."""
    base = make('base', Config(frame_length=64, bit_depth=16, channels=1), 5, 90, orders=[4])
    cfg = base.cfg
    rng = np.random.default_rng(91)
    pcm = signal(rng, 64, 1, 16, 'mixed')
    el = [Element(chans=[_chan_params(rng, order=4)])]
    out = []

    def frame(**kw):
        return encode_frame(kw.pop('cfg', cfg), kw.pop('pcm', pcm), kw.pop('elems', el), **kw)

    # an element tag FFmpeg refuses (CCE)
    out.append(('bad_tag', cfg, _damage(base, 2, frame(tags=[2])), 2, 'element tag'))
    # a CPE in a mono stream: more channels than the config declares
    st = Config(frame_length=64, bit_depth=16, channels=2)
    cpe = encode_frame(st, np.repeat(pcm, 2, 1), [Element(shift=0, weight=0, chans=[_chan_params(rng, order=4)] * 2)])
    out.append(('too_many_channels', cfg, _damage(base, 3, cpe), 3, 'more channels'))
    # a stereo config fed a mono frame: fewer channels
    out.append(('too_few_channels', st, [cpe, cpe, frame(), cpe], 2, 'fewer channels'))
    # sample counts 0 and above frameLength
    out.append(('count_above', cfg, _damage(base, 1, frame(has_size=True, pcm=np.repeat(pcm, 2, 0)[:65])), 1,
                'sample count'))
    out.append(('count_zero', cfg, _damage(base, 4, _with_size(frame(has_size=True, pcm=pcm[:10]), 0)), 4,
                'sample count'))
    # prediction type 3
    bad = [Element(chans=[(3,) + _chan_params(rng, order=4)[1:]])]
    out.append(('prediction_type', cfg, _damage(base, 0, encode_frame(cfg, pcm, bad)), 0, 'prediction type'))
    # a frame cut short
    out.append(('cut_frame', cfg, _damage(base, 2, base.frames[2][:len(base.frames[2]) // 2]), 2, 'reads past'))
    # no END: the frame ends within 3 bits of its last element
    out.append(('no_end', cfg, _damage(base, 3, _without_end(cfg, pcm, el)), 3, 'without END element'))
    # the last frame cut inside its predictor: order 31 declared, no coefficient left (the reads must stay inside the
    # buffer's padding)
    cut = encode_frame(cfg, pcm, [Element(chans=[_chan_params(rng, order=31)])])[:7]
    out.append(('cut_last_frame', cfg, _damage(base, len(base.frames) - 1, cut), len(base.frames) - 1, 'reads past'))
    return base, out


def _with_size(frame, n):
    """The frame with the 32-bit sample count of its first element (has_size set) replaced by n."""
    b = Bits()
    bits = ''.join(format(x, '08b') for x in frame)
    s = bits[:23] + format(n, '032b') + bits[55:]
    b.parts = [s]
    return b.bytes()


def _without_end(cfg, pcm, el):
    """A frame without END whose padding to a byte leaves fewer than 3 bits, so no further tag can be read: the
    sample count (has-size) is chosen for it."""
    for m in range(len(pcm), 1, -1):
        nbits = []
        frame = encode_frame(cfg, pcm[:m], el, has_size=m != len(pcm), no_end=True, nbits=nbits)
        if -nbits[0] % 8 < 3:
            return frame
    raise AssertionError('no sample count leaves the frame within 3 bits of a byte')


def long_stream(bits=24, minutes=90, frame_length=4096, seed=7, n_unique=16):
    """(frames, pcm, reps): n_unique frames of Apple's default coding (pb 40, mb 10, kb 14, LPC order 8, stereo) whose
    repetition `reps` times makes `minutes` of 48 kHz audio (the last repetition may be cut by the caller)."""
    cfg = Config(frame_length=frame_length, bit_depth=bits, channels=2)
    rng = np.random.default_rng(seed)
    frames, pcms = [], []
    for f in range(n_unique):
        pcm = signal(rng, frame_length, 2, bits, 'tone')
        el = [Element(extra=1 if bits > 16 else 0, chans=[_chan_params(rng, order=8, quant=9, rhm=4)] * 2)]
        frames.append(encode_frame(cfg, pcm, el))
        pcms.append(pcm)
    reps = -(-minutes * 60 * 48000 // (frame_length * n_unique))
    return cfg, frames, np.concatenate(pcms), reps


def escape_stream(pcm, cfg):
    """Frames of escape (uncompressed) elements for 16-bit pcm (frames, channels), written with NumPy: for long
    signals where the per-sample coder would be slow.  Channel layouts as LAYOUTS; has-size on a short last frame."""
    assert cfg.bit_depth == 16
    frames = []
    n = len(pcm)
    for a in range(0, n, cfg.frame_length):
        part = pcm[a:a + cfg.frame_length]
        m = len(part)
        bits = []
        ch = 0
        for t in LAYOUTS[cfg.channels]:
            nch = 2 if t == CPE else 1
            off = OFFSETS[cfg.channels][ch]
            ch += nch
            head = format(t, '03b') + '0' * 16 + ('1' if m != cfg.frame_length else '0') + '00' + '1'
            if m != cfg.frame_length:
                head += format(m, '032b')
            bits.append(np.array([int(x) for x in head], np.uint8))
            raw = np.ascontiguousarray(part[:, off:off + nch].astype('>i2')).view(np.uint8)
            bits.append(np.unpackbits(raw.reshape(-1)))
        bits.append(np.array([1, 1, 1], np.uint8))
        frames.append(np.packbits(np.concatenate(bits)).tobytes())
    return AlacCase('escape', cfg, frames, np.asarray(pcm, np.int64), {'escape_element'})
