"""A seeded NumPy FLAC encoder and the FLAC files the tests decode.

Pure NumPy, shared by the CPU tests (tests/test_flac_cases.py against the libavcodec decoder of oracle/ref_flac.py,
tests/test_kernel_emulation_flac.py against sb_flac.cuh compiled with g++) and the GPU test of the loader
(tests/test_gpu_flac.py).  A case is a FLAC file as bytes, written bit by bit so that every coding choice is the case's
own, plus the PCM it holds.  The PCM comes from loader_cases.family_pcm (so the median selector's edge families go
through FLAC too); 24-bit samples are the int16 values in the top 16 bits over seeded low bytes.

The set spans (assert_coverage checks it):
* every subframe type: CONSTANT, VERBATIM, FIXED orders 0-4, LPC orders 1-32 with coefficient precisions 1-15 and
  shifts 0-15; LPC coefficients come from Levinson-Durbin on the frame, so residuals look like a real encoder's;
* wasted bits, on an independent channel and on a side channel;
* all four channel assignments, with full-scale values so that the side channel needs 17 or 25 bits;
* Rice with 4-bit and 5-bit parameters, escape partitions of 0 and of n raw bits, partition orders 0-8 (the first
  partition is shortened by the predictor order);
* every block-size code and every sample-rate code (STREAMINFO, table, kHz, Hz, tens of Hz), explicit and
  STREAMINFO bit depths, a short last frame;
* fixed and variable blocking, with UTF-8 coded numbers of 1 to 5 bytes;
* each skippable metadata block and an ID3v2 prefix;
* 16 and 24 bits, 1 to 8 channels.

corrupt_cases() damages one file in each way the decoder must refuse, with the frame the error must name and the text
it must carry; baseline_file() builds the 90-minute, 1 GB file of the BASELINE-size test."""
import functools
import math
import struct

import numpy as np

from tests import loader_cases as lc

SEED = 20261016
BLOCK_CODES = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13,
               16384: 14, 32768: 15}
RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
              96000: 11}
BITS_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}
SUBFRAME_KINDS = ('constant', 'verbatim', 'fixed', 'lpc')


# ---- bits --------------------------------------------------------------------------------------------------------
class BitWriter(object):
    """MSB-first bit string built from NumPy arrays of 0/1."""

    def __init__(self):
        self.parts = []
        self.n = 0

    def put(self, values, nbits):
        """values (scalar or array) as two's complement fields of nbits bits each."""
        if nbits == 0:
            return
        v = np.atleast_1d(np.asarray(values, np.int64)) & ((1 << nbits) - 1)
        bits = ((v[:, None] >> np.arange(nbits - 1, -1, -1, dtype=np.int64)[None, :]) & 1).astype(np.uint8).reshape(-1)
        self.parts.append(bits)
        self.n += bits.size

    def put_rice(self, values, k):
        """Zigzag-folded values as Rice codes with parameter k: the quotient in unary (zeros, then a one), then k bits."""
        v = np.asarray(values, np.int64)
        if v.size == 0:
            return
        u = np.where(v >= 0, 2 * v, -2 * v - 1)
        q = u >> k
        length = q + 1 + k
        start = np.concatenate([[0], np.cumsum(length)[:-1]])
        bits = np.zeros(int(length.sum()), np.uint8)
        bits[start + q] = 1
        if k:
            low = (u[:, None] >> np.arange(k - 1, -1, -1, dtype=np.int64)[None, :]) & 1
            bits[(start + q + 1)[:, None] + np.arange(k)[None, :]] = low
        self.parts.append(bits)
        self.n += bits.size

    def put_unary(self, n):
        self.put(1, n + 1)                     # n zeros, then a one

    def align(self):
        if self.n % 8:
            self.put(0, 8 - self.n % 8)

    def tobytes(self):
        assert self.n % 8 == 0
        return np.packbits(np.concatenate(self.parts) if self.parts else np.zeros(0, np.uint8)).tobytes()


def crc8(data):
    crc = 0
    for b in data:
        crc ^= b
        for _ in range(8):
            crc = ((crc << 1) ^ 0x07) & 0xFF if crc & 0x80 else (crc << 1) & 0xFF
    return crc


def _crc16_table():
    t = np.zeros(256, np.uint32)
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        t[i] = c
    return t


CRC16_TABLE = _crc16_table()


def crc16_many(frames):
    """CRC-16 of many byte strings at once: right-aligned in one matrix (leading zero bytes leave a zero CRC at 0)."""
    if not frames:
        return []
    width = max(len(f) for f in frames)
    m = np.zeros((len(frames), width), np.uint8)
    for i, f in enumerate(frames):
        m[i, width - len(f):] = np.frombuffer(f, np.uint8)
    return list(crc16_matrix(m))


def _zero_shift(v, nbytes):
    """The CRC register v after nbytes zero bytes (a linear map of v)."""
    v = np.asarray(v, np.uint32)
    for _ in range(nbytes):
        v = ((v << 8) ^ CRC16_TABLE[(v >> 8) & 0xFF]) & 0xFFFF
    return v


def crc16_matrix(m):
    """CRC-16 of every row of a uint8 matrix.  Rows are cut into K chunks of c bytes (zeros in front, which leave the
    CRC unchanged); the chunk CRCs are combined by Horner's rule, crc = shift(crc, c) ^ crc_k, the shift being a
    linear map applied with two 256-entry tables.  About 2 sqrt(width) vector steps instead of width."""
    rows, width = m.shape
    c = max(1, int(math.ceil(math.sqrt(width))))
    k = -(-width // c)
    pad = np.zeros((rows, k * c), np.uint8)
    pad[:, k * c - width:] = m
    chunks = pad.reshape(rows * k, c)
    crc = np.zeros(rows * k, np.uint32)
    for j in range(c):
        crc = ((crc << 8) ^ CRC16_TABLE[((crc >> 8) ^ chunks[:, j]) & 0xFF]) & 0xFFFF
    crc = crc.reshape(rows, k)
    b = np.arange(256, dtype=np.uint32)
    t_lo, t_hi = _zero_shift(b, c), _zero_shift(b << 8, c)
    out = np.zeros(rows, np.uint32)
    for j in range(k):
        out = t_hi[out >> 8] ^ t_lo[out & 0xFF] ^ crc[:, j]
    return out


def utf8_number(n):
    if n < 0x80:
        return bytes([n])
    for nbytes, limit in ((2, 1 << 11), (3, 1 << 16), (4, 1 << 21), (5, 1 << 26), (6, 1 << 31), (7, 1 << 36)):
        if n < limit:
            break
    else:
        raise ValueError(n)
    out = []
    for _ in range(nbytes - 1):
        out.append(0x80 | (n & 0x3F))
        n >>= 6
    lead = (0xFF00 >> nbytes) & 0xFF
    return bytes([lead | n] + out[::-1])


# ---- prediction --------------------------------------------------------------------------------------------------
def fixed_residual(x, order):
    r = x.astype(np.int64)
    for _ in range(order):
        r = np.diff(r)
    return r                                  # len(x) - order values


def levinson(x, order):
    """LPC coefficients (x[i] ~ sum a[j] x[i-1-j]) from the autocorrelation of the Welch-windowed frame."""
    n = len(x)
    w = 1.0 - ((np.arange(n) - (n - 1) / 2.0) / ((n + 1) / 2.0)) ** 2
    xw = x.astype(np.float64) * w
    r = np.array([np.dot(xw[:n - k], xw[k:]) for k in range(order + 1)])
    if r[0] == 0:
        return np.zeros(order)
    r[0] *= 1.0 + 1e-9
    a = np.zeros(order)
    err = r[0]
    for i in range(order):
        k = (r[i + 1] - np.dot(a[:i], r[i:0:-1])) / err
        a[:i] = a[:i] - k * a[:i][::-1]
        a[i] = k
        err *= (1 - k * k)
        if err <= 0:
            break
    return a


def quantise_lpc(a, precision, shift=None):
    """libFLAC's rule when shift is None (the largest shift that keeps the largest coefficient in range, at most 15);
    otherwise the given shift, coefficients clipped to the precision."""
    lim = 1 << (precision - 1)
    if shift is None:
        cmax = np.max(np.abs(a)) if len(a) else 0.0
        if cmax <= 0:
            shift = 0
        else:
            shift = precision - 1 - (int(math.floor(math.log2(cmax))) + 1)
            shift = min(max(shift, 0), 15)
    q = np.clip(np.round(a * (1 << shift)), -lim, lim - 1).astype(np.int64)
    return q, shift


def lpc_residual(x, coef, shift):
    x = x.astype(np.int64)
    order = len(coef)
    n = len(x)
    pred = np.zeros(n - order, np.int64)
    for j in range(order):
        pred += coef[j] * x[order - 1 - j:n - 1 - j]
    return x[order:] - (pred >> shift)


# ---- subframes ---------------------------------------------------------------------------------------------------
def partition_params(res, n, order, porder, kmax):
    """Rice parameter of every partition (the best of three around log2 of the mean) and the bits they cost."""
    u = np.concatenate([np.zeros(order, np.int64), np.where(res >= 0, 2 * res, -2 * res - 1)]).reshape(1 << porder, -1)
    mean = u.mean(axis=1)
    k0 = np.clip(np.floor(np.log2(mean + 1)).astype(np.int64), 0, kmax)
    ks = np.stack([np.clip(k0 + d, 0, kmax) for d in (-1, 0, 1)])                    # (3, parts)
    cost = (u[None, :, :] >> ks[:, :, None]).sum(axis=2) + u.shape[1] * (ks + 1)
    best = cost.argmin(axis=0)
    return ks[best, np.arange(u.shape[0])], int(cost.min(axis=0).sum())


def write_residual(bw, res, n, order, spec):
    """spec: method ('rice' or 'rice2'), porder (largest wanted; the largest valid one at most this is used, or with
    porder_search the cheapest valid one up to it), escape: None, 'zero' (every partition escaped) or the index of the
    partition to escape."""
    method = spec.get('method', 'rice')
    pbits = 4 if method == 'rice' else 5
    escape_code = (1 << pbits) - 1
    valid = [po for po in range(spec.get('porder', 0) + 1) if (n >> po) << po == n and (n >> po) >= order]
    porder = valid[-1]
    if spec.get('porder_search'):
        porder = min(valid, key=lambda po: partition_params(res, n, order, po, escape_code - 1)[1] + (pbits << po))
    ks, _ = partition_params(res, n, order, porder, escape_code - 1)
    bw.put(0 if method == 'rice' else 1, 2)
    bw.put(porder, 4)
    psize = n >> porder
    used = {'porder': porder, 'method': method, 'escape': set(), 'params': set()}
    at = 0
    esc = spec.get('escape')
    for p in range(1 << porder):
        cnt = psize - (order if p == 0 else 0)
        part = res[at:at + cnt]
        at += cnt
        if esc == 'zero' or (esc is not None and esc == p):
            raw = 0 if not len(part) or not np.any(part) else int(max(np.max(part), -np.min(part) - 1)).bit_length() + 1
            bw.put(escape_code, pbits)
            bw.put(raw, 5)
            if raw:
                bw.put(part, raw)
            used['escape'].add(raw)
            continue
        k = int(ks[p])
        bw.put(k, pbits)
        bw.put_rice(part, k)
        used['params'].add(k)
    return used


def wasted_bits(x):
    nz = x[x != 0]
    if not len(nz):
        return 0
    w = 0
    v = np.bitwise_or.reduce(np.abs(nz.astype(np.int64)))
    while not (v >> w) & 1:
        w += 1
    return w


def write_subframe(bw, x, bps, spec, rng):
    """write_coded, or VERBATIM where the coded subframe would be larger, as a real encoder does (decoders may bound a
    frame by its verbatim size: FFmpeg's parser does)."""
    sub = BitWriter()
    info = write_coded(sub, x, bps, spec, rng)
    if info['kind'] not in ('verbatim', 'constant') and sub.n > 8 + bps * len(x):
        sub = BitWriter()
        info = write_coded(sub, x, bps, dict(spec, kind='verbatim'), rng)
        info['fallback'] = True
    bw.parts += sub.parts
    bw.n += sub.n
    return info


def write_coded(bw, x, bps, spec, rng):
    """One subframe of x (int64) at bps bits.  spec: kind ('constant', 'verbatim', 'fixed', 'lpc', 'auto'), order,
    precision, shift, wasted (use the wasted-bits flag when the samples allow), residual spec.  Returns what was
    written, for the coverage report."""
    n = len(x)
    kind = spec.get('kind', 'auto')
    if kind == 'constant' and not np.all(x == x[0]):
        kind = 'auto'
    w = wasted_bits(x) if spec.get('wasted', True) and kind != 'constant' else 0
    w = min(w, bps - 1)
    xs = x >> w
    sbps = bps - w
    info = {'kind': kind, 'wasted': w, 'bps': bps}
    if kind == 'auto':
        kind = 'lpc' if n > 32 else 'fixed'
        spec = dict(spec, order=min(spec.get('order') or 8, n - 1), porder_search=True, porder=spec.get('porder', 8))
        info['kind'] = kind
    if kind == 'lpc' and spec.get('order', 8) > n - 1:
        kind = info['kind'] = 'fixed'
        spec = dict(spec, order=min(2, n))
    header = {'constant': 0, 'verbatim': 1}.get(kind)
    if kind == 'fixed':
        order = min(spec.get('order', 2), 4, n)
        header = 8 + order
    elif kind == 'lpc':
        order = spec.get('order', 8)
        prec = spec.get('precision', 14)
        a = levinson(xs, order)
        coef, shift = quantise_lpc(a, prec, spec.get('shift'))
        res = lpc_residual(xs, coef, shift)
        if len(res) and np.max(np.abs(res)) >= (1 << 30):      # a forced shift that cannot predict: libFLAC's rule
            coef, shift = quantise_lpc(a, prec)
            res = lpc_residual(xs, coef, shift)
        header = 31 + order
        info.update(order=order, precision=prec, shift=shift)
    bw.put(0, 1)
    bw.put(header, 6)
    if w:
        bw.put(1, 1)
        bw.put_unary(w - 1)
    else:
        bw.put(0, 1)
    if kind == 'constant':
        bw.put(int(xs[0]), sbps)
    elif kind == 'verbatim':
        bw.put(xs, sbps)
    elif kind == 'fixed':
        bw.put(xs[:order], sbps)
        info['order'] = order
        info['residual'] = write_residual(bw, fixed_residual(xs, order), n, order, spec.get('residual', spec))
    else:
        bw.put(xs[:order], sbps)
        bw.put(prec - 1, 4)
        bw.put(shift, 5)
        bw.put(coef, prec)
        info['residual'] = write_residual(bw, res, n, order, spec.get('residual', spec))
    return info


# ---- frames ------------------------------------------------------------------------------------------------------
def frame_header(number, block_size, rate, channels, assignment, bits, hdr):
    """hdr: block ('code' canonical, 'byte' code 6, 'word' code 7), rate ('code', 'streaminfo', 'khz', 'hz', 'tens'),
    bits ('code' or 'streaminfo'), variable (blocking strategy)."""
    out = bytearray([0xFF, 0xF8 | (1 if hdr.get('variable') else 0)])
    bmode = hdr.get('block', 'code')
    if bmode == 'code' and block_size in BLOCK_CODES:
        bcode, bextra = BLOCK_CODES[block_size], b''
    elif bmode != 'word' and block_size <= 256:
        bcode, bextra = 6, bytes([block_size - 1])
    else:
        bcode, bextra = 7, struct.pack('>H', block_size - 1)
    rmode = hdr.get('rate', 'code')
    if rmode == 'code' and rate in RATE_CODES:
        rcode, rextra = RATE_CODES[rate], b''
    elif rmode == 'khz':
        assert rate % 1000 == 0 and rate // 1000 < 256
        rcode, rextra = 12, bytes([rate // 1000])
    elif rmode == 'hz':
        rcode, rextra = 13, struct.pack('>H', rate)
    elif rmode == 'tens':
        assert rate % 10 == 0
        rcode, rextra = 14, struct.pack('>H', rate // 10)
    else:
        rcode, rextra = 0, b''
    out.append(bcode << 4 | rcode)
    scode = BITS_CODES[bits] if hdr.get('bits', 'code') == 'code' else 0
    out.append(assignment << 4 | scode << 1)
    out += utf8_number(number) + bextra + rextra
    out.append(crc8(out))
    return bytes(out), {'block_code': bcode, 'rate_code': rcode, 'bits_code': scode,
                        'utf8_bytes': len(utf8_number(number))}


def encode_frame(x, number, rate, bits, assignment, hdr, specs, rng):
    """x: (block, channels) int64 samples.  specs: one subframe spec per channel.  Returns (bytes, info)."""
    n, ch = x.shape
    head, hinfo = frame_header(number, n, rate, ch, assignment, bits, hdr)
    if assignment < 8:
        chans, side = [x[:, c] for c in range(ch)], [False] * ch
    else:
        l, r = x[:, 0], x[:, 1]
        s = l - r
        if assignment == 8:
            chans, side = [l, s], [False, True]
        elif assignment == 9:
            chans, side = [s, r], [True, False]
        else:
            chans, side = [(l + r) >> 1, s], [False, True]
    bw = BitWriter()
    subs = []
    for c in range(ch):
        subs.append(write_subframe(bw, chans[c], bits + (1 if side[c] else 0), specs[c], rng))
        subs[-1]['side'] = side[c]
    bw.align()
    body = head + bw.tobytes()
    return body, dict(hinfo, assignment=assignment, subframes=subs, block_size=n)


def metadata(rate, channels, bits, total, min_block, max_block, extra_blocks):
    info = struct.pack('>HH', min_block, max_block) + b'\0' * 6
    packed = (rate << 44) | ((channels - 1) << 41) | ((bits - 1) << 36) | total
    info += packed.to_bytes(8, 'big') + b'\0' * 16
    blocks = [(0, info)] + list(extra_blocks)
    out = bytearray()
    for i, (kind, body) in enumerate(blocks):
        out.append((0x80 if i == len(blocks) - 1 else 0) | kind)
        out += len(body).to_bytes(3, 'big') + body
    return bytes(out)


def extra_block(kind, rng):
    if kind == 'PADDING':
        return 1, b'\0' * int(rng.integers(0, 64))
    if kind == 'APPLICATION':
        return 2, b'test' + rng.integers(0, 256, 13, dtype=np.uint8).tobytes()
    if kind == 'SEEKTABLE':
        return 3, b''.join(struct.pack('>QQH', 4096 * i, 1000 * i, 4096) for i in range(3))
    if kind == 'VORBIS_COMMENT':
        vendor = b'flac_cases'
        comments = [b'TITLE=sync \xff\xf8 inside a tag', b'ARTIST=nobody']
        body = struct.pack('<L', len(vendor)) + vendor + struct.pack('<L', len(comments))
        return 4, body + b''.join(struct.pack('<L', len(c)) + c for c in comments)
    if kind == 'PICTURE':
        mime, desc, data = b'image/png', b'cover', b'\x89PNG\xff\xf8\xff\xf9' + rng.integers(0, 256, 40, dtype=np.uint8).tobytes()
        return 6, struct.pack('>LL', 3, len(mime)) + mime + struct.pack('>L', len(desc)) + desc + \
            struct.pack('>LLLLL', 1, 1, 24, 0, len(data)) + data
    raise ValueError(kind)


def id3v2(rng):
    frame = b'TIT2' + struct.pack('>L', 6) + b'\0\0' + b'\0title'
    body = frame + b'\0' * int(rng.integers(0, 20))
    n = len(body)
    size = bytes([(n >> 21) & 0x7F, (n >> 14) & 0x7F, (n >> 7) & 0x7F, n & 0x7F])
    return b'ID3\x04\x00\x00' + size + body


# ---- cases -------------------------------------------------------------------------------------------------------
class FlacCase(object):
    """A FLAC file (bytes), the PCM it holds ((frames, channels) int64 at `bits`), where its frames are, and what the
    encoder chose for them (`frames`: one info dict per frame)."""

    def __init__(self, name, flac, pcm, rate, bits, frames, offsets, sample_rate, sample_type, corrupt=None):
        self.name, self.flac, self.pcm, self.rate, self.bits = name, flac, pcm, rate, bits
        self.frames, self.offsets = frames, offsets
        self.sample_rate, self.sample_type = sample_rate, sample_type
        self.corrupt = corrupt            # None, or (kind, frame index, byte offset, message regex)

    @property
    def channels(self):
        return self.pcm.shape[1]

    def pcm16(self):
        """What the WAV loader reads of these samples: int16, 24-bit by its top 16 bits."""
        return (self.pcm >> (self.bits - 16)).astype(np.int16)

    def wav(self):
        """The plain PCM WAV of the same samples at the same bit depth (loader_cases.riff)."""
        width = self.bits // 8
        if width == 2:
            payload = self.pcm.astype('<i2').tobytes()
        else:
            u = (self.pcm.reshape(-1) & 0xFFFFFF).astype(np.uint32)
            payload = np.stack([u & 0xFF, (u >> 8) & 0xFF, u >> 16], 1).astype(np.uint8).tobytes()
        return lc.riff(self.channels, self.rate, width, payload, len(payload))

    def write(self, directory, suffix='.flac'):
        import os
        path = os.path.join(str(directory), self.name + suffix)
        with open(path, 'wb') as f:
            f.write(self.flac)
        return path

    def write_wav(self, directory):
        import os
        path = os.path.join(str(directory), self.name + '.wav')
        with open(path, 'wb') as f:
            f.write(self.wav())
        return path

    def __repr__(self):
        return 'FlacCase(%s)' % self.name


def make_pcm(family, frames, channels, bits, rate, rng, wasted=0):
    pcm16, lo = lc.family_pcm(family, frames, channels, rng, rate)
    x = pcm16.astype(np.int64)
    if bits == 24:
        low = rng.integers(0, 256, x.shape) if lo is None else lo.astype(np.int64)
        x = (x << 8) | low
    if wasted:
        x = (x >> wasted) << wasted
    return x


def encode(pcm, rate, bits, blocks, plan, rng, hdr=None, variable=False, extra=(), id3=False, total=None,
           min_block=None, max_block=None):
    """pcm: (frames, channels) int64.  blocks: list of block sizes (summing to the frame count).  plan(i, n, rng) ->
    (assignment, [subframe spec per channel], header overrides).  Returns (bytes, frame infos, frame offsets)."""
    hdr = dict(hdr or {}, variable=variable)
    ch = pcm.shape[1]
    bodies, infos = [], []
    start = 0
    for i, n in enumerate(blocks):
        assignment, specs, hover = plan(i, n, rng)
        number = start if variable else i
        body, info = encode_frame(pcm[start:start + n], number, rate, bits, assignment, dict(hdr, **hover), specs, rng)
        bodies.append(body)
        infos.append(info)
        start += n
    assert start == len(pcm)
    crcs = crc16_many(bodies)
    frames = [b + struct.pack('>H', int(c)) for b, c in zip(bodies, crcs)]
    mb = [b for b in blocks[:-1]] or blocks or [16]
    head = (id3v2(rng) if id3 else b'') + b'fLaC' + metadata(
        rate, ch, bits, len(pcm) if total is None else total, min_block or min(mb), max_block or max(blocks or [16]),
        [extra_block(k, rng) for k in extra])
    offsets = np.cumsum([len(head)] + [len(f) for f in frames])
    return head + b''.join(frames), infos, offsets


def stereo_plan(kinds, assignments=(0, 8, 9, 10), **spec):
    def plan(i, n, rng):
        a = assignments[i % len(assignments)]
        k = kinds[i % len(kinds)]
        return (1 if a == 0 else a), [dict(spec, kind=k), dict(spec, kind=kinds[(i + 1) % len(kinds)])], {}
    return plan


def make(name, family, frames, channels, bits, rate, blocks, plan, seed, sample_rate=12000, sample_type='uint8',
         wasted=0, **kw):
    rng = np.random.default_rng([SEED, seed])
    pcm = make_pcm(family, frames, channels, bits, rate, rng, wasted)
    flac, infos, offsets = encode(pcm, rate, bits, blocks, plan, rng, **kw)
    return FlacCase(name, flac, pcm, rate, bits, infos, offsets, sample_rate, sample_type)


def fixed_blocks(frames, size):
    return [size] * (frames // size) + ([frames % size] if frames % size else [])


def uniform_plan(channels, **spec):
    def plan(i, n, rng):
        return channels - 1, [dict(spec) for _ in range(channels)], {}
    return plan


def named_cases():
    cases = []
    stypes = ('uint8', 'float32')

    def add(name, *a, **kw):
        kw.setdefault('seed', len(cases))
        kw.setdefault('sample_type', stypes[len(cases) % 2])
        cases.append(make(name, *a, **kw))

    # every LPC order, precision and shift, 24-bit full-scale audio where the 64-bit sum matters
    def lpc_sweep(i, n, rng):
        spec = dict(kind='lpc', order=i % 32 + 1, precision=i % 15 + 1, shift=(i * 7) % 16,
                    method=('rice', 'rice2')[i % 2], porder=i % 9)
        return 1, [spec, dict(spec, order=(i + 16) % 32 + 1)], {}
    for bits in (16, 24):
        add('lpc_sweep_%d' % bits, 'programme', 4096 * 48, 2, bits, 44100, fixed_blocks(4096 * 48, 4096), lpc_sweep)
    # LPC at the highest precision and shift on full-scale 24-bit samples: sums far beyond 32 bits
    def lpc_full(i, n, rng):
        spec = dict(kind='lpc', order=32, precision=15, porder_search=True, porder=8, method='rice2')
        return 0, [spec], {}
    add('lpc_full_scale_24', 'full_scale', 4608 * 3 + 77, 1, 24, 48000, fixed_blocks(4608 * 3 + 77, 4608), lpc_full)
    # every FIXED order, VERBATIM and CONSTANT, each channel assignment, wasted bits
    kinds = ['verbatim', 'fixed', 'constant', 'lpc']

    def fixed_orders(i, n, rng):
        a = (1, 8, 9, 10)[i % 4]
        specs = [dict(kind='fixed', order=(i + c) % 5, porder=(i + c) % 9, method=('rice', 'rice2')[(i // 2) % 2])
                 for c in range(2)]
        return a, specs, {}
    add('fixed_orders_16', 'programme', 1152 * 20 + 31, 2, 16, 48000, fixed_blocks(1152 * 20 + 31, 1152), fixed_orders)
    add('fixed_orders_24', 'programme', 1152 * 20 + 5, 2, 24, 96000, fixed_blocks(1152 * 20 + 5, 1152), fixed_orders)
    # full-scale stereo in every assignment: the side channel needs 17 / 25 bits
    for bits in (16, 24):
        add('full_scale_sides_%d' % bits, 'full_scale', 576 * 16, 2, bits, 32000, fixed_blocks(576 * 16, 576),
            stereo_plan(['verbatim', 'fixed', 'lpc', 'verbatim'], porder=3))
    # wasted bits: independent channels and side channels (both channels multiples of 8)
    add('wasted_bits_16', 'programme', 4608 * 6, 2, 16, 44100, fixed_blocks(4608 * 6, 4608),
        stereo_plan(['fixed', 'lpc', 'verbatim'], order=2, porder=4), wasted=3)
    add('wasted_bits_24', 'programme', 2304 * 8, 2, 24, 48000, fixed_blocks(2304 * 8, 2304),
        stereo_plan(['lpc', 'verbatim', 'fixed'], order=10, porder=5), wasted=9)
    # constant and silence, escape partitions of zero raw bits
    add('silence_escape', 'silence', 1024 * 6, 2, 16, 48000, fixed_blocks(1024 * 6, 1024),
        lambda i, n, rng: (1, [dict(kind='fixed', order=1, escape='zero'), dict(kind='constant')], {}))
    add('dc_constant_24', 'dc_pos', 512 * 9, 1, 24, 22050, fixed_blocks(512 * 9, 512),
        lambda i, n, rng: (0, [dict(kind=('constant', 'fixed')[i % 2], order=0, escape=i % 3)], {}))
    # escape partitions with n raw bits, Rice and Rice2
    add('escape_raw', 'programme', 4096 * 8, 1, 16, 16000, fixed_blocks(4096 * 8, 4096),
        lambda i, n, rng: (0, [dict(kind=('fixed', 'lpc')[i % 2], order=(3, 6)[i % 2], porder=i % 9, escape=i % 4,
                                    method=('rice', 'rice2')[i // 2 % 2])], {}))
    # every block-size code (canonical, and explicit 8- and 16-bit sizes), a short last frame
    sizes = [192, 576, 1152, 2304, 4608, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768]
    blocks = sizes + [100, 256, 4000, 65535 - 30000, 33]
    hdrs = [{}] * len(sizes) + [{'block': 'byte'}, {'block': 'byte'}, {'block': 'word'}, {'block': 'word'},
                                {'block': 'word'}]
    add('block_codes', 'programme', sum(blocks), 2, 16, 48000, blocks,
        lambda i, n, rng: (10, [dict(kind='auto', order=8), dict(kind='auto', order=12)], hdrs[i]), variable=True)
    # every sample-rate code
    for j, rate in enumerate(sorted(RATE_CODES)):
        bl = 1152 if rate < 100000 else 4608
        add('rate_%d' % rate, ('programme', 'bin_edges', 'exact_quant')[j % 3], bl * 3 + 17 * j, 1 + j % 3,
            (16, 24)[j % 2], rate, fixed_blocks(bl * 3 + 17 * j, bl), uniform_plan(1 + j % 3, kind='auto', order=8),
            hdr={'rate': 'code', 'bits': ('code', 'streaminfo')[j % 2]}, sample_rate=(12000, 8000, 24000)[j % 3])
    for mode, rate in (('streaminfo', 44100), ('khz', 12000), ('khz', 48000), ('hz', 7919), ('hz', 11025),
                       ('tens', 12010), ('tens', 44100)):
        add('rate_%s_%d' % (mode, rate), 'programme', 1000 * 5 + 3, 2, 16, rate, fixed_blocks(5003, 1000),
            uniform_plan(2, kind='auto', order=6), hdr={'rate': mode})
    # 1 to 8 channels, both depths
    for ch in range(1, 9):
        for bits in (16, 24):
            add('channels_%d_%d' % (ch, bits), ('programme', 'two_valued', 'bin_edges')[ch % 3], 4096 + 123 * ch, ch,
                bits, 44100, fixed_blocks(4096 + 123 * ch, 1024 + 512 * (ch % 3)),
                lambda i, n, rng, ch=ch: (ch - 1, [dict(kind=kinds[(i + c) % 4], order=1 + (i + c) % 4, porder=2)
                                                   for c in range(ch)], {}))
    # variable blocking with sample numbers of 1 to 5 UTF-8 bytes (past 2^21 samples)
    rng = np.random.default_rng(SEED)
    vb = [int(v) for v in rng.integers(16, 200, 12)] + [4608] * 4 + [32768] * 64 + [4321, 999]
    add('variable_utf8', 'programme', sum(vb), 1, 16, 48000, vb,
        lambda i, n, rng: (0, [dict(kind=('verbatim', 'fixed', 'lpc', 'constant')[i % 4], order=2)], {}), variable=True)
    # fixed blocking past frame 2^11: 3-byte frame numbers (4-byte ones are in the BASELINE-size file)
    add('fixed_utf8', 'programme', 192 * 2100, 1, 16, 8000, fixed_blocks(192 * 2100, 192),
        uniform_plan(1, kind='fixed', order=2), sample_rate=8000)
    # metadata: every skippable block, an ID3v2 prefix, an unknown total
    add('metadata_blocks', 'programme', 4096 * 3, 2, 16, 44100, fixed_blocks(4096 * 3, 4096),
        uniform_plan(2, kind='auto', order=8),
        extra=('SEEKTABLE', 'VORBIS_COMMENT', 'PADDING', 'PICTURE', 'APPLICATION'))
    add('id3_prefix_total_unknown', 'programme', 4096 * 3 + 9, 2, 24, 48000, fixed_blocks(4096 * 3 + 9, 4096),
        uniform_plan(2, kind='auto', order=12), id3=True, total=0, extra=('VORBIS_COMMENT', 'PADDING'))
    # the value families of the median selector
    for i, fam in enumerate(lc.FAMILIES):
        for bits in (16, 24):
            add('family_%s_%d' % (fam, bits), fam, 48000 + 101 * i, 1 + (i + bits) % 3, bits, (44100, 48000)[i % 2],
                fixed_blocks(48000 + 101 * i, 4096), uniform_plan(1 + (i + bits) % 3, kind='auto', order=8))
    # an empty stream: metadata and no frames
    add('empty', 'programme', 0, 2, 16, 48000, [], uniform_plan(2))
    return cases


@functools.lru_cache(maxsize=None)
def corrupt_cases():
    """(case, kind, frame, byte offset, message regex): the same file damaged in one way each."""
    base = make('corrupt_base', 'programme', 4096 * 10 + 500, 2, 16, 44100, fixed_blocks(4096 * 10 + 500, 4096),
                stereo_plan(['verbatim', 'lpc', 'fixed'], assignments=(0, 10), order=8, porder=4), seed=999)
    off = [int(o) for o in base.offsets]
    out = []

    def damaged(kind, data, frame, where, regex, total=None):
        c = FlacCase('corrupt_' + kind, data, base.pcm, base.rate, base.bits, base.frames, base.offsets,
                     base.sample_rate, base.sample_type, corrupt=(kind, frame, where, regex))
        out.append(c)

    f = bytearray(base.flac)
    k = 4
    hdr_len = len(frame_header(k, 4096, base.rate, 2, 1 if k % 2 == 0 else 10, 16, {})[0])
    f[off[k] + hdr_len - 1] ^= 0x5A                                 # the header's CRC-8 byte
    damaged('crc8', bytes(f), k, off[k], 'frame %d at byte offset %d: frame header CRC-8 mismatch' % (k, off[k]))
    f = bytearray(base.flac)
    k = 6                                                          # a VERBATIM channel 0 (independent stereo)
    assert base.frames[k]['subframes'][0]['kind'] == 'verbatim'
    f[off[k] + 100] ^= 0x10
    damaged('crc16', bytes(f), k, off[k], 'frame %d at byte offset %d: frame CRC-16 mismatch' % (k, off[k]))
    k = 3
    damaged('gap', base.flac[:off[k + 1]] + b'\0\0\0' + base.flac[off[k + 1]:], k, off[k],
            'frame %d at byte offset %d: frame does not end where the next frame starts' % (k, off[k]))
    k = len(base.frames) - 1
    damaged('truncated', base.flac[:off[k] + (off[k + 1] - off[k]) // 2], k, off[k],
            'frame %d at byte offset %d: truncated frame' % (k, off[k]))
    k = len(base.frames) - 1
    damaged('truncated_header', base.flac[:off[k] + 3], k, off[k], 'frame %d at byte offset %d: truncated frame' % (k, off[k]))
    # STREAMINFO total one more than the frames hold (the 36-bit field ends at byte 8 + 18 of the file)
    f = bytearray(base.flac)
    tot = int.from_bytes(f[8 + 13:8 + 18], 'big')
    f[8 + 13:8 + 18] = (tot + 1).to_bytes(5, 'big')
    damaged('total', bytes(f), None, None, 'STREAMINFO says %d samples, the frames hold %d' % (len(base.pcm) + 1, len(base.pcm)))
    return base, out


def unsupported_bits_case():
    """A 20-bit file: valid FLAC, refused by the loader."""
    rng = np.random.default_rng([SEED, 77])
    pcm = make_pcm('programme', 4096, 2, 24, 44100, rng) >> 4
    flac, infos, offsets = encode(pcm, 44100, 20, [4096], uniform_plan(2, kind='auto', order=8), rng)
    return FlacCase('bits20', flac, pcm, 44100, 20, infos, offsets, 12000, 'uint8')


@functools.lru_cache(maxsize=None)
def all_cases():
    cases = named_cases()
    names = [c.name for c in cases]
    assert len(set(names)) == len(names)
    assert_coverage(cases)
    return cases


def assert_coverage(cases):
    subs = [s for c in cases for f in c.frames for s in f['subframes']]
    kinds = {s['kind'] for s in subs}
    assert kinds >= set(SUBFRAME_KINDS), kinds
    assert {s['order'] for s in subs if s['kind'] == 'fixed'} == set(range(5))
    lpc = [s for s in subs if s['kind'] == 'lpc']
    assert {s['order'] for s in lpc} == set(range(1, 33))
    assert {s['precision'] for s in lpc} == set(range(1, 16))
    assert {s['shift'] for s in lpc} == set(range(16))
    assert any(s['wasted'] and not s['side'] for s in subs) and any(s['wasted'] and s['side'] for s in subs)
    res = [s['residual'] for s in subs if 'residual' in s]
    assert {r['method'] for r in res} == {'rice', 'rice2'}
    assert {r['porder'] for r in res} >= set(range(9))
    esc = set().union(*[r['escape'] for r in res])
    assert 0 in esc and any(e > 0 for e in esc)
    frames = [f for c in cases for f in c.frames]
    assert {f['assignment'] for f in frames} >= {1, 8, 9, 10}
    assert any(s['side'] and s['bps'] == 17 for s in subs) and any(s['side'] and s['bps'] == 25 for s in subs)
    assert {f['block_code'] for f in frames} == set(range(1, 16))
    assert {f['rate_code'] for f in frames} == set(range(0, 15))
    assert {f['bits_code'] for f in frames} >= {0, 4, 6}
    assert {f['utf8_bytes'] for f in frames} >= {1, 2, 3, 5}
    assert {c.bits for c in cases} == {16, 24}
    assert {c.channels for c in cases} == set(range(1, 9))
    assert {c.sample_rate for c in cases} == set(lc.OUT_RATES)
    assert {c.sample_type for c in cases} == {'uint8', 'float32'}
    assert any(c.flac.startswith(b'ID3') for c in cases)
    # a short last frame under fixed blocking
    assert any(len({f['block_size'] for f in c.frames[:-1]}) == 1 and c.frames[-1]['block_size'] < c.frames[0]['block_size']
               for c in cases if len(c.frames) > 1)


# ---- the BASELINE-size file --------------------------------------------------------------------------------------
BASELINE_RATE, BASELINE_BLOCK, BASELINE_FRAMES, BASELINE_TAIL = 48000, 1152, 225000, 500
BASELINE_PERIOD = 4096            # distinct frame payloads: the PCM repeats every 4096 frames (98.3 s)


def periodic_file(n_frames, tail, bits, coded, seed, rate=48000, block=1152, period=4096, spec=None, parts=False):
    """A long stereo file cheaply: the PCM repeats every `period` frames of `block` samples, so only that many frame
    payloads are built; headers and CRC-16s are per frame (the CRCs vectorised across frames).  coded(j) -> None for a
    VERBATIM frame (byte-swapped samples behind a subframe header byte), or the channel assignment (1 or 10) of a
    frame whose subframes write_subframe codes with `spec`.  A last frame of `tail` samples follows.
    Returns (file bytes, PCM (frames, 2) int64)."""
    rng = np.random.default_rng([SEED, seed])
    spec = spec or dict(kind='lpc', order=8, precision=12, porder=4)
    width = bits // 8
    base = make_pcm('programme', period * block, 2, bits, rate, rng)
    blocks = base.reshape(period, block, 2)
    # verbatim payloads: per channel 0x02 (VERBATIM, no wasted bits) then the big-endian samples
    be = np.stack([(blocks >> (8 * (width - 1 - b))) & 0xFF for b in range(width)], -1).astype(np.uint8)
    be = be.transpose(0, 2, 1, 3).reshape(period, 2, block * width)
    verb = np.concatenate([np.full((period, 2, 1), 2, np.uint8), be], axis=2).reshape(period, -1)
    payloads, assign = [], np.ones(period, np.int64)
    for j in range(period):
        a = coded(j)
        if a is None:
            payloads.append(verb[j].tobytes())
            continue
        assign[j] = a
        x = blocks[j]
        if a == 10:
            chans, bps = [(x[:, 0] + x[:, 1]) >> 1, x[:, 0] - x[:, 1]], [bits, bits + 1]
        else:
            chans, bps = [x[:, 0], x[:, 1]], [bits, bits]
        bw = BitWriter()
        for c in range(2):
            write_subframe(bw, chans[c], bps[c], spec, rng)
        bw.align()
        payloads.append(bw.tobytes())
    frames = []
    for i in range(n_frames):
        j = i % period
        head, _ = frame_header(i, block, rate, 2, int(assign[j]), bits, {})
        frames.append(head + payloads[j])
    tail_pcm = make_pcm('programme', tail, 2, bits, rate, rng)
    body, _ = encode_frame(tail_pcm, n_frames, rate, bits, 10, {}, [dict(spec), dict(kind='fixed', order=2)], rng)
    frames.append(body)
    crcs = []
    for a in range(0, len(frames), 16384):
        crcs += crc16_many(frames[a:a + 16384])
    head = b'fLaC' + metadata(rate, 2, bits, n_frames * block + tail, block, block,
                              [extra_block('SEEKTABLE', rng), extra_block('PADDING', rng)])
    data = head + b''.join(f + struct.pack('>H', int(c)) for f, c in zip(frames, crcs))
    if parts:
        return data, base, tail_pcm
    pcm = np.concatenate([np.tile(base, (n_frames // period, 1)), base[:(n_frames % period) * block], tail_pcm])
    return data, pcm


def baseline_file(seed=7):
    """A 90-minute, 48 kHz, stereo, 16-bit file of 225 000 frames of 1152 samples and a short last frame of 500:
    about 1 GB, so bit positions pass 2^32, and frame numbers take 4 UTF-8 bytes.  Most frames are VERBATIM; every
    16th is LPC order 8 with Rice partitions, every 64th of those mid/side (periodic_file).
    Returns (file bytes, PCM (frames, 2) int16)."""
    data, pcm = periodic_file(BASELINE_FRAMES, BASELINE_TAIL, 16, lambda j: None if j % 16 else (10 if j % 64 == 0 else 1),
                              seed, BASELINE_RATE, BASELINE_BLOCK, BASELINE_PERIOD)
    return data, pcm.astype(np.int16)
