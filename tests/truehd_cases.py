"""Seeded NumPy writer of Dolby TrueHD streams for the tests (test infrastructure, in the style of flac_cases.py).

A stream is a run of access units (AUs).  Each AU holds `samples per AU` samples (40 << rate code), an optional major
sync, a substream directory and the substreams' data; a restart segment is a major-sync AU in which every substream
opens with a restart header, and the AUs after it up to the next one.  The writer encodes a given PCM losslessly with
the coding tools the decoder has to handle:

* 1-8 channels in 1, 2 or 3 decoded substreams, plus a fourth (object) substream of filler that is only skipped;
* Huffman codebooks 0-3 with Huffman offsets and raw LSBs, quant step sizes and output shifts;
* FIR orders 0-8 and IIR orders 0-4 with filter shifts, coefficient precisions and transmitted IIR state;
* primitive matrices with fractional coefficients, LSB bypass and the LFSR noise channels of noise type 0;
* block sizes that change inside a segment, blocks that omit their parameters, restart intervals of 1-128 AUs;
* the end-of-stream marker with a short last AU, and substream parity / CRC bytes.

The values decoded from a stream are int32 samples in a 24-bit frame (FFmpeg returns them as S32 shifted up by 8);
`pcm` holds them, and `pcm16` the top 16 bits the loader reads.  Each segment is written so that no prediction reaches
back past its restart (the first block after a restart is unfiltered and at least 8 samples long), so a decoder that
starts a segment from zero filter history decodes it exactly."""
import os

import numpy as np

SEED = 20261016
SYNC = b'\xf8\x72\x6f\xba'
RATE_CODES = {48000: 0, 96000: 1, 192000: 2, 44100: 8, 88200: 9, 176400: 10}

# Huffman tables: (code, length) per symbol
_HEAD = [(1, 9 - i) for i in range(7)]
_TAIL = [(3, 3), (5, 4), (9, 5), (0x11, 6), (0x21, 7), (0x41, 8), (0x81, 9)]
HUFF = [_HEAD + [(4, 3), (5, 3), (6, 3), (7, 3)] + _TAIL, _HEAD + [(2, 2), (3, 2)] + _TAIL, _HEAD + [(1, 1)] + _TAIL]

# channel layouts: thd_layout bit -> FFmpeg channel bits; the order in which restart headers count channels
THD_LAYOUT = [(0, 1), (2,), (3,), (9, 10), (12, 14), (6, 7), (4, 5), (8,), (11,), (33, 34), (31, 32), (13,), (35,)]
THD_ORDER = [0, 1, 2, 3, 9, 10, 12, 14, 6, 7, 4, 5, 8, 11, 33, 34, 31, 32, 13, 35]
# an arrangement of the 5-bit stream-1 field (at most 8 channels) per channel count
ARRANGE1 = {1: 0b00010, 2: 0b00001, 3: 0b00011, 4: 0b01001, 5: 0b01011, 6: 0b01111, 7: 0b11011, 8: 0b11111}
# 13-bit stream-2 arrangements (7.1 with back surrounds, 6.1 with a back centre, ...)
ARRANGE2 = {6: 0b0000000001111, 7: 0b0000010001111, 8: 0b0000001001111, 5: 0b0000001000011, 4: 0b0000001000001}


def layout_bits(arrangement):
    return sorted(b for i, bits in enumerate(THD_LAYOUT) if arrangement >> i & 1 for b in bits)


def channel_codes(arrangement):
    """code k of a restart header's channel assignment -> output channel (FFmpeg's native order of the layout)"""
    native = layout_bits(arrangement)
    return [native.index(b) for b in THD_ORDER if b in native]


# ---- bits and checks -----------------------------------------------------------------------------------------------
class Bits(object):
    def __init__(self):
        self.parts = []
        self.n = 0

    def put(self, nbits, v):
        if nbits:
            self.parts.append(format(int(v) & ((1 << nbits) - 1), '0%db' % nbits))
            self.n += nbits

    def align(self, k):
        self.put((-self.n) % k, 0)

    def tobytes(self):
        s = ''.join(self.parts)
        s += '0' * ((-len(s)) % 8)
        return int(s, 2).to_bytes(len(s) // 8, 'big') if s else b''


def _crc_table(poly, bits):
    top, mask = 1 << (bits - 1), (1 << bits) - 1
    out = []
    for i in range(256):
        c = i << (bits - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
        out.append(c)
    return out


CRC_1D, CRC_63, CRC_2D = _crc_table(0x1D, 8), _crc_table(0x63, 8), _crc_table(0x2D, 16)


def parity(data):
    p = 0
    for b in data:
        p ^= b
    return p


def checksum8(data):
    """substream check byte over data (the bytes before the parity / check pair)"""
    c = 0x3C
    for b in data[:-1]:
        c = CRC_63[c ^ b]
    return c ^ data[-1]


def checksum16(data):
    """major sync check word over data (its first 26 bytes), as the big-endian value of bytes 26-27"""
    c = 0
    for b in data[:-2]:
        c = ((c << 8) & 0xFFFF) ^ CRC_2D[(c >> 8) ^ b]
    return c ^ (data[-2] << 8 | data[-1])


def restart_checksum(buf, bit_size):
    """check byte of a restart header: `buf` is the substream data from its start, the header ends bit_size bits after
    bit 2 (the two flag bits in front of it are left out)"""
    nb = (bit_size + 2) // 8
    crc = CRC_1D[buf[0] & 0x3F]
    for b in buf[1:nb - 1]:
        crc = CRC_1D[crc ^ b]
    crc ^= buf[nb - 1]
    for i in range((bit_size + 2) & 7):
        crc <<= 1
        if crc & 0x100:
            crc ^= 0x11D
        crc ^= (buf[nb] >> (7 - i)) & 1
    return crc & 0xFF


def xor8(v):
    v ^= v >> 16
    v ^= v >> 8
    return v & 0xFF


def major_sync(rate, n_sub, arr1, arr2):
    b = Bits()
    b.put(32, 0xF8726FBA)
    b.put(4, RATE_CODES[rate]); b.put(4, 0)
    b.put(2, 0); b.put(2, 0); b.put(5, arr1); b.put(2, 0); b.put(13, arr2)
    b.put(16, 0xB752); b.put(16, 0); b.put(16, 0)
    b.put(1, 1); b.put(15, 0x7FFF)
    b.put(4, n_sub); b.put(4, 0)
    b.put(8, 0); b.put(64, 0)
    d = bytearray(b.tobytes())
    c = checksum16(bytes(d))
    return bytes(d) + bytes([c >> 8, c & 0xFF])


# ---- the encoder --------------------------------------------------------------------------------------------------
class Channel(object):
    """What a decoder keeps per channel: filters (order, shift, coefficients), their history, the Huffman coding."""

    def __init__(self):
        self.fir, self.iir = [0, 0, []], [0, 0, []]
        self.fir_hist, self.iir_hist = [0] * 8, [0] * 4              # most recent first
        self.huff_offset, self.codebook, self.huff_lsbs = 0, 0, 24

    def reset(self):
        self.fir[0] = self.iir[0] = self.fir[1] = self.iir[1] = 0
        self.huff_offset, self.codebook, self.huff_lsbs = 0, 0, 24

    def copy(self):
        c = Channel()
        c.fir, c.iir = list(self.fir), list(self.iir)
        c.fir_hist, c.iir_hist = list(self.fir_hist), list(self.iir_hist)
        c.huff_offset, c.codebook, c.huff_lsbs = self.huff_offset, self.codebook, self.huff_lsbs
        return c


def sign_huff_offset(cb, lsb, ho):
    shift = lsb + (2 - cb if cb else -1)
    return ho - ((7 << lsb) if cb else 0) - ((1 << shift) if shift >= 0 else 0)


def fits(R, cb, lsb, ho):
    u = R - sign_huff_offset(cb, lsb, ho)
    top = (len(HUFF[cb - 1]) << lsb) if cb else (1 << lsb)
    return u.min() >= 0 and u.max() < top


def filter_residuals(ch, q, block):
    """Residuals (in quant steps) that make channel ch's filters reproduce `block`; returns them and the new history"""
    mask = ~((1 << q) - 1)
    fo, io, shift = ch.fir[0], ch.iir[0], ch.fir[1]
    fc, ic = ch.fir[2], ch.iir[2]
    fh, ih = list(ch.fir_hist), list(ch.iir_hist)
    if not fo and not io:                             # no prediction: the residuals are the samples
        assert not np.any(block & ~mask), 'quant step leaves low bits'
        vals = block.tolist()
        tail = (vals[::-1] + fh)[:8]
        return block >> q, tail, (vals[::-1] + ih)[:4]
    out = []
    for v in block.tolist():
        acc = 0
        for k in range(fo):
            acc += fh[k] * fc[k]
        for k in range(io):
            acc += ih[k] * ic[k]
        acc >>= shift
        r = v - (acc & mask)
        assert r & ~mask == 0, 'quant step leaves low bits'
        out.append(r >> q)
        fh.insert(0, v); fh.pop()
        d = (v - acc + (1 << 31)) % (1 << 32) - (1 << 31)
        ih.insert(0, d); ih.pop()
    return np.array(out, np.int64), fh, ih


def noise_pair(seed, n, shift):
    """The two noise channels of noise type 0 for n samples, and the seed after them."""
    a, b = np.zeros(n, np.int64), np.zeros(n, np.int64)
    for i in range(n):
        s7 = (seed >> 7) & 0xFFFF
        a[i] = (((seed >> 15) & 0xFF) ^ 0x80) - 0x80
        b[i] = ((s7 & 0xFF) ^ 0x80) - 0x80
        seed = ((seed << 16) ^ s7 ^ (s7 << 5)) & 0xFFFFFFFF
    return a << shift, b << shift, seed


class Substream(object):
    """Encoder of one substream: channels 0..n-1, all of them matrix channels (min channel 0)."""

    def __init__(self, n, codes, style):
        self.n, self.codes, self.style = n, codes, style
        self.ch = [Channel() for _ in range(n)]
        self.check = 0xFFFFFFFF

    def restart(self, rng, noise_type):
        self.noise_type = noise_type
        self.noise_shift = int(rng.integers(0, 4)) if self.style.get('matrix') else 0
        self.seed = int(rng.integers(0, 1 << 23))
        self.presence, self.blocksize = 0xFF, 8
        self.matrices, self.out_shift, self.quant = [], [0] * self.n, [0] * self.n
        for c in self.ch:
            c.reset()
        self.known = [0] * self.n                     # samples of history decoded since the restart, per channel
        self.perm = [int(v) for v in rng.permutation(self.n)] if self.style.get('permute', True) else list(range(self.n))

    def restart_header(self, b, check_byte):
        start = b.n
        b.put(13, 0x31EA >> 1); b.put(1, self.noise_type)
        b.put(16, 0)
        b.put(4, 0); b.put(4, self.n - 1); b.put(4, self.n - 1)
        b.put(4, self.noise_shift); b.put(23, self.seed)
        b.put(19, 0); b.put(1, 0); b.put(8, check_byte); b.put(16, 0)
        inv = [0] * self.n
        for out_ch, mat in enumerate(self.perm):
            inv[mat] = out_ch
        for mat in range(self.n):
            b.put(6, self.codes.index(inv[mat]))
        b.put(8, restart_checksum(b.tobytes(), b.n - start))


class Writer(object):
    def __init__(self, rate, pcm, bits, n_sub=1, arr2=None, seed=0, style=None, restarts=(16,), eos_short=0,
                 objects=False, parity=True, bad_check=None, false_sync=False, short_at=None, first_check=None):
        self.bad_check, self.false_sync, self.short_at = bad_check, false_sync, short_at
        self.first_check = first_check
        self.rate, self.bits = rate, bits
        self.spa = 40 << (RATE_CODES[rate] & 7)
        self.pcm = np.asarray(pcm, np.int64)
        self.nch = self.pcm.shape[1]
        self.n_sub = n_sub + (1 if objects else 0)
        self.objects, self.parity = objects, parity
        self.rng = np.random.default_rng(seed)
        self.style = dict(style or {})
        self.restarts, self.eos_short = list(restarts), eos_short
        self.used = {'codebooks': set(), 'lsbs': set(), 'fir': set(), 'iir': set(), 'iir_state': 0, 'matrices': set(),
                     'bypass': 0, 'frac': set(), 'quant': set(), 'shift': set(), 'blocks': set(), 'omitted': 0,
                     'noise': 0, 'huff_offset': 0, 'presence': set()}
        # the top decoded substream carries the output in the layout of the 13-bit field (stream 2); below it sit a
        # stereo substream and, in three-substream files, one in the layout of the 5-bit field (stream 1)
        out = arr2 if arr2 is not None else (ARRANGE2[self.nch] if n_sub == 3 else ARRANGE1[self.nch])
        assert n_sub > 1 or self.nch <= 2, 'a single substream carries at most 2 channels'
        self.arr2 = out
        self.arr1 = ARRANGE1[6] if n_sub == 3 else ARRANGE1[self.nch]
        masks = [0b1, self.arr1, out][3 - n_sub:] if n_sub > 1 else [out]
        if n_sub == 2:
            masks = [0b1, out]
        self.subs = [Substream(len(layout_bits(m)), channel_codes(m), self.style if k == len(masks) - 1 else {'permute': False})
                     for k, m in enumerate(masks)]
        self.top = self.subs[-1]
        assert self.top.n == self.nch

    def encode(self):
        n_frames, spa = len(self.pcm), self.spa
        n_au = -(-n_frames // spa)
        short = n_au * spa - n_frames
        assert short == self.eos_short, (short, self.eos_short)
        starts, a, k = [], 0, 0
        while a < n_au:
            starts.append(a)
            a += self.restarts[k % len(self.restarts)]
            k += 1
        seg = set(starts)
        out, offsets = bytearray(), []
        self.sub_starts, self.sub_lens = [], []
        for au in range(n_au):
            restart, last = au in seg, au == n_au - 1
            self._segment = starts.index(au) if restart else self._segment
            self._au_index = au
            nsamp = spa - (short if last else 0)
            target = np.zeros((spa, self.nch), np.int64)
            target[:nsamp] = self.pcm[au * spa: au * spa + nsamp]
            datas = []
            for s in self.subs:
                t = target if s is self.top else np.ascontiguousarray(np.pad(target, ((0, 0), (0, max(0, s.n - self.nch))))[:, :s.n])
                datas.append(self._substream(s, t, restart, last, short, nsamp))
            if self.objects:
                filler = bytes(self.rng.integers(0, 256, 2 * int(self.rng.integers(4, 40)), dtype=np.uint8))
                if self.false_sync and au % 5 == 2:
                    # an AU header and a major sync with a valid CRC inside data the decoder skips
                    filler = b'\x40\x20\x00\x00' + major_sync(self.rate, self.n_sub, self.arr1, self.arr2) + filler
                    self.used['false_syncs'] = self.used.get('false_syncs', 0) + 1
                datas.append(filler)
            offsets.append(len(out))
            au_bytes = self._au(datas, restart, au)
            head = len(au_bytes) - sum(len(d) for d in datas)
            self.sub_starts.append([len(out) + head + sum(len(d) for d in datas[:k]) for k in range(len(datas))])
            self.sub_lens.append([len(d) for d in datas])
            out += au_bytes
        self.au_offsets, self.seg_starts = offsets, starts
        return bytes(out)

    def _au(self, datas, restart, au):
        ms = major_sync(self.rate, self.n_sub, self.arr1, self.arr2) if restart else b''
        dirb, end = bytearray(), 0
        for k, d in enumerate(datas):
            assert len(d) % 2 == 0
            end += len(d) // 2
            w = ((0 if restart else 1) << 14) | ((1 if (self.parity and k < len(self.subs)) else 0) << 13) | end
            dirb += bytes([w >> 8, w & 0xFF])
        length = 4 + len(ms) + len(dirb) + sum(len(d) for d in datas)
        assert length % 2 == 0 and length // 2 < 4096, length
        head = bytearray([(length // 2) >> 8, (length // 2) & 0xFF, (au * 7 >> 8) & 0xFF, (au * 7) & 0xFF])
        p = parity(head) ^ parity(dirb)
        head[0] |= ((0xF ^ (p >> 4) ^ p) & 0xF) << 4
        return bytes(head) + ms + bytes(dirb) + b''.join(datas)

    # -- one substream of one AU
    def _substream(self, s, target, restart, last, short, nsamp):
        rng, spa, top = self.rng, self.spa, s is self.top
        b = Bits()
        check_byte = xor8(s.check) if s.check != 0xFFFFFFFF else int(rng.integers(0, 256))
        if top and s.check == 0xFFFFFFFF and self.first_check is not None:
            check_byte = self.first_check
        if restart and top and self.bad_check is not None and self._segment == self.bad_check:
            check_byte ^= 0x5A
        new_matrix = new_shift = None
        if restart:
            s.restart(rng, 1 if s.n > 6 else 0)
            s.check = 0
            if top and s.style.get('matrix'):
                new_matrix = self._matrices(s)
            if top and s.style.get('shift'):
                lim = 8 if self.bits == 16 else 1
                new_shift = [int(rng.integers(0, lim)) if rng.random() < 0.7 else 0 for _ in range(s.n)]
                self.used['shift'].update(new_shift)
        s.changes = {}                                   # filter changes in this AU: at most 2 per channel and filter
        mats = new_matrix if new_matrix is not None else s.matrices
        shifts = new_shift if new_shift is not None else s.out_shift
        final, pre, bypass, mats = self._invert_output(s, target, nsamp, mats, shifts)
        if new_matrix is not None:
            new_matrix = mats
            self.used['matrices'].add(len(mats))
            self.used['bypass'] += sum(m['bypass'] for m in mats)
            self.used['frac'].update(m['frac'] for m in mats)
        sizes = [spa]
        if top and self._au_index == self.short_at:
            sizes = [spa - 8]                                   # an AU 8 samples short, with no end-of-stream marker
        elif top and s.style.get('blocks'):
            sizes, rem = [], spa
            while rem:
                bs = rem if rem < 16 else int(rng.integers(8, min(64, rem - 8) + 1))
                sizes.append(bs)
                rem -= bs
        pos = 0
        for k, bs in enumerate(sizes):
            blk = pre[pos:pos + bs]
            p = self._params(s, bs, restart and k == 0, new_matrix if k == 0 else None, new_shift if k == 0 else None, blk)
            self._write_block(b, s, p, blk, bypass[pos:pos + bs], restart and k == 0, check_byte)
            if top:
                self.used['blocks'].add(bs)
            pos += bs
            b.put(1, k == len(sizes) - 1)
        b.align(16)
        if last and short:
            b.put(16, 0xD234); b.put(16, 0x2000 | short)
        data = b.tobytes()
        if self.parity:
            data += bytes([parity(data) ^ 0xA9, checksum8(data)])
        if top:
            x = 0
            for mat in range(s.n):
                v = ((final[:nsamp, mat] << s.out_shift[mat]) & 0xFFFFFF) << mat
                x ^= int(np.bitwise_xor.reduce(v)) if nsamp else 0
            s.check ^= x & 0xFFFFFFFF
            if s.noise_type == 0:
                s.seed = noise_pair(s.seed, nsamp, 0)[2]
        if last and short:
            s.check = 0xFFFFFFFF
        return data

    def _matrices(self, s):
        rng, n = self.rng, s.n
        nsrc = n + (2 if s.noise_type == 0 else 0)
        mats = []
        for _ in range(int(rng.integers(1, 5))):
            d, frac = int(rng.integers(0, n)), int(rng.integers(0, 15))
            coeff = [0] * nsrc
            coeff[d] = 1 << frac
            # off-diagonal terms add up to at most a quarter, so a chain of matrices keeps the channels in 24 bits
            others = [c for c in range(nsrc) if c != d and rng.random() < (0.6 if c < n else 0.5)]
            lim = (1 << frac) // (4 * max(len(others), 1))
            for c in others:
                coeff[c] = int(rng.integers(-lim, lim + 1)) if lim else 0
            mats.append({'out': d, 'frac': frac, 'bypass': bool(rng.random() < 0.5), 'coeff': coeff})
        if s.noise_type == 0 and any(any(m['coeff'][n:]) for m in mats):
            self.used['noise'] += 1
        return mats

    def _invert_output(self, s, target, nsamp, mats, shifts):
        """Matrix-channel values that give `target` at the output after the AU's matrices and output shifts"""
        rng, n, spa = self.rng, s.n, self.spa
        final = np.zeros((spa, n), np.int64)
        for out_ch in range(n):
            mat = s.perm[out_ch]
            assert not np.any(target[:, out_ch] & ((1 << shifts[mat]) - 1))
            final[:, mat] = target[:, out_ch] >> shifts[mat]
        cur = final.copy()
        noise = np.zeros((spa, 2), np.int64)
        if s.noise_type == 0:
            a, b, _ = noise_pair(s.seed, nsamp, s.noise_shift)
            noise[:nsamp, 0], noise[:nsamp, 1] = a, b
        bypass = np.zeros((spa, 8), np.int64)
        for m in range(len(mats) - 1, -1, -1):
            mt, x = mats[m], np.zeros(spa, np.int64)
            d, sh = mt['out'], 14 - mt['frac']
            for c in range(n):
                if c != d:
                    x += cur[:, c] * (mt['coeff'][c] << sh)
            if s.noise_type == 0:
                x += noise[:, 0] * (mt['coeff'][n] << sh) + noise[:, 1] * (mt['coeff'][n + 1] << sh)
            if mt['bypass']:
                bypass[:nsamp, m] = rng.integers(0, 2, nsamp)
            cur[:, d] = cur[:, d] - bypass[:, m] - (x >> 14)
        if mats and np.abs(cur).max() >= 1 << (23 if mats is s.matrices else 22):
            assert mats is not s.matrices, 'matrix-channel values leave 24 bits inside a segment'
            return self._invert_output(s, target, nsamp, [], shifts)
        return final, cur, bypass, mats

    # -- the parameters of one block
    def _params(self, s, bs, restart, new_matrix, new_shift, blk):
        rng, top = self.rng, s is self.top
        st = s.style if top else {}
        need = restart or bs != s.blocksize
        if not need and st.get('omit') and rng.random() < 0.4:
            if all(self._codes_as_is(s, c, blk[:, c]) for c in range(s.n)):
                self.used['omitted'] += 1
                return None
        p = {'presence': None, 'blocksize': bs if bs != s.blocksize else None, 'matrix': new_matrix,
             'shift': new_shift, 'quant': None}
        presence = s.presence
        if top and not restart and presence & 1 and rng.random() < 0.15:
            presence = p['presence'] = int(rng.choice([0xFF, 0xFE, 0xBE, 0xFA]))
            self.used['presence'].add(presence)
        quant = s.quant
        if top and st.get('quant') and presence & 0x10 and rng.random() < (0.5 if restart else 0.2):
            mats = new_matrix if new_matrix is not None else s.matrices
            shifts = new_shift if new_shift is not None else s.out_shift
            dest = {m['out'] for m in mats}
            quant = p['quant'] = [0 if (c in dest or self.bits == 24) else int(rng.integers(0, 9 - shifts[c]))
                                  for c in range(s.n)]
            self.used['quant'].update(quant)
        p['chans'] = []
        for c in range(s.n):
            send = p['quant'] is not None or (rng.random() < 0.9 if restart else rng.random() < 0.5) or \
                not self._codes_as_is(s, c, blk[:, c], quant[c])
            p['chans'].append(self._channel(s, c, blk[:, c], quant[c], presence, st) if (send and (top or restart)) or
                              (send and not self._codes_as_is(s, c, blk[:, c], quant[c])) else None)
        return p

    def _codes_as_is(self, s, c, col, q=None):
        ch = s.ch[c]
        q = s.quant[c] if q is None else q
        if ch.huff_lsbs < q:
            return False
        try:
            R = filter_residuals(ch, q, col)[0]
        except AssertionError:
            return False
        return fits(R, ch.codebook, ch.huff_lsbs - q, ch.huff_offset)

    def _filter(self, order, shift, iir, state):
        rng = self.rng
        if not order:
            return {'order': 0}
        cbits = int(rng.integers(1, 17))
        cshift = int(rng.integers(0, min(7, 16 - cbits) + 1))
        budget = (1 << shift) // (2 * order) if iir else (1 << shift) // order
        lim = min((1 << (cbits - 1)) - 1, budget >> cshift)
        f = {'order': order, 'shift': shift, 'cbits': cbits, 'cshift': cshift,
             'coeffs': [int(rng.integers(-lim, lim + 1)) if lim > 0 else 0 for _ in range(order)], 'state': None}
        if state:
            sbits, sshift = int(rng.integers(0, 12)), int(rng.integers(0, 5))
            half = 1 << max(sbits - 1, 0)
            f['state'] = (sbits, sshift, [int(rng.integers(-half, half)) if sbits else 0 for _ in range(order)])
        return f

    @staticmethod
    def _apply_filter(ch, f, iir):
        fp = ch.iir if iir else ch.fir
        fp[0] = f['order']
        if f['order']:
            fp[1], fp[2] = f['shift'], [v << f['cshift'] for v in f['coeffs']]
            if f.get('state'):
                sbits, sshift, vals = f['state']
                for i, v in enumerate(vals):
                    ch.iir_hist[i] = v << sshift

    def _channel(self, s, c, col, q, presence, st):
        """Channel c's parameters for a block: filters (none reaching back past the restart) and the coding"""
        rng = self.rng
        known = s.known[c]
        for attempt in range(2):
            trial = s.ch[c].copy()
            out = {'fir': None, 'iir': None, 'ho': None}
            if st.get('filters') and attempt == 0:
                if presence & 0x08 and s.changes.get((c, 'fir'), 0) < 2 and rng.random() < 0.7:
                    order = int(rng.integers(0, max(0, min(8 - trial.iir[0], known)) + 1))
                    shift = trial.iir[1] if trial.iir[0] and order else int(rng.integers(0, 15))
                    out['fir'] = self._filter(order, shift, False, False)
                    self._apply_filter(trial, out['fir'], False)
                if presence & 0x04 and s.changes.get((c, 'iir'), 0) < 2 and rng.random() < 0.6:
                    give = rng.random() < 0.4
                    room = min(4, 8 - trial.fir[0])
                    order = int(rng.integers(0, (room if give else max(0, min(room, known))) + 1))
                    shift = trial.fir[1] if trial.fir[0] and order else int(rng.integers(0, 15))
                    out['iir'] = self._filter(order, shift, True, give and order > 0)
                    self._apply_filter(trial, out['iir'], True)
            elif attempt == 1:                                 # the filters would not code: switch them off
                if presence & 0x08 and trial.fir[0] and s.changes.get((c, 'fir'), 0) < 2:
                    out['fir'] = {'order': 0}
                    self._apply_filter(trial, out['fir'], False)
                if presence & 0x04 and trial.iir[0] and s.changes.get((c, 'iir'), 0) < 2:
                    out['iir'] = {'order': 0}
                    self._apply_filter(trial, out['iir'], True)
            if not trial.fir[0] and trial.iir[0]:
                trial.fir[1] = trial.iir[1]
            R = filter_residuals(trial, q, col)[0]
            mid = max(-16384, min(16383, int((int(R.min()) + int(R.max())) // 2)))
            ho = trial.huff_offset
            if presence & 0x02 and rng.random() < 0.6:
                ho = out['ho'] = max(-16384, min(16383, mid + int(rng.integers(-3, 4))))
            cb = int(rng.choice([0, 1, 2, 3])) if st.get('huff', True) else 0
            for h in ([ho] + ([mid] if presence & 0x02 else [])):
                for cbx in (cb, 0):
                    for L in range(0, 25 - q):
                        if fits(R, cbx, L, h):
                            if h != trial.huff_offset:
                                out['ho'] = h
                            out['cb'], out['lsbs'] = cbx, L + q
                            return out
        raise AssertionError('no coding for channel %d' % c)

    def _write_block(self, b, s, p, blk, bypass, restart, check_byte):
        used, n = self.used, s.n
        b.put(1, p is not None)
        if p is not None:
            b.put(1, restart)
            if restart:
                s.restart_header(b, check_byte)
            if s.presence & 1:
                b.put(1, p['presence'] is not None)
                if p['presence'] is not None:
                    s.presence = p['presence']
                    b.put(8, s.presence)
            if s.presence & 0x80:
                b.put(1, p['blocksize'] is not None)
                if p['blocksize'] is not None:
                    s.blocksize = p['blocksize']
                    b.put(9, s.blocksize)
            assert p['blocksize'] is None or s.blocksize == p['blocksize']
            if s.presence & 0x40:
                b.put(1, p['matrix'] is not None)
                if p['matrix'] is not None:
                    s.matrices = p['matrix']
                    b.put(4, len(s.matrices))
                    for mt in s.matrices:
                        b.put(4, mt['out']); b.put(4, mt['frac']); b.put(1, mt['bypass'])
                        for v in mt['coeff']:
                            b.put(1, v != 0)
                            if v:
                                b.put(mt['frac'] + 2, v)
                        if s.noise_type:
                            b.put(4, 0)
            else:
                assert p['matrix'] is None
            if s.presence & 0x20:
                b.put(1, p['shift'] is not None)
                if p['shift'] is not None:
                    s.out_shift = list(p['shift'])
                    for v in s.out_shift:
                        b.put(4, v)
            else:
                assert p['shift'] is None
            if s.presence & 0x10:
                b.put(1, p['quant'] is not None)
                if p['quant'] is not None:
                    s.quant = list(p['quant'])
                    for v in s.quant:
                        b.put(4, v)
            else:
                assert p['quant'] is None
            for c in range(n):
                cp = p['chans'][c]
                b.put(1, cp is not None)
                if cp is None:
                    continue
                ch = s.ch[c]
                for key, flag, iir in (('fir', 0x08, False), ('iir', 0x04, True)):
                    if s.presence & flag:
                        f = cp[key]
                        b.put(1, f is not None)
                        if f is not None:
                            s.changes[(c, key)] = s.changes.get((c, key), 0) + 1
                            b.put(4, f['order'])
                            used[key].add(f['order'])
                            if f['order']:
                                b.put(4, f['shift']); b.put(5, f['cbits']); b.put(3, f['cshift'])
                                for v in f['coeffs']:
                                    b.put(f['cbits'], v)
                                b.put(1, f.get('state') is not None)
                                if f.get('state'):
                                    sbits, sshift, vals = f['state']
                                    b.put(4, sbits); b.put(4, sshift)
                                    for v in vals:
                                        b.put(sbits, v)
                                    used['iir_state'] += 1
                            self._apply_filter(ch, f, iir)
                    else:
                        assert cp[key] is None
                if not ch.fir[0] and ch.iir[0]:
                    ch.fir[1] = ch.iir[1]
                if s.presence & 0x02:
                    b.put(1, cp['ho'] is not None)
                    if cp['ho'] is not None:
                        ch.huff_offset = cp['ho']
                        b.put(15, ch.huff_offset)
                        used['huff_offset'] += 1
                else:
                    assert cp['ho'] is None
                ch.codebook, ch.huff_lsbs = cp['cb'], cp['lsbs']
                b.put(2, ch.codebook); b.put(5, ch.huff_lsbs)
        # block data: bypassed LSBs, then per channel the Huffman code and the raw LSBs
        codes = []
        for c in range(n):
            ch, q = s.ch[c], s.quant[c]
            R, ch.fir_hist, ch.iir_hist = filter_residuals(ch, q, blk[:, c])
            s.known[c] = min(8, s.known[c] + len(R))
            L = ch.huff_lsbs - q
            u = R - sign_huff_offset(ch.codebook, L, ch.huff_offset)
            assert u.min() >= 0 and (u >> L).max() < (len(HUFF[ch.codebook - 1]) if ch.codebook else 1), c
            codes.append((u >> L, u & ((1 << L) - 1), L, ch.codebook))
            if s is self.top:
                used['codebooks'].add(ch.codebook)
                used['lsbs'].add(L)
        bp = [m for m, mt in enumerate(s.matrices) if mt['bypass']]
        for i in range(len(blk)):
            for m in bp:
                b.put(1, bypass[i, m])
            for sym, low, L, cb in codes:
                if cb:
                    b.put(HUFF[cb - 1][sym[i]][1], HUFF[cb - 1][sym[i]][0])
                b.put(L, low[i])


# ---- cases ---------------------------------------------------------------------------------------------------------
class TrueHDCase(object):
    """A TrueHD stream with the PCM it decodes to; `damage` = (kind, AU index, byte offset, regex) for a damaged copy."""

    def __init__(self, name, data, pcm, rate, au_offsets, seg_starts, damage=None, spa=40, sub_starts=None,
                 sub_lens=None):
        self.sub_starts, self.sub_lens = sub_starts, sub_lens
        self.name, self.data, self.pcm, self.rate = name, data, pcm, rate
        self.au_offsets, self.seg_starts, self.damage, self.spa = au_offsets, seg_starts, damage, spa

    @property
    def channels(self):
        return self.pcm.shape[1]

    @property
    def pcm16(self):
        return (self.pcm >> 8).astype(np.int16)

    def wav(self):
        import struct
        body = self.pcm16.astype('<i2').tobytes()
        ch = self.channels
        return (b'RIFF' + struct.pack('<I', 36 + len(body)) + b'WAVEfmt ' +
                struct.pack('<IHHIIHH', 16, 1, ch, self.rate, self.rate * ch * 2, ch * 2, 16) + b'data' +
                struct.pack('<I', len(body)) + body)

    def write(self, directory, suffix='.thd'):
        path = os.path.join(str(directory), self.name + suffix)
        with open(path, 'wb') as f:
            f.write(self.data)
        return path

    def write_wav(self, directory):
        path = os.path.join(str(directory), self.name + '.wav')
        with open(path, 'wb') as f:
            f.write(self.wav())
        return path

    def __repr__(self):
        return 'TrueHDCase(%s)' % self.name


def make_pcm(frames, channels, bits, rate, rng, amp=0.25):
    t = np.arange(frames) / float(rate)
    out = np.zeros((frames, channels), np.int64)
    full = (1 << (bits - 1)) - 1
    for c in range(channels):
        f = 150.0 + 90.0 * c + rng.random() * 50
        x = 0.6 * np.sin(2 * np.pi * f * t + c) + 0.3 * np.sin(2 * np.pi * 3.1 * f * t) + 0.1 * rng.standard_normal(frames)
        v = np.clip(np.round(x * amp * full), -full - 1, full).astype(np.int64)
        out[:, c] = v << (24 - bits)
    return out


def make(name, channels, bits, rate, seconds=None, n_au=None, n_sub=1, seed=0, style=None, restarts=(16,),
         eos_short=0, objects=False, arr2=None, amp=0.25, parity=True, **kw):
    rng = np.random.default_rng([SEED, seed])
    spa = 40 << (RATE_CODES[rate] & 7)
    if n_au is None:
        n_au = int(round(seconds * rate / spa))
    frames = n_au * spa - eos_short
    pcm = make_pcm(frames, channels, bits, rate, rng, amp)
    w = Writer(rate, pcm, bits, n_sub=n_sub, seed=int(rng.integers(1 << 30)), style=style, restarts=restarts,
               eos_short=eos_short, objects=objects, arr2=arr2, parity=parity, **kw)
    data = w.encode()
    case = TrueHDCase(name, data, pcm, rate, w.au_offsets, w.seg_starts, spa=spa, sub_starts=w.sub_starts,
                      sub_lens=w.sub_lens)
    case.used = w.used
    case.n_sub = w.n_sub
    return case


FULL = {'matrix': True, 'shift': True, 'quant': True, 'filters': True, 'blocks': True, 'omit': True}


def named_cases():
    cases = []
    add = lambda *a, **kw: cases.append(make(*a, **kw))
    add('mono16', 1, 16, 48000, n_au=60, seed=1)
    add('stereo16_raw', 2, 16, 48000, n_au=50, seed=2, style={'huff': False, 'permute': False})
    add('stereo24_full', 2, 24, 48000, n_au=120, seed=3, style=FULL, restarts=(7, 16, 1, 30))
    add('stereo16_full', 2, 16, 48000, n_au=120, seed=4, style=FULL, restarts=(12, 5))
    add('ch3_44k', 3, 16, 44100, n_au=80, n_sub=2, seed=5, style=FULL, restarts=(9,))
    add('ch4_96k', 4, 24, 96000, n_au=60, n_sub=3, seed=6, style=FULL, restarts=(20,))
    add('ch5_192k', 5, 16, 192000, n_au=30, n_sub=2, seed=7, style=FULL, restarts=(8,))
    add('ch6_two_sub', 6, 24, 48000, n_au=146, n_sub=2, seed=8, style=FULL, restarts=(13, 128))
    add('ch7_three_sub', 7, 16, 48000, n_au=50, n_sub=3, seed=9, style=FULL, restarts=(11,))
    add('ch8_three_sub', 8, 24, 48000, n_au=50, n_sub=3, seed=10, style=FULL, restarts=(16,))
    add('ch8_objects', 8, 24, 48000, n_au=40, n_sub=3, seed=11, style=FULL, restarts=(10,), objects=True)
    add('stereo_one_sub', 2, 16, 48000, n_au=40, seed=12, style=FULL, restarts=(128,))
    add('ch6_noise', 6, 16, 48000, n_au=60, n_sub=2, seed=13, style=dict(FULL, noise1=False), restarts=(6,))
    add('stereo_restart_every_au', 2, 16, 48000, n_au=40, seed=14, style=FULL, restarts=(1,))
    add('eos_short', 2, 24, 48000, n_au=33, seed=15, style=FULL, restarts=(10,), eos_short=17)
    add('ch6_eos', 6, 16, 96000, n_au=41, n_sub=2, seed=16, style=FULL, restarts=(8,), eos_short=63)
    add('no_parity', 2, 16, 48000, n_au=30, seed=17, style=FULL, parity=False)
    add('loud24', 2, 24, 48000, n_au=40, seed=18, style=FULL, amp=0.95)
    add('false_sync', 8, 24, 48000, n_au=30, n_sub=3, seed=19, style=FULL, restarts=(6,), objects=True, false_sync=True)
    return cases


def all_cases():
    """The undamaged cases, built once."""
    global _ALL
    if _ALL is None:
        _ALL = named_cases()
    return _ALL


_ALL = None


def _damaged(base, name, data, au, regex, offset=None):
    off = base.au_offsets[au] if offset is None else offset
    return TrueHDCase(base.name + '_' + name, bytes(data), base.pcm, base.rate, base.au_offsets, base.seg_starts,
                      damage=(name, au, off, regex), spa=base.spa)


def damaged_cases():
    """One damaged copy per refusal: (base, [cases]); case.damage = (kind, AU index, byte offset, regex)."""
    base = make('damage_base', 6, 16, 48000, n_au=40, n_sub=2, seed=40, style=FULL, restarts=(8,))
    n_au = len(base.au_offsets)
    seg = base.seg_starts[2]                        # a segment start that is not the first
    mid = seg + 3                                   # an AU inside a segment
    top = len(base.sub_starts[0]) - 1
    out = []

    def flip(at, mask):
        d = bytearray(base.data)
        d[at] ^= mask
        return d

    def msg(au, what, off=None):
        return r'TrueHD access unit {0} at byte offset {1}: .*({2})'.format(au, base.au_offsets[au] if off is None else off,
                                                                         what)
    out.append(_damaged(base, 'nibble', flip(base.au_offsets[mid], 0x10), mid, msg(mid, 'check nibble')))
    out.append(_damaged(base, 'sync_crc', flip(base.au_offsets[seg] + 14, 0x01), seg, msg(seg, 'major sync CRC')))
    rh = base.sub_starts[seg][top]
    out.append(_damaged(base, 'restart_crc', flip(rh + 2, 0x01), seg, msg(seg, 'restart header checksum')))
    out.append(_damaged(base, 'no_restart', flip(rh + 1, 0x20), seg, msg(seg, 'without a restart header')))
    end = base.sub_starts[mid][top] + base.sub_lens[mid][top]
    out.append(_damaged(base, 'parity', flip(end - 2, 0x04), mid, msg(mid, 'parity')))
    out.append(_damaged(base, 'crc', flip(end - 1, 0x80), mid, msg(mid, 'CRC mismatch')))
    last = n_au - 1
    out.append(_damaged(base, 'truncated', base.data[:base.au_offsets[last] + 10], last,
                        msg(last, 'runs past its block or the file')))
    # AU `mid` 2 bytes shorter (its last two bytes cut out, its length field and check nibble updated): the chain of
    # lengths still holds, but the substream directory runs past the AU
    at, nxt = base.au_offsets[mid], base.au_offsets[mid + 1]
    d = bytearray(base.data[:nxt - 2] + base.data[nxt:])
    w = ((d[at] & 0xF) << 8 | d[at + 1]) - 1
    d[at] = (d[at] & 0xF0) | (w >> 8); d[at + 1] = w & 0xFF
    p = parity(d[at:at + 4]) ^ parity(base.data[at:at + 4])          # keep the check nibble valid
    d[at] ^= (((p >> 4) ^ p) & 0xF) << 4
    out.append(_damaged(base, 'length', d, mid, msg(mid, 'substream directory')))
    bad = make('damage_base', 6, 16, 48000, n_au=40, n_sub=2, seed=40, style=FULL, restarts=(8,), bad_check=3)
    assert len(bad.data) == len(base.data)
    s3 = bad.seg_starts[3]
    out.append(TrueHDCase(base.name + '_lossless', bad.data, base.pcm, base.rate, bad.au_offsets, bad.seg_starts,
                          damage=('lossless', s3, bad.au_offsets[s3], msg(s3, 'lossless check'))))
    eos = make('damage_eos', 6, 16, 48000, n_au=12, n_sub=2, seed=41, style=FULL, restarts=(4,), eos_short=9)
    tail = make('damage_tail', 6, 16, 48000, n_au=8, n_sub=2, seed=42, style=FULL, restarts=(4,))
    after = len(eos.au_offsets)
    out.append(TrueHDCase(base.name + '_after_end', eos.data + tail.data, eos.pcm, eos.rate, None, None,
                          damage=('after_end', after, len(eos.data),
                                  r'TrueHD access unit {0} at byte offset {1}: data after the end-of-stream'.format(
                                      after, len(eos.data)))))
    short = make('damage_base', 6, 16, 48000, n_au=40, n_sub=2, seed=40, style=FULL, restarts=(8,), short_at=mid)
    out.append(TrueHDCase(base.name + '_short_au', short.data, base.pcm, base.rate, short.au_offsets, short.seg_starts,
                          damage=('short_au', mid, short.au_offsets[mid],
                                  r'TrueHD access unit {0} at byte offset {1}: short access unit before the end'.format(
                                      mid, short.au_offsets[mid]))))
    mlp = bytearray(base.data)
    mlp[base.au_offsets[0] + 7] = 0xBB
    out.append(_damaged(base, 'mlp', mlp, 0, r'MLP \(DVD-Audio\) is not supported'))
    return base, out


def assert_coverage(cases):
    used = {}
    for c in cases:
        for k, v in c.used.items():
            if isinstance(v, set):
                used.setdefault(k, set()).update(v)
            else:
                used[k] = used.get(k, 0) + v
    assert used['codebooks'] == {0, 1, 2, 3}, used['codebooks']
    assert min(used['lsbs']) == 0 and max(used['lsbs']) >= 20, used['lsbs']
    assert used['fir'] == set(range(9)), used['fir']
    assert used['iir'] == set(range(5)), used['iir']
    assert used['iir_state'] > 0 and used['huff_offset'] > 0 and used['omitted'] > 0 and used['noise'] > 0
    assert used['bypass'] > 0 and {1, 2, 3, 4} <= used['matrices'] and len(used['frac']) >= 10
    assert max(used['quant']) >= 4 and max(used['shift']) >= 4
    assert min(used['blocks']) == 8 and len(used['blocks']) > 20
    chans = {(c.channels, c.n_sub) for c in cases}
    assert {c for c, _ in chans} == set(range(1, 9)), chans
    assert {n for _, n in chans} == {1, 2, 3, 4}, chans
    assert {c.rate for c in cases} == {44100, 48000, 96000, 192000}
    assert any(c.used.get('false_syncs') for c in cases), 'no false major sync inside coded data'
    assert {1, 128} <= {b - a for c in cases for a, b in zip(c.seg_starts, c.seg_starts[1:] + [len(c.au_offsets)])}


LONG_AUS = 64                          # AUs in the repeated segment of long_stream


def periodic_segment(pcm, bits, n_sub=1, style=None, seed=0):
    """One restart segment coding `pcm` (a whole number of 48 kHz AUs) whose restart header carries the segment's own
    lossless check, so that the segment repeated any number of times is a valid stream."""
    n_au = len(pcm) // 40
    probe = Writer(48000, pcm, bits, n_sub=n_sub, seed=seed, style=style, restarts=(n_au,))
    probe.encode()
    return Writer(48000, pcm, bits, n_sub=n_sub, seed=seed, style=style, restarts=(n_au,),
                  first_check=xor8(probe.top.check)).encode()


def long_stream(minutes=90.0, seed=50):
    """A long 24-bit 7.1 stream at 48 kHz in two substreams: one restart segment of 64 AUs, repeated (every repetition
    checks the one before).  Quiet samples keep 90 minutes near 1.2 GB, past 2^32 bits.  -> (segment bytes, int16 PCM
    of one segment, repetitions)."""
    rng = np.random.default_rng([SEED, seed])
    pcm = rng.integers(-1, 1, (LONG_AUS * 40, 8)).astype(np.int64)
    seg = periodic_segment(pcm, 24, n_sub=2, style={'permute': True, 'omit': True}, seed=seed)
    reps = int(round(minutes * 60 * 48000 / (LONG_AUS * 40)))
    return seg, (pcm >> 8).astype(np.int16), reps
