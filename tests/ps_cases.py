"""Seeded writer of MPEG program streams for the tests, with MP2 audio from tests/mp2_cases.py.

A case is a list of packs.  MPEG-1 (VCD-style) cases have 12-byte pack headers and MPEG-1 PES headers (0xFF stuffing,
the STD buffer field, PTS or PTS + DTS, or the lone 0x0F); MPEG-2 (DVD / DVB-style) cases have 14-byte pack headers
with stuffing, MPEG-2 PES headers, and optionally a PSM, DVD nav packs (private stream 2), private-stream-1 AC-3,
DTS, LPCM and subpicture blobs and padding packets.  Each pack holds one PES packet of random length, so PES packets
start anywhere and any chunk size splits some of them; video payloads hold start codes (pack, audio PES) that lie off
the packet chain.  The audio streams carry MP2 streams cut into PES payloads regardless of their frames.

`good_cases()` the cases that load, `refused_cases()` the ones whose audio is refused by codec name, `damaged_cases()`
copies with one fault each and the byte offset the refusal names, `cut_case()` a copy cut inside an audio PES."""
import struct

import numpy as np

from tests import mp2_cases as mc

VIDEO, AUDIO, PRIV1, PAD, PRIV2, PSM, SYS = 0xE0, 0xC0, 0xBD, 0xBE, 0xBF, 0xBC, 0xBB
SEQ_HEADER = bytes.fromhex('000001b3') + bytes([0x2D, 0x02, 0x40, 0x33, 0xFF, 0xFF, 0xE0, 0x18])
SEQ_EXT = bytes.fromhex('000001b5') + bytes([0x14, 0x8A, 0x00, 0x01, 0x00, 0x00])     # MPEG-2 video


def _ts(v, prefix):
    """a 33-bit time stamp in the 5 bytes of a PES header"""
    return bytes([prefix | ((v >> 29) & 0x0E) | 1, (v >> 22) & 0xFF, ((v >> 14) & 0xFE) | 1, (v >> 7) & 0xFF,
                  ((v << 1) & 0xFE) | 1])


def pack_header(scr, mpeg2, stuffing=0):
    if mpeg2:
        b = bytes([0x44 | ((scr >> 27) & 0x38) | ((scr >> 28) & 3), (scr >> 20) & 0xFF,
                   ((scr >> 12) & 0xF8) | 4 | ((scr >> 13) & 3), (scr >> 5) & 0xFF, ((scr << 3) & 0xF8) | 4 | 0, 1,
                   0x01, 0x89, 0xC3, 0xF8 | stuffing])
        return b'\x00\x00\x01\xba' + b + b'\xff' * stuffing
    return b'\x00\x00\x01\xba' + _ts(scr, 0x20)[:5] + bytes([0x80, 0x1B, 0x83])


def system_header(ids):
    body = bytes([0x80, 0xC4, 0xE1, 0x04, 0xE1, 0xFF])
    for sid in ids:
        body += bytes([sid, 0xE0 if sid >= 0xE0 else 0xC0, 0xE8 if sid >= 0xE0 else 0x20])
    return b'\x00\x00\x01\xbb' + struct.pack('>H', len(body)) + body


def psm(entries):
    """entries: [(stream_type, elementary stream id)]"""
    es = b''.join(bytes([t, i, 0, 0]) for t, i in entries)
    body = bytes([0x80, 0x01, 0, 0]) + struct.pack('>H', len(es)) + es
    crc = mc_crc(b'\x00\x00\x01\xbc' + struct.pack('>H', len(body) + 4) + body)
    return b'\x00\x00\x01\xbc' + struct.pack('>H', len(body) + 4) + body + crc.to_bytes(4, 'big')


def mc_crc(data):
    from tests.ts_cases import crc32_mpeg
    return crc32_mpeg(data)


def pes2(sid, payload, pts, sub=None):
    """MPEG-2 PES: PTS; `sub` a private-stream-1 substream header put in front of the payload"""
    opt = _ts(pts, 0x20)
    body = bytes([0x81, 0x80, len(opt)]) + opt + (sub or b'') + payload
    return b'\x00\x00\x01' + bytes([sid]) + struct.pack('>H', len(body)) + body


def pes1(sid, payload, pts, stuffing=0, std=True, dts=False):
    """MPEG-1 PES: 0xFF stuffing, the STD buffer field, then PTS, PTS + DTS, or (pts None) the lone 0x0F"""
    h = b'\xff' * stuffing + (bytes([0x60, 0x20]) if std else b'')
    if pts is None:
        h += b'\x0f'
    elif dts:
        h += _ts(pts, 0x30) + _ts(pts - 3000, 0x10)
    else:
        h += _ts(pts, 0x20)
    body = h + payload
    return b'\x00\x00\x01' + bytes([sid]) + struct.pack('>H', len(body)) + body


def nav_pack():
    pci = b'\x00\x00\x01\xbf\x03\xd4\x00' + bytes(0x3D3)
    dsi = b'\x00\x00\x01\xbf\x03\xfa\x01' + bytes(0x3F9)
    return pci + dsi


def padding(n):
    return b'\x00\x00\x01\xbe' + struct.pack('>H', n) + b'\xff' * n


class Elem(object):
    """One elementary stream of a case: `sid` its stream id, `sub` its private-stream-1 substream id (or None), `kind`
    ('mp2', 'video', 'ac3', 'dts', 'lpcm', 'subpicture'), `data` the bytes it carries; for audio `case` the MP2 case
    (mp2_cases) the data came from."""

    def __init__(self, sid, kind, data, sub=None, case=None):
        self.sid, self.kind, self.data, self.sub, self.case = sid, kind, data, sub, case
        self.pes_offsets = []              # byte offset of each of its PES packets in the file
        self.es = b''                      # the payload bytes its PES packets carry, in order


def video_blob(rng, n, mpeg2=False):
    """MPEG video as FFmpeg's content probe recognises it: a sequence header (and extension for MPEG-2), then pictures
    of slices holding random bytes with no zero byte.  Past the first 12 kB (what the probe reads) a pack start code and an audio PES start
    code are written into slice data, to lie off the packet chain."""
    out = bytearray(SEQ_HEADER + (SEQ_EXT if mpeg2 else b''))
    while len(out) < n:
        out += b'\x00\x00\x01\x00' + bytes([0x00, 0x0F, 0xFF, 0xF8])
        for s in range(1, 9):
            body = rng.integers(1, 256, int(rng.integers(100, 400)), dtype=np.uint8).tobytes()
            out += b'\x00\x00\x01' + bytes([s]) + body
    for at, code in ((n // 2, b'\x00\x00\x01\xba'), (3 * n // 4, b'\x00\x00\x01\xc0\x01\x00')):
        assert at > 12000
        out[at:at + len(code)] = code
    return bytes(out)


class PsCase(object):
    def __init__(self, name, mpeg2, elems, seed, psm_types=None, nav=False, pad=False, sys_header=True, end_code=True):
        self.name, self.mpeg2, self.elems = name, mpeg2, elems
        rng = np.random.default_rng([seed])
        out = bytearray()
        left = {id(e): 0 for e in elems}
        scr, k = 0, 0
        first = True
        while any(left[id(e)] < len(e.data) for e in elems):
            live = [e for e in elems if left[id(e)] < len(e.data)]
            e = live[int(rng.integers(len(live)))]
            out += pack_header(scr, mpeg2, int(rng.integers(0, 8)) if mpeg2 else 0)
            scr += 1800
            if first:
                if sys_header:
                    out += system_header([x.sid for x in elems if x.sid != PRIV1] + ([PRIV1] if any(
                        x.sid == PRIV1 for x in elems) else []))
                if psm_types:
                    out += psm(psm_types)
                first = False
            if nav and k % 4 == 0:
                out += nav_pack()
            n = int(rng.integers(200, 2100))
            at = left[id(e)]
            chunk = e.data[at:at + n]
            left[id(e)] = at + len(chunk)
            e.pes_offsets.append(len(out))
            pts = 90000 + 3600 * k
            if e.sub is not None:
                extra = {'ac3': b'\x01\x00\x01', 'dts': b'\x01\x00\x01', 'lpcm': b'\x07\x00\x04\x0c\x01\x80',
                         'subpicture': b''}[e.kind]
                out += pes2(PRIV1, chunk, pts, bytes([e.sub]) + extra)
            elif mpeg2:
                out += pes2(e.sid, chunk, pts)
            else:
                form = k % 4
                out += pes1(e.sid, chunk, pts if form != 3 else None, stuffing=int(rng.integers(0, 4)),
                            std=form != 1, dts=form == 2)
            e.es += chunk
            if pad and k % 3 == 0:
                out += padding(int(rng.integers(1, 300)))
            k += 1
        if end_code:
            out += b'\x00\x00\x01\xb9'
        self.data = bytes(out)

    @property
    def ext(self):
        return '.mpg' if not self.mpeg2 else '.vob' if any(e.sid == PRIV1 for e in self.elems) else '.mpg'

    def audio(self):
        return [e for e in self.elems if e.kind == 'mp2']

    def write(self, directory, data=None, suffix=None):
        path = str(directory / (self.name + (suffix or self.ext)))
        with open(path, 'wb') as f:
            f.write(self.data if data is None else data)
        return path

    def __repr__(self):
        return self.name


def _mp2(name, seed, n, **kw):
    return mc.stream(name, seed, n, **kw)


def good_cases():
    cases = []
    stereo = _mp2('ps_stereo', 301, 40, rate_index=0, bitrate_index=10, mode=0)
    cases.append(PsCase('vcd_stereo', False, [Elem(VIDEO, 'video', video_blob(np.random.default_rng([1]), 30000)),
                                             Elem(AUDIO, 'mp2', stereo.data, case=stereo)], 11))
    joint = _mp2('ps_joint', 302, 40, bitrate_index=[10, 12], mode=1, mode_ext=[0, 2], crc=[False, True])
    cases.append(PsCase('dvd_joint', True, [
        Elem(VIDEO, 'video', video_blob(np.random.default_rng([2]), 40000, True)),
        Elem(AUDIO, 'mp2', joint.data, case=joint),
        Elem(PRIV1, 'ac3', bytes(np.random.default_rng([3]).integers(0, 256, 4000, dtype=np.uint8)), sub=0x80),
        Elem(PRIV1, 'lpcm', bytes(4000), sub=0xA0),
        Elem(PRIV1, 'subpicture', bytes(np.random.default_rng([4]).integers(0, 256, 1500, dtype=np.uint8)), sub=0x20)],
        12, nav=True, pad=True))
    mono = _mp2('ps_mono', 303, 30, bitrate_index=8, mode=3, crc=True)
    cases.append(PsCase('dvb_mono_psm', True, [Elem(VIDEO, 'video', video_blob(np.random.default_rng([5]), 30000)),
                                               Elem(AUDIO, 'mp2', mono.data, case=mono)], 13,
                        psm_types=[(0x02, VIDEO), (0x04, AUDIO)]))
    lsf = _mp2('ps_lsf', 304, 30, lsf=1, rate_index=1, bitrate_index=[8, 10], mode=2)
    cases.append(PsCase('dvb_lsf', True, [Elem(AUDIO, 'mp2', lsf.data, case=lsf)], 14, pad=True, end_code=False))
    a = _mp2('ps_first', 305, 25, bitrate_index=10, mode=0)
    b = _mp2('ps_second', 306, 25, rate_index=2, bitrate_index=6, mode=3)
    cases.append(PsCase('two_audio', True, [Elem(VIDEO, 'video', video_blob(np.random.default_rng([6]), 30000, True)),
                                            Elem(AUDIO, 'mp2', a.data, case=a),
                                            Elem(AUDIO + 1, 'mp2', b.data, case=b)], 15))
    return cases


def refused_cases():
    """[(case, stream index, codec name)]: a case whose chosen audio stream is refused by FFmpeg's codec name"""
    rng = np.random.default_rng([7])
    l3 = _mp2('ps_l3', 307, 20, bitrate_index=10, mode=0)
    frames = []
    for f in l3.frames:
        f = bytearray(f)
        f[1] = (f[1] & ~0x06) | 0x02                      # layer III
        frames.append(bytes(f))
    c = PsCase('layer3', True, [Elem(AUDIO, 'mp3', b''.join(frames))], 16)
    d = PsCase('dvd_lossy', True, [Elem(PRIV1, 'ac3', bytes(rng.integers(0, 256, 3000, dtype=np.uint8)), sub=0x80),
                                   Elem(PRIV1, 'dts', bytes(rng.integers(0, 256, 3000, dtype=np.uint8)), sub=0x88),
                                   Elem(PRIV1, 'lpcm', bytes(3000), sub=0xA0)], 17)
    return c, d


def damaged_cases():
    """[(name, file bytes, byte offset named, regex)] from dvd_joint"""
    base = next(c for c in good_cases() if c.name == 'dvd_joint')
    data = base.data
    a = base.audio()[0]
    out = []
    k = a.pes_offsets[5]
    broken = bytearray(data)
    broken[k + 2] = 0x02
    out.append(('broken_start_code', bytes(broken), k, 'no start code'))
    k = a.pes_offsets[7]
    longer = bytearray(data)
    n = struct.unpack('>H', data[k + 4:k + 6])[0]
    longer[k + 4:k + 6] = struct.pack('>H', n + 5)
    out.append(('length_past_next', bytes(longer), k + 6 + n + 5, 'no start code'))
    k = a.pes_offsets[9]
    out.append(('garbage_between', data[:k] + b'\x11\x22\x33' + data[k:], k, 'no start code'))
    k = a.pes_offsets[3]
    hdr = bytearray(data)
    hdr[k + 6] = 0x01                                      # neither an MPEG-1 nor an MPEG-2 header
    out.append(('bad_pes_header', bytes(hdr), k, 'invalid PES header'))
    return base, out


def cut_case():
    """(case, file bytes cut inside an audio PES, the audio bytes that survive)"""
    base = next(c for c in good_cases() if c.name == 'dvb_mono_psm')
    a = base.audio()[0]
    k = a.pes_offsets[-3]
    n = struct.unpack('>H', base.data[k + 4:k + 6])[0]
    cut = k + 6 + n // 2
    before = sum(1 for o in a.pes_offsets if o < k)
    return base, base.data[:cut], before
