"""Raw MPEG audio files (.mp2) for the tests, from tests/mp2_cases.py streams: plain, behind one or two ID3v2 tags,
ahead of an APEv2 and an ID3v1 tag, starting mid-frame, cut inside the last frame, and layer III."""
import struct

from tests import mp2_cases as mc


def id3v2(n, footer=False):
    size = bytes([(n >> 21) & 0x7F, (n >> 14) & 0x7F, (n >> 7) & 0x7F, n & 0x7F])
    body = b'TIT2' + struct.pack('>I', n - 10) + b'\x00\x00' + b'\x00' + b'x' * (n - 11)
    return b'ID3\x04\x00' + bytes([0x10 if footer else 0]) + size + body + (b'3DI\x04\x00\x10' + size if footer else b'')


def apev2():
    item = struct.pack('<II', 5, 0) + b'Title\x00' + b'hello'
    footer = b'APETAGEX' + struct.pack('<IIII', 2000, 32 + len(item), 1, 0x80000000) + bytes(8)
    header = b'APETAGEX' + struct.pack('<IIII', 2000, 32 + len(item), 1, 0xA0000000) + bytes(8)
    return header + item + footer


def id3v1():
    return b'TAG' + b'title'.ljust(30, b'\0') + bytes(95)


def _starts(c):
    out, at = [], 0
    for f in c.frames:
        out.append(at)
        at += len(f)
    return out


def all_cases():
    """[(name, file bytes, mp2_cases.Case, the stream bytes in it)]"""
    c = mc.stream('mpa_joint', 401, 24, bitrate_index=[10, 12], mode=1, mode_ext=[1, 3], crc=[False, True])
    d = c.data
    out = [('plain', d, c, d),
           ('id3v2', id3v2(300) + id3v2(40, footer=True) + d, c, d),
           ('ape_id3v1', d + apev2() + id3v1(), c, d),
           ('mid_frame', d[300:], c, d[next(o for o in _starts(c) if o >= 300):]),
           ('cut_tail', d[:-100], c, d[:-100])]
    lsf = mc.stream('mpa_lsf', 402, 24, lsf=1, rate_index=0, bitrate_index=8, mode=3)
    out.append(('lsf_mono', lsf.data, lsf, lsf.data))
    return out


def layer3():
    c = mc.stream('l3', 400, 24, bitrate_index=10)
    frames = []
    for f in c.frames:
        f = bytearray(f)
        f[1] = (f[1] & ~0x06) | 0x02
        frames.append(bytes(f))
    return b''.join(frames)
