"""Ogg FLAC load on one GPU: 90 minutes (or --minutes) of 48 kHz stereo 24-bit FLAC (tests/flac_cases.py's periodic
file: VERBATIM frames of 1152 samples, every 16th LPC) in Ogg pages as libFLAC's Ogg encoder lays them out, one frame
per page, about 1.6 GB.  It is loaded once untimed, then --runs times, and the tool prints one JSON line per load: file
bytes, pages, wall ms of WavStream(path), device ms per kernel class from sb_profile_* (ogg_mark, ogg_chain, ogg_crc,
ogg_compact for the demux; flac_frames, flac_decode, flac_decorrelate for the decode; ...), timed by device events.
The card's name, power limit and SM clock are read in the same run.
    python tools/ogg_load.py [--minutes 90] [--runs 3] [--dir /tmp]
Files go to a temporary directory (or --dir) and are removed afterwards.  Nothing is asserted."""
import argparse
import json
import os
import shutil
import struct
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import alac_load  # noqa: E402
import flac_load  # noqa: E402
from sushi_b200 import _native  # noqa: E402
from tests import flac_cases as fc  # noqa: E402
from tests import ogg_cases as oc  # noqa: E402

SERIAL = 0x0665


def frame_offsets(data, first):
    """the offsets of a FLAC file's frames: the sync codes whose coded frame number is the next one and whose header
    passes its CRC-8 (false syncs inside VERBATIM payloads are passed over)"""
    d = np.frombuffer(data, np.uint8)
    cand = np.flatnonzero((d[first:-1] == 0xFF) & (d[first + 1:] == 0xF8)) + first
    out, want = [], 0
    for c in cand.tolist():
        b = data[c + 4]
        extra = 0
        if b < 0x80:
            n = b
        else:
            extra = 1 if b < 0xE0 else 2 if b < 0xF0 else 3
            n = b & (0x3F >> extra)
            for k in range(extra):
                n = (n << 6) | (data[c + 5 + k] & 0x3F)
        bs, sr = data[c + 2] >> 4, data[c + 2] & 15
        hl = 5 + extra + {6: 1, 7: 2}.get(bs, 0) + {12: 1, 13: 2, 14: 2}.get(sr, 0)
        if n == want and fc.crc8(data[c:c + hl]) == data[c + hl]:
            out.append(c)
            want += 1
    return out + [len(data)]


def crc_batch(pages):
    """Ogg CRC-32 of each page (CRC field zero), vectorised across pages: leading zeros leave a CRC from 0 unchanged,
    so the pages are right-aligned in one array and folded a column at a time"""
    width = max(len(p) for p in pages)
    m = np.zeros((len(pages), width), np.uint8)
    for i, p in enumerate(pages):
        m[i, width - len(p):] = np.frombuffer(p, np.uint8)
    c = np.zeros(len(pages), np.uint32)
    table = oc.CRC_TABLE
    for j in range(width):
        c = (c << np.uint32(8)) ^ table[(c >> np.uint32(24)) ^ m[:, j]]
    return c


def write(path, data, first):
    offs = frame_offsets(data, first)
    blocks = oc.split_blocks(data, first)
    info = bytes([blocks[0][0] & 0x7F]) + bytes(blocks[0][1:])
    mapping = b'\x7fFLAC\x01\x00' + struct.pack('>H', 1) + b'fLaC' + info
    comment = oc.vorbis_comment_block([b'ENCODER=tools/ogg_load.py'])
    comment[0] |= 0x80
    packets = [mapping, bytes(comment)] + [data[a:b] for a, b in zip(offs, offs[1:])]
    n_pages = 0
    with open(path, 'wb') as f:
        for a in range(0, len(packets), 8192):
            raw = []
            for i, pk in enumerate(packets[a:a + 8192], a):
                lacing = [255] * (len(pk) // 255) + [len(pk) % 255]
                flags = (2 if i == 0 else 0) | (4 if i == len(packets) - 1 else 0)
                raw.append(b'OggS' + bytes([0, flags]) + struct.pack('<qII', 1152 * max(0, i - 1), SERIAL, i) +
                           b'\0\0\0\0' + bytes([len(lacing)]) + bytes(lacing) + pk)
            crcs = crc_batch(raw)
            f.write(b''.join(p[:22] + struct.pack('<I', int(c)) + p[26:] for p, c in zip(raw, crcs)))
            n_pages += len(raw)
    return n_pages, len(offs) - 1


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=float, default=90.0)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': alac_load.card()}), flush=True)
    directory = tempfile.mkdtemp(prefix='ogg_load_', dir=args.dir)
    try:
        n_frames = int(args.minutes * 60 * 48000) // 1152
        data, _ = fc.periodic_file(n_frames, 500, 24, lambda j: None if j % 16 else 1, 11)
        first = 4
        while not data[first] & 0x80:
            first += 4 + int.from_bytes(data[first + 1:first + 4], 'big')
        first += 4 + int.from_bytes(data[first + 1:first + 4], 'big')
        path = os.path.join(directory, 'long.oga')
        pages, frames = write(path, data, first)
        del data
        flac_load.load_once(lib, path)                             # warm-up: page cache, device pool
        for r in range(args.runs):
            wall, phases = flac_load.load_once(lib, path)
            print(json.dumps({'minutes': args.minutes, 'input': 'flac 24-bit stereo (Ogg)', 'run': r, 'frames': frames,
                              'pages': pages, 'bytes': os.path.getsize(path), 'wall_ms': round(1e3 * wall, 1),
                              'kernel_ms': phases}), flush=True)
        print(json.dumps({'card_after': alac_load.card()}), flush=True)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
