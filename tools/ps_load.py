"""MPEG program stream load on one GPU: a synthetic DVD-style program stream of 2048-byte packs, 48 kHz stereo MP2 at
192 kbit/s (tests/mp2_cases.py's long stream) for 90 minutes (or --minutes), with video packs of random bytes (no
zero byte, one off-chain pack start code each) to about 1.5 GB.  It is loaded once untimed, then --runs times, and the
tool prints one JSON line per load: file bytes, wall ms of WavStream(path), device ms per kernel class from
sb_profile_* (ps_mark, ps_chain, ps_compact, mp2_unpack, mp2_dct, mp2_window, ...), timed by device events.  The
card's name, power limit and SM clock are read in the same run.
    python tools/ps_load.py [--minutes 90] [--runs 3] [--dir /tmp]
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
from tests import mp2_cases as mc  # noqa: E402
from tests import ps_cases as pc  # noqa: E402

PACK = 2048
VIDEO_PER_AUDIO = 11              # video packs between audio packs: about 1.5 GB for 90 minutes


def write(path, data):
    """the program stream of MP2 stream `data`: every pack a 14-byte pack header and one PES filling it"""
    rng = np.random.default_rng([3])
    room = PACK - 14 - 14                              # pack header, PES header with PTS
    video = bytearray(rng.integers(1, 256, room, dtype=np.uint8).tobytes())
    video[room // 2:room // 2 + 4] = b'\x00\x00\x01\xba'
    vpes = pc.pes2(pc.VIDEO, bytes(video), 90000)
    scr = 0
    with open(path, 'wb') as f:
        for at in range(0, len(data), room):
            out = [pc.pack_header(scr, True), pc.pes2(pc.AUDIO, data[at:at + room], 90000 + at)]
            for _ in range(VIDEO_PER_AUDIO):
                scr += 300
                out += [pc.pack_header(scr, True), vpes]
            f.write(b''.join(out))
        f.write(b'\x00\x00\x01\xb9')
    assert len(vpes) + 14 == PACK and struct.unpack('>H', vpes[4:6])[0] == PACK - 20


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=float, default=90.0)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': alac_load.card()}), flush=True)
    directory = tempfile.mkdtemp(prefix='ps_load_', dir=args.dir)
    try:
        frames, data = mc.long_stream(args.minutes)
        path = os.path.join(directory, 'long.vob')
        write(path, data)
        flac_load.load_once(lib, path)                             # warm-up: page cache, device pool
        for r in range(args.runs):
            wall, phases = flac_load.load_once(lib, path)
            print(json.dumps({'minutes': args.minutes, 'input': 'mp2 (program stream)', 'run': r, 'frames': len(frames),
                              'bytes': os.path.getsize(path), 'wall_ms': round(1e3 * wall, 1),
                              'kernel_ms': phases}), flush=True)
        print(json.dumps({'card_after': alac_load.card()}), flush=True)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
