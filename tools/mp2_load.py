"""MP2 load on one GPU against FFmpeg's `mp2` decoder on one CPU core.  The stream is tests/mp2_cases.py's long stream:
48 kHz stereo at 192 kbit/s, 120 random layer II frames cycled for 90 minutes (or --minutes), in a Matroska file of
one block per 100 frames.  It is loaded once untimed, then --runs times, and the tool prints one JSON line per load:
file bytes, wall ms of WavStream(path), device ms per kernel class from sb_profile_* (mp2_unpack, mp2_dct,
mp2_window, decode_resample_pad, ...).  Then FFmpeg decodes the same frames through ctypes (tests/ref_mp2.py), timed
once.  The card's name, power limit and SM clock are read in the same run.
    python tools/mp2_load.py [--minutes 90] [--runs 3] [--dir /tmp]
Files go to a temporary directory (or --dir) and are removed afterwards.  Nothing is asserted."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import alac_load  # noqa: E402
import flac_load  # noqa: E402
from sushi_b200 import _native  # noqa: E402
from tests import mp2_cases as mc  # noqa: E402
from tests import ref_mp2  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=float, default=90.0)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': alac_load.card()}), flush=True)
    directory = tempfile.mkdtemp(prefix='mp2_load_', dir=args.dir)
    try:
        frames, data = mc.long_stream(args.minutes)
        sizes = [len(f) for f in frames]
        pieces = [sum(sizes[k:k + 100]) for k in range(0, len(sizes), 100)]
        case = mc.Case('long', frames, [mc.FrameSpec(mode=0, rate=48000)])
        path = mc.mkv_file('long', case, pieces).write(__import__('pathlib').Path(directory))
        flac_load.load_once(lib, path)                             # warm-up: page cache, device pool
        for r in range(args.runs):
            wall, phases = flac_load.load_once(lib, path)
            print(json.dumps({'minutes': args.minutes, 'input': 'mp2 (Matroska)', 'run': r, 'frames': len(frames),
                              'bytes': os.path.getsize(path), 'wall_ms': round(1e3 * wall, 1),
                              'kernel_ms': phases}), flush=True)
        t0 = time.perf_counter()
        pcm = ref_mp2.decode_packets(frames)[0]
        t1 = time.perf_counter()
        print(json.dumps({'ffmpeg_mp2_one_core_ms': round(1e3 * (t1 - t0), 1), 'samples': int(pcm.shape[0])}),
              flush=True)
        print(json.dumps({'card_after': alac_load.card()}), flush=True)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
