"""Transport stream load against the WAV load of the same PCM and against a plain chunked read of the same file, on one
GPU.  The .m2ts files are BDAV streams of 48 kHz stereo LPCM (tests/ts_cases.py long_m2ts: one second of 240-frame PES
packets and video filler packets, repeated): 24 minutes at about 40 Mbit/s and 90 minutes at about 10 Mbit/s, at 16
and 24 bits.  (A TrueHD stream's load is its TS demux plus tools/truehd_load.py's decode.)  Each file is loaded once
untimed, then WavStream(.m2ts), WavStream(.wav) and the plain read alternate, 3 runs each, and the tool prints one JSON
line per load: file bytes, bytes read, wall ms, device ms per kernel class from sb_profile_* (ts_scan, ts_compact,
pes_index, bdlpcm_decode, decode_resample_pad, ...).  The card's name, power limit and clocks are read in the same run.
The files were just written, so they are read from the page cache: the plain read is the host's memory bandwidth, not
a disk's.
    python tools/ts_load.py [--runs 3] [--dir /tmp]
Files go to a temporary directory (or --dir) and are removed afterwards.  Nothing is asserted."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402

import flac_load  # noqa: E402
from sushi_b200 import _native, mpegts  # noqa: E402
from tests import ts_cases as tsc  # noqa: E402

# (minutes, bits, video filler packets per second): about 40 Mbit/s and 10 Mbit/s in all
FILES = ((24, 16, 25152), (24, 24, 24752), (90, 16, 5440), (90, 24, 5040))


def plain_read(path):
    """The file read as WavStream reads it: chunks of mpegts.CHUNK_BYTES into one page-locked buffer."""
    buf = _native.pinned_empty((mpegts.CHUNK_BYTES,), np.uint8)
    view = memoryview(buf)
    t = time.perf_counter()
    n = 0
    with open(path, 'rb', buffering=0) as f:
        while True:
            got = f.readinto(view)
            if not got:
                break
            n += got
    return time.perf_counter() - t, n


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    try:
        clocks = subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm,clocks.max.sm,clocks.mem', '--format=csv,noheader'],
                                capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        clocks = 'unknown'
    print(json.dumps({'card': flac_load.card(), 'clocks_sm_maxsm_mem': clocks}), flush=True)
    directory = tempfile.mkdtemp(prefix='ts_load_', dir=args.dir)
    try:
        jobs = []
        for minutes, bits, video in FILES:
            path = os.path.join(directory, 'a%d_%d.m2ts' % (minutes, bits))
            pcm, reps = tsc.long_m2ts(path, minutes, bits=bits, video_packets=video)
            wav = tsc.write_wav(os.path.join(directory, 'a%d_%d.wav' % (minutes, bits)), np.tile(pcm, (reps, 1)), 48000)
            jobs.append(('%d min %d-bit LPCM' % (minutes, bits), path, wav))
        for name, path, wav in jobs:
            mbps = os.path.getsize(path) * 8 / 1e6 / (len(np.memmap(wav, np.uint8, mode='r')) / 192000.0)
            for p in (path, wav):
                flac_load.load_once(lib, p)                     # warm-up: page cache, device pool
            for r in range(args.runs):
                for kind, p in (('m2ts', path), ('wav', wav), ('plain_read', path)):
                    if kind == 'plain_read':
                        wall, n = plain_read(p)
                        phases = {}
                    else:
                        wall, phases = flac_load.load_once(lib, p)
                        n = os.path.getsize(p)
                    print(json.dumps({'file': name, 'mbit_s': round(mbps, 1), 'input': kind, 'run': r,
                                      'bytes': os.path.getsize(p), 'bytes_read': n, 'wall_ms': round(1e3 * wall, 1),
                                      'kernel_ms': phases}), flush=True)
            for p in (path, wav):
                os.remove(p)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
