"""FLAC load against WAV load of the same audio, on one GPU.

Builds 48 kHz stereo files of 24 and 90 minutes at 16 and 24 bits, encoded at realistic settings (every frame LPC
order 10, coefficient precision 13, Rice partitions up to order 6 chosen per frame, mid/side on one frame in four; the
PCM repeats every 1024 frames, which the decoder does not know), and the plain PCM WAV of the same samples.  Each pair
is loaded with WavStream alternating FLAC and WAV, 3 runs each (after one untimed warm-up load of each), and the tool
prints one JSON line per load: file bytes, wall time of WavStream(path), and device ms per kernel class from
sb_profile_* (flac_sync, flac_decode, flac_decorrelate, decode_resample_pad, median_select_fine, normalise_quantise,
and the running-sum scan).  The card's name and power limit are read in the same run.

    python tools/flac_load.py [--minutes 24 90] [--bits 16 24] [--runs 3] [--dir /tmp]

Files go to a temporary directory (or --dir) and are removed afterwards.  Nothing is asserted."""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from sushi_b200 import _native  # noqa: E402
from sushi_b200.wavstream import WavStream  # noqa: E402
from tests import flac_cases as fc  # noqa: E402
from tests import loader_cases as lc  # noqa: E402

BLOCK = 4608
SPEC = dict(kind='lpc', order=10, precision=13, porder=6, porder_search=True, method='rice')


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def pcm_bytes(pcm, width):
    if width == 2:
        return pcm.astype('<i2').tobytes()
    u = (pcm.reshape(-1) & 0xFFFFFF).astype(np.uint32)
    return np.stack([u & 0xFF, (u >> 8) & 0xFF, u >> 16], 1).astype(np.uint8).tobytes()


def build(directory, minutes, bits):
    n = minutes * 60 * 48000
    period = 1024 * 1152 // BLOCK
    frames, tail = n // BLOCK, n % BLOCK or 100
    data, base, tail_pcm = fc.periodic_file(frames, tail, bits, lambda j: 10 if j % 4 == 0 else 1, 11, 48000, BLOCK,
                                            period, SPEC, parts=True)
    flac = os.path.join(directory, 'a%d_%d.flac' % (minutes, bits))
    with open(flac, 'wb') as f:
        f.write(data)
    del data
    width = bits // 8
    one = pcm_bytes(base, width)
    rest = pcm_bytes(base[:(frames % period) * BLOCK], width) + pcm_bytes(tail_pcm, width)
    size = len(one) * (frames // period) + len(rest)
    wav = os.path.join(directory, 'a%d_%d.wav' % (minutes, bits))
    with open(wav, 'wb') as f:
        f.write(lc.riff(2, 48000, width, b'', size))
        for _ in range(frames // period):
            f.write(one)
        f.write(rest)
    return flac, wav


def load_once(lib, path):
    lib.sb_profile_reset()
    _native.check(lib.sb_sync(), 'sb_sync')
    t0 = time.perf_counter()
    s = WavStream(path, 12000, 'uint8')
    _native.check(lib.sb_sync(), 'sb_sync')
    wall = time.perf_counter() - t0
    phases = {}
    for name in lib.sb_profile_names().decode().split(','):
        if not name:
            continue
        ms, n = ctypes.c_double(), ctypes.c_int64()
        lib.sb_profile_get(name.encode(), ctypes.byref(ms), ctypes.byref(n))
        if n.value:
            phases[name] = round(ms.value, 3)
    s.close()
    return wall, phases


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=int, nargs='+', default=[24, 90])
    ap.add_argument('--bits', type=int, nargs='+', default=[16, 24])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': card()}), flush=True)
    directory = tempfile.mkdtemp(prefix='flac_load_', dir=args.dir)
    try:
        for minutes in args.minutes:
            for bits in args.bits:
                flac, wav = build(directory, minutes, bits)
                sizes = {'flac': os.path.getsize(flac), 'wav': os.path.getsize(wav)}
                for path in (flac, wav):
                    load_once(lib, path)                       # warm-up: page cache, device pool
                for r in range(args.runs):
                    for kind, path in (('flac', flac), ('wav', wav)):
                        wall, phases = load_once(lib, path)
                        print(json.dumps({'minutes': minutes, 'bits': bits, 'input': kind, 'run': r,
                                          'bytes': sizes[kind], 'wall_ms': round(1e3 * wall, 1),
                                          'kernel_ms': phases}), flush=True)
                os.remove(flac)
                os.remove(wav)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
