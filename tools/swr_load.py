"""What --ffmpeg-audio costs, on one GPU, and what the reference's ffmpeg call spends on the same conversion.

1. 48 kHz stereo 16-bit FLAC files of 24 and 90 minutes (built as tools/flac_load.py builds them) are loaded with
   WavStream(path) and WavStream(path, ffmpeg_audio=True), alternating, 3 runs each after one untimed warm-up load of
   each: wall time and device ms per kernel class from sb_profile_*.
2. sb_pcm_swr alone (48 kHz -> 12 kHz) on 24 and 90 minutes of stereo and of 5.1 noise already on the device
   (sb_pcm_from_le): wall and swr_resample device ms, best of 3; and the host time of libswresample itself on the same
   PCM (tests/ref_swr.py, FMA3 path, 4096-frame feeds) -- what the reference's ffmpeg spends on this step.

One JSON line per measurement; the first names the card, its power limit and its SM clock, read in the same run.

    python tools/swr_load.py [--minutes 24 90] [--runs 3] [--dir /tmp]

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
from tests import ref_swr  # noqa: E402

BLOCK = 4608
SPEC = dict(kind='lpc', order=10, precision=13, porder=6, porder_search=True, method='rice')


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def kernels(lib):
    out = {}
    for name in lib.sb_profile_names().decode().split(','):
        ms, n = ctypes.c_double(), ctypes.c_int64()
        if name and lib.sb_profile_get(name.encode(), ctypes.byref(ms), ctypes.byref(n)) == 0 and n.value:
            out[name] = round(ms.value, 3)
    return out


def load_once(lib, path, ffmpeg_audio):
    lib.sb_profile_reset()
    _native.check(lib.sb_sync(), 'sb_sync')
    t0 = time.perf_counter()
    s = WavStream(path, 12000, 'uint8', ffmpeg_audio=ffmpeg_audio)
    _native.check(lib.sb_sync(), 'sb_sync')
    wall = time.perf_counter() - t0
    s.close()
    return wall, kernels(lib)


def flac_loads(lib, directory, minutes, runs):
    n = minutes * 60 * 48000
    period = 1024 * 1152 // BLOCK
    data, _, _ = fc.periodic_file(n // BLOCK, n % BLOCK or 100, 16, lambda j: 10 if j % 4 == 0 else 1, 11, 48000,
                                  BLOCK, period, SPEC, parts=True)
    path = os.path.join(directory, 'a%d.flac' % minutes)
    with open(path, 'wb') as f:
        f.write(data)
    del data
    for mode in (False, True):
        load_once(lib, path, mode)
    for r in range(runs):
        for mode in (False, True):
            wall, phases = load_once(lib, path, mode)
            print(json.dumps({'minutes': minutes, 'input': 'flac stereo', 'ffmpeg_audio': mode, 'run': r,
                              'wall_ms': round(1e3 * wall, 1), 'kernel_ms': phases}), flush=True)
    os.remove(path)


def stage(lib, minutes, mask, runs):
    channels = bin(mask).count('1')
    rng = np.random.default_rng(minutes * mask)
    pcm = (rng.standard_normal((minutes * 60 * 48000, channels), np.float32) * 6000).astype(np.int16)
    h = _native.decode(None, 'sb_pcm_from_le', pcm.ctypes.data_as(ctypes.c_void_p), len(pcm), channels, 2, 48000)
    best = None
    try:
        for _ in range(runs + 1):
            lib.sb_profile_reset()
            out = ctypes.c_void_p()
            t0 = time.perf_counter()
            _native.check(lib.sb_pcm_swr(h, mask, 12000, ctypes.byref(out)), 'sb_pcm_swr')
            wall = time.perf_counter() - t0
            lib.sb_pcm_destroy(out)
            k = kernels(lib).get('swr_resample')
            if best is None or wall < best[0]:
                best = (wall, k)
    finally:
        lib.sb_pcm_destroy(h)
    t0 = time.perf_counter()
    ref_swr.convert(pcm, mask, 48000, 12000)
    host = time.perf_counter() - t0
    print(json.dumps({'minutes': minutes, 'layout': hex(mask), 'sb_pcm_swr_wall_ms': round(1e3 * best[0], 2),
                      'swr_resample_ms': best[1], 'libswresample_host_s': round(host, 2)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=int, nargs='+', default=[24, 90])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': card()}), flush=True)
    directory = tempfile.mkdtemp(prefix='swr_load_', dir=args.dir)
    try:
        for minutes in args.minutes:
            flac_loads(lib, directory, minutes, args.runs)
        for minutes in args.minutes:
            for mask in (0x3, 0x3f):
                stage(lib, minutes, mask, args.runs)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
