"""TrueHD load against WAV and FLAC loads of 48 kHz stereo audio of the same length, on one GPU.
The TrueHD stream is one restart segment of 64 AUs (16-bit programme material coded with FIR / IIR prediction,
Huffman codebooks, quant steps and matrices) repeated for 24 and 90 minutes; the WAV holds the same samples; the FLAC
is tools/flac_load.py's file of the same length (LPC order 10, 16 bits; other audio of the same shape).  Each file is
loaded once untimed, then WavStream alternates TrueHD, WAV and FLAC, 3 runs each, and the tool prints one JSON line per
load: file bytes, wall time of WavStream(path), device ms per kernel class from sb_profile_* (truehd_sync,
truehd_decode, flac_*, decode_resample_pad, ...), and for TrueHD the restart segments and decode threads per SM.  The
card's name and power limit are read in the same run.
    python tools/truehd_load.py [--minutes 24 90] [--runs 3] [--dir /tmp]
Files go to a temporary directory (or --dir) and are removed afterwards.  Nothing is asserted."""
import argparse
import json
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402

import flac_load  # noqa: E402
from sushi_b200 import _native  # noqa: E402
from tests import loader_cases as lc  # noqa: E402
from tests import truehd_cases as tc  # noqa: E402

SEG_AUS = 64


def build(directory, minutes):
    rng = np.random.default_rng([tc.SEED, 70])
    pcm = tc.make_pcm(SEG_AUS * 40, 2, 16, 48000, rng)
    style = {'permute': False, 'filters': True, 'huff': True, 'quant': True, 'matrix': True, 'omit': True}
    seg = tc.periodic_segment(pcm, 16, n_sub=1, style=style, seed=71)
    reps = minutes * 60 * 48000 // (SEG_AUS * 40)
    thd = os.path.join(directory, 'a%d.thd' % minutes)
    with open(thd, 'wb') as f:
        for _ in range(reps):
            f.write(seg)
    one = (pcm >> 8).astype('<i2').tobytes()
    wav = os.path.join(directory, 'a%d.wav' % minutes)
    with open(wav, 'wb') as f:
        f.write(lc.riff(2, 48000, 2, b'', len(one) * reps))
        for _ in range(reps):
            f.write(one)
    flac, _ = flac_load.build(directory, minutes, 16)
    return thd, wav, flac, reps


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=int, nargs='+', default=[24, 90])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    sms = None
    try:
        import torch
        sms = torch.cuda.get_device_properties(_native.bound_device() or 0).multi_processor_count
    except Exception:
        pass
    print(json.dumps({'card': flac_load.card(), 'sms': sms}), flush=True)
    directory = tempfile.mkdtemp(prefix='truehd_load_', dir=args.dir)
    try:
        for minutes in args.minutes:
            thd, wav, flac, reps = build(directory, minutes)
            files = (('truehd', thd), ('wav', wav), ('flac', flac))
            for _, path in files:
                flac_load.load_once(lib, path)                 # warm-up: page cache, device pool
            for r in range(args.runs):
                for kind, path in files:
                    wall, phases = flac_load.load_once(lib, path)
                    row = {'minutes': minutes, 'input': kind, 'run': r, 'bytes': os.path.getsize(path),
                           'wall_ms': round(1e3 * wall, 1), 'kernel_ms': phases}
                    if kind == 'truehd':
                        row['segments'] = reps
                        row['threads_per_sm'] = round(reps / sms, 1) if sms else None
                    print(json.dumps(row), flush=True)
            for _, path in files:
                os.remove(path)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
