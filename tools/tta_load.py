"""TTA (.tta) load against FLAC and WAV loads of 48 kHz stereo audio of the same length, on one GPU.
The TTA stream is tests/tta_cases.py's long stream: one whole frame of 50155 samples (about 1.045 s, the frame length
at 48 kHz) repeated for 24 and 90 minutes at 16 and 24 bits, then a short last frame; the WAV holds the same samples;
the FLAC is tools/flac_load.py's file of the same length and depth (other audio of the same shape).  Each file is
loaded once untimed, then WavStream alternates TTA, FLAC and WAV, 3 runs each, and the tool prints one JSON line per
load: file bytes, wall ms of WavStream(path), device ms per kernel class from sb_profile_* (tta_decode,
decode_resample_pad, ...), and for TTA the host walk's ms (TTAFile: the file read, header, seek table and tags, timed
apart from the load).  The card's name, power limit and SM clock are read in the same run.
    python tools/tta_load.py [--minutes 24 90] [--bits 16 24] [--runs 3] [--dir /tmp]
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
from sushi_b200 import _native, tta  # noqa: E402
from tests import loader_cases as lc  # noqa: E402
from tests import tta_cases as tc  # noqa: E402


def build(directory, minutes, bits):
    case, data, reps = tc.long_stream(bits=bits, minutes=minutes)
    path = os.path.join(directory, 'tta%d_%d.tta' % (minutes, bits))
    with open(path, 'wb') as f:
        f.write(data)
    del data
    width = bits // 8
    fl = case.frame_length
    one = flac_load.pcm_bytes(case.pcm[:fl], width)
    tail = flac_load.pcm_bytes(case.pcm[fl:], width)
    wav = os.path.join(directory, 'tta%d_%d.wav' % (minutes, bits))
    with open(wav, 'wb') as f:
        f.write(lc.riff(2, 48000, width, b'', len(one) * reps + len(tail)))
        for _ in range(reps):
            f.write(one)
        f.write(tail)
    flac, other_wav = flac_load.build(directory, minutes, bits)
    os.remove(other_wav)
    return path, flac, wav


def walk(path):
    t0 = time.perf_counter()
    f = tta.TTAFile(path)
    t1 = time.perf_counter()
    return {'walk_ms': round(1e3 * (t1 - t0), 1), 'frames': len(f.offsets)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--minutes', type=int, nargs='+', default=[24, 90])
    ap.add_argument('--bits', type=int, nargs='+', default=[16, 24])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': alac_load.card()}), flush=True)
    directory = tempfile.mkdtemp(prefix='tta_load_', dir=args.dir)
    try:
        for minutes in args.minutes:
            for bits in args.bits:
                files = list(zip(('tta', 'flac', 'wav'), build(directory, minutes, bits)))
                for _, path in files:
                    flac_load.load_once(lib, path)                 # warm-up: page cache, device pool
                for r in range(args.runs):
                    for kind, path in files:
                        wall, phases = flac_load.load_once(lib, path)
                        row = {'minutes': minutes, 'bits': bits, 'input': kind, 'run': r,
                               'bytes': os.path.getsize(path), 'wall_ms': round(1e3 * wall, 1), 'kernel_ms': phases}
                        if kind == 'tta':
                            row['host'] = walk(path)
                        print(json.dumps(row), flush=True)
                for _, path in files:
                    os.remove(path)
        print(json.dumps({'card_after': alac_load.card()}), flush=True)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
