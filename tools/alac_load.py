"""ALAC (.m4a) load against FLAC and WAV loads of 48 kHz stereo audio of the same length, on one GPU.
The ALAC stream uses Apple's default coding (pb 40, mb 10, kb 14, frames of 4096, LPC order 8; 24-bit samples with one
shifted byte): 16 frames of programme material repeated for 24 and 90 minutes, at 16 and 24 bits; the WAV holds the same
samples; the FLAC is tools/flac_load.py's file of the same length and depth (other audio of the same shape).  Each file
is loaded once untimed, then WavStream alternates ALAC, FLAC and WAV, 3 runs each, and the tool prints one JSON line per
load: file bytes, wall ms of WavStream(path), device ms per kernel class from sb_profile_* (alac_frames, alac_decode,
decode_resample_pad, ...), and for ALAC the MP4 reader's host ms (Mp4File and its sample table read, timed apart) and
bytes read.  The card's name, power limit and SM clock are read in the same run.
    python tools/alac_load.py [--minutes 24 90] [--bits 16 24] [--runs 3] [--dir /tmp]
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

import flac_load  # noqa: E402
from sushi_b200 import _native, mp4  # noqa: E402
from tests import alac_cases as ac  # noqa: E402
from tests import loader_cases as lc  # noqa: E402
from tests import mp4_cases as m  # noqa: E402


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def build(directory, minutes, bits):
    cfg, frames, pcm, reps = ac.long_stream(bits=bits, minutes=minutes, n_unique=16)
    reps = minutes * 60 * 48000 // (len(frames) * cfg.frame_length)
    case = ac.AlacCase('a', cfg, frames * reps, pcm[:0], set())
    case.pcm = pcm
    m4a = os.path.join(directory, 'alac%d_%d.m4a' % (minutes, bits))
    with open(m4a, 'wb') as f:
        f.write(m.build('a', [m.alac_trak(case, per_chunk=(64,), edits=None)], ftyp=b'M4A '))
    width = bits // 8
    one = flac_load.pcm_bytes(pcm, width)
    wav = os.path.join(directory, 'alac%d_%d.wav' % (minutes, bits))
    with open(wav, 'wb') as f:
        f.write(lc.riff(2, 48000, width, b'', len(one) * reps))
        for _ in range(reps):
            f.write(one)
    flac, other_wav = flac_load.build(directory, minutes, bits)
    os.remove(other_wav)
    return m4a, flac, wav


def reader(path):
    t0 = time.perf_counter()
    with mp4.Mp4File(path) as f:
        t1 = time.perf_counter()
        table = f.frames(f.select('audio', None))
        t2 = time.perf_counter()
        return {'open_ms': round(1e3 * (t1 - t0), 1), 'table_ms': round(1e3 * (t2 - t1), 1),
                'bytes_read': f.bytes_read, 'samples': len(table)}


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
    directory = tempfile.mkdtemp(prefix='alac_load_', dir=args.dir)
    try:
        for minutes in args.minutes:
            for bits in args.bits:
                files = list(zip(('alac', 'flac', 'wav'), build(directory, minutes, bits)))
                for _, path in files:
                    flac_load.load_once(lib, path)                 # warm-up: page cache, device pool
                for r in range(args.runs):
                    for kind, path in files:
                        wall, phases = flac_load.load_once(lib, path)
                        row = {'minutes': minutes, 'bits': bits, 'input': kind, 'run': r,
                               'bytes': os.path.getsize(path), 'wall_ms': round(1e3 * wall, 1), 'kernel_ms': phases}
                        if kind == 'alac':
                            row['reader'] = reader(path)
                        print(json.dumps(row), flush=True)
                for _, path in files:
                    os.remove(path)
        print(json.dumps({'card_after': card()}), flush=True)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
