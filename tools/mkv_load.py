"""Matroska load against FLAC load of the same audio, on one GPU.

Writes two remux-shaped MKVs, each a 48 kHz stereo 16-bit FLAC track (LPC order 10 with Rice partitions, mid/side on
one frame in four, 4096-sample frames, one frame per block) beside a 23.976 fps video track of random-byte frames:
24 minutes at 40 Mbit/s (about 7 GB) and 90 minutes at 8 Mbit/s (about 5.5 GB), and the .flac file of the same audio.
Free disk space is checked first.  Each file is read through once (untimed) to bring it into the page cache, then
each pair is loaded with WavStream alternating MKV and FLAC, 3 runs each after one untimed warm-up load of each
(nothing is dropped from the cache; a load alone would not cache an MKV's video pages, since the walk reads only their
block headers).  One JSON line per load: file bytes, wall ms of WavStream(path), and device ms per kernel class from
sb_profile_* (flac_frames for the MKV, flac_sync for the FLAC file, then flac_decode, flac_decorrelate and the
loader's classes).  Before each MKV load the container walk alone is timed (MatroskaFile + frames of the audio
track): host ms, bytes read and blocks walked.  The card's name, power limit and SM clocks are read in the same run.

    python tools/mkv_load.py [--cases 24:40 90:8] [--runs 3] [--dir /tmp]

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

from sushi_b200 import _native  # noqa: E402
from sushi_b200 import matroska as mk  # noqa: E402
from sushi_b200.wavstream import FlacFile, WavStream  # noqa: E402
from tests import flac_cases as fc  # noqa: E402
from tests import mkv_cases as mc  # noqa: E402

RATE, BLOCK, PERIOD = 48000, 4096, 256
SPEC = dict(kind='lpc', order=10, precision=13, porder=6, porder_search=True, method='rice')
FPS = 24000 / 1001.0


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def coded(j):
    return 10 if j % 4 == 0 else 1


def frame_slices(data, n_frames):
    """Every frame of a periodic_file: the payloads repeat every PERIOD frames, so the lengths of the first PERIOD
    frames (found by their exact headers) give every offset."""
    first = FlacFile.from_bytes(data[:65536], 'audio').frame_offset
    heads = [fc.frame_header(i, BLOCK, RATE, 2, coded(i % PERIOD), 16, {})[0] for i in range(PERIOD + 1)]
    at, payload = first, []
    for i in range(PERIOD):
        nxt = data.index(heads[i + 1], at + len(heads[i]))
        payload.append(nxt - at - len(heads[i]))
        at = nxt
    view = memoryview(data)
    frames, at = [], first
    for i in range(n_frames):
        n = len(fc.frame_header(i, BLOCK, RATE, 2, coded(i % PERIOD), 16, {})[0]) + payload[i % PERIOD]
        frames.append(view[at:at + n])
        at += n
    frames.append(view[at:])
    return data[:first], frames


def build(directory, minutes, mbps):
    n = minutes * 60 * RATE
    n_frames, tail = n // BLOCK, n % BLOCK or 100
    data, _ = fc.periodic_file(n_frames, tail, 16, coded, 11, RATE, BLOCK, PERIOD, SPEC)
    flac = os.path.join(directory, 'a%d.flac' % minutes)
    with open(flac, 'wb') as f:
        f.write(data)
    private, frames = frame_slices(data, n_frames)
    mkv = os.path.join(directory, 'a%d.mkv' % minutes)
    video = int(minutes * 60 * FPS)
    size, vbytes = mc.write_av(mkv, private, frames, [BLOCK] * n_frames + [tail], RATE, 2, 16, video,
                               int(mbps * 1e6 / 8 / FPS), 12)
    return flac, mkv, {'audio_frames': n_frames + 1, 'video_frames': video, 'video_bytes': vbytes}


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
        ms, k = ctypes.c_double(), ctypes.c_int64()
        lib.sb_profile_get(name.encode(), ctypes.byref(ms), ctypes.byref(k))
        if k.value:
            phases[name] = round(ms.value, 3)
    s.close()
    return wall, phases


def read_through(path):
    """Read the whole file once (the page cache keeps what it can); returns the seconds it took."""
    t0 = time.perf_counter()
    with open(path, 'rb', buffering=0) as f:
        while f.read(64 << 20):
            pass
    return time.perf_counter() - t0


def walk_once(path):
    t0 = time.perf_counter()
    with mk.MatroskaFile(path) as f:
        table = f.frames([f.select('audio', None).id])[1]
        read = f.bytes_read
    return time.perf_counter() - t0, read, len(table)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--cases', nargs='+', default=['24:40', '90:8'], help='minutes:Mbit/s of the video')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    cases = [tuple(float(x) for x in c.split(':')) for c in args.cases]
    directory = tempfile.mkdtemp(prefix='mkv_load_', dir=args.dir)
    need = sum(m * 60 * (mbps * 1e6 / 8 + 2 * 100000) for m, mbps in cases)     # video + MKV and FLAC audio
    free = shutil.disk_usage(directory).free
    if free < 1.2 * need:
        shutil.rmtree(directory, ignore_errors=True)
        sys.exit('mkv_load: %.1f GB free in %s, %.1f GB needed' % (free / 1e9, directory, 1.2 * need / 1e9))
    lib = _native.lib()
    lib.sb_profile_enable(1)
    print(json.dumps({'card': card()}), flush=True)
    try:
        for minutes, mbps in cases:
            minutes = int(minutes)
            t0 = time.perf_counter()
            flac, mkv, shape = build(directory, minutes, mbps)
            sizes = {'mkv': os.path.getsize(mkv), 'flac': os.path.getsize(flac)}
            print(json.dumps(dict(shape, minutes=minutes, mbps=mbps, bytes=sizes,
                                  build_s=round(time.perf_counter() - t0, 1))), flush=True)
            print(json.dumps({'minutes': minutes, 'read_through_s': {k: round(read_through(p), 2) for k, p in
                                                                      (('mkv', mkv), ('flac', flac))}}), flush=True)
            for path in (mkv, flac):
                load_once(lib, path)                           # warm-up: device pool
            for r in range(args.runs):
                walk, read, blocks = walk_once(mkv)
                print(json.dumps({'minutes': minutes, 'input': 'mkv_walk', 'run': r, 'host_ms': round(1e3 * walk, 1),
                                  'bytes_read': read, 'audio_frames': blocks}), flush=True)
                for kind, path in (('mkv', mkv), ('flac', flac)):
                    wall, phases = load_once(lib, path)
                    print(json.dumps({'minutes': minutes, 'input': kind, 'run': r, 'bytes': sizes[kind],
                                      'wall_ms': round(1e3 * wall, 1), 'kernel_ms': phases}), flush=True)
            print(json.dumps({'card': card()}), flush=True)
            os.remove(flac)
            os.remove(mkv)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
