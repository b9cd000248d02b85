#!/usr/bin/env python3
"""The shift solver over a season of episodes on one GPU: sequential against lockstep.

    python tools/season.py [--jobs 12] [--steps 3] [--sample-type uint8]

J seeded synthetic episodes, each a pair of 24-minute 12 kHz streams with ~350 events from synth.make_events and
piecewise-constant shifts of 2-3 segments; episode 0 jumps by more than the 10 s window half-way, so the solver rewinds
to its 30 s window there.  Streams are resident before timing (their load is reported apart).  After one untimed pass
of each, (a) shift_events job after job and (b) shift_events_many (all jobs in lockstep) run alternating, --steps
passes each.  One JSON line: episodes/s and script events/s of both (median pass), the matcher calls (GPU round trips:
every sb_find* / sb_match_curves* call) and kernel launches per pass, whether (a) and (b) gave equal per-event
results, and the card's name and power limit read in the same run."""
import argparse
import json
import logging
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sushi_b200 import WavStream, synth, _hostmem, _native, shift_events, shift_events_many   # noqa: E402
from sushi_b200.events import ScriptEvent                                                    # noqa: E402

_hostmem.keep_heap()
RATE = 12000
DURATION = 1440.0
EVENTS = 350


def gpu_identity():
    """Name and power limit of the card, read in the same process as the measurement."""
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(',')]
        return name, power
    except Exception as e:          # no nvidia-smi: say so instead of guessing
        return 'unknown (%s)' % e.__class__.__name__, 'unknown'


def episode(j):
    """Episode j of the season: (src_pcm, dst_pcm, starts, ends)."""
    rng = np.random.default_rng(1000 + j)
    nseg = 2 + j % 2
    cuts = np.sort(rng.uniform(0.2 * DURATION, 0.8 * DURATION, nseg - 1))
    shifts = np.round(rng.uniform(-3.0, 3.0, nseg), 3)
    if j == 0:
        shifts[1] = shifts[0] + 14.0
    segments = [(0.0, float(shifts[0]))] + [(float(c), float(s)) for c, s in zip(cuts, shifts[1:])]
    src, dst = synth.make_pair(DURATION, 2000 + j, segments)
    starts, ends = synth.make_events(EVENTS, DURATION, 3000 + j, 1.0, 4.0)
    return src, dst, starts, ends


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--jobs', type=int, default=12, help='number of episodes')
    ap.add_argument('--steps', type=int, default=3, help='timed passes of each mode (at least 3)')
    ap.add_argument('--sample-type', default='uint8', choices=['uint8', 'float32'])
    args = ap.parse_args()
    logging.disable(logging.WARNING)
    lib = _native.lib()
    inputs = [episode(j) for j in range(args.jobs)]
    t0 = time.perf_counter()
    streams = [(WavStream.from_pcm(src, RATE, sample_type=args.sample_type),
                WavStream.from_pcm(dst, RATE, sample_type=args.sample_type)) for src, dst, _, _ in inputs]
    lib.sb_sync()
    load_s = time.perf_counter() - t0
    n_events = sum(len(x[2]) for x in inputs)
    # matcher calls = GPU round trips: every sb_find* / sb_match_curves* entry point, counted at the binding
    calls = {'n': 0}
    for name in ('sb_find', 'sb_find_batch', 'sb_find_multi', 'sb_match_curves', 'sb_match_curves_multi', 'sb_match_curve'):
        fn = getattr(lib, name)

        def counted(*a, _fn=fn):
            calls['n'] += 1
            return _fn(*a)
        setattr(lib, name, counted)

    def one_pass(mode):
        for src, dst in streams:                      # no curve cache carried over from an earlier pass
            src.__dict__.pop('_curve_cache', None)
            dst.__dict__.pop('_curve_cache', None)
        evs = [[ScriptEvent(i, float(a), float(b)) for i, (a, b) in enumerate(zip(x[2], x[3]))] for x in inputs]
        c0, l0 = calls['n'], lib.sb_launch_count()
        t = time.perf_counter()
        if mode == 'sequential':
            for ev, (src, dst) in zip(evs, streams):
                shift_events(ev, src, dst)
        else:
            shift_events_many([(ev, src, dst) for ev, (src, dst) in zip(evs, streams)])
        lib.sb_sync()
        dt = time.perf_counter() - t
        out = [[(e.shift, e.diff, e._link.source_index if e.linked else -1) for e in ev] for ev in evs]
        return dt, calls['n'] - c0, lib.sb_launch_count() - l0, out

    one_pass('sequential')                            # untimed warm-up of both
    one_pass('lockstep')
    res = {'sequential': [], 'lockstep': []}
    outs = {}
    for _ in range(max(args.steps, 3)):
        for mode in ('sequential', 'lockstep'):
            dt, ncalls, nlaunch, out = one_pass(mode)
            res[mode].append((dt, ncalls, nlaunch))
            outs[mode] = out
    name, power = gpu_identity()
    line = {'workload': 'season: %d episodes of 2x24 min 12 kHz streams, ~%d events each, solver defaults' % (args.jobs, EVENTS),
            'jobs': args.jobs, 'events': n_events, 'sample_type': args.sample_type, 'load_s': round(load_s, 3),
            'gpu': name, 'power_limit': power, 'outputs_equal': outs['sequential'] == outs['lockstep']}
    for mode, rows in res.items():
        times = [r[0] for r in rows]
        med = float(np.median(times))
        line[mode] = {'episodes_per_s': round(args.jobs / med, 3), 'events_per_s': round(n_events / med, 1),
                      'pass_s': [round(t, 4) for t in times], 'round_trips': rows[-1][1], 'launches': rows[-1][2]}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
