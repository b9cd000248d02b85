#!/usr/bin/env python3
"""BASELINE config 5: event length x search span sweep at 1 or N GPUs (device-timed, streams resident).

    python tools/sweep.py [--queries 512] [--duration 5400]                                     # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29519 tools/sweep.py --out sweep_8gpu.json                                # N GPUs

(torchrun is only the launcher; this process never imports torch.)  Every cell sends ONE list of `--queries`
queries through sushi_b200.parallel.ShardedMatcher against resident streams (open_resident: one broadcast, running
sums and block spectra built once): each rank matches its contiguous shard, results are all-gathered.  Time per
cell = CUDA events on the library stream around match + all-gather, maximum over ranks, best of `--reps`.
Writes gpurun_out/<out> and prints a markdown table: events/s, algorithmic GB/s (SURVEY.md 8d bytes) and the
fraction of N x the measured HBM peak per cell.  With --oracle-check (default) rank 0 also compares one query per
row (event length) at the row's widest window with the CPU oracle (tests/helpers: cv2.matchTemplate through the
reference's find_substream) -- shift within +-1 sample, diff within 1e-5.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sushi_b200 import parallel, synth, _native   # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--queries', type=int, default=512)
ap.add_argument('--duration', type=float, default=5400.0)
ap.add_argument('--sample-type', default='uint8')
ap.add_argument('--reps', type=int, default=3)
ap.add_argument('--premac-mode', type=int, default=-1)
ap.add_argument('--events', default='0.5,1,3,10,30')
ap.add_argument('--windows', default='5,10,30,60,120,300,600')
ap.add_argument('--engine', type=int, default=-1, help='library engine (default: the library default)')
ap.add_argument('--epilogue', type=int, default=0, help='body variant of the packed kernels: 1 | 3 (default: the library default)')
ap.add_argument('--no-oracle-check', action='store_true')
ap.add_argument('--out', default='sweep.json', help='file name under gpurun_out/')
a = ap.parse_args()

rank, world = int(os.environ.get('RANK', '0')), int(os.environ.get('WORLD_SIZE', '1'))
lib = _native.lib(int(os.environ.get('LOCAL_RANK', '0')))
if a.engine >= 0:
    _native.check(lib.sb_set_engine(a.engine))
if a.epilogue > 0:
    _native.check(lib.sb_set_epilogue(a.epilogue))
if a.premac_mode >= 0:
    _native.check(lib.sb_set_premac_mode(a.premac_mode))
peak = 6650.0
try:
    peak = float(json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'])
except (OSError, ValueError, KeyError):
    pass

be = parallel.DeviceBackend(lib)
comm = parallel.NcclComm(rank, world, lib) if world > 1 else parallel.SingleComm(be)
m = parallel.ShardedMatcher(comm, be)
root = rank == 0
rs = rd = None
if root:
    from sushi_b200.wavstream import WavStream
    src_pcm, dst_pcm = synth.make_pair(a.duration, 2, 1.5)
    if a.no_oracle_check:
        class _Host(object):
            pass
        hs = []
        for pcm in (src_pcm, dst_pcm):
            w = WavStream.from_pcm(pcm, 12000, sample_type=a.sample_type)     # GPU loader; keep the host mirror only
            h = _Host()
            h.data, h.sample_rate, h.padding_size, h.sample_count = w.data.copy(), w.sample_rate, w.padding_size, w.sample_count
            w.close()
            hs.append(h)
        rs, rd = hs
    else:
        from tests.helpers import oracle_stream_from_pcm
        rs = oracle_stream_from_pcm(src_pcm, 12000, 1, 12000, a.sample_type)
        rd = oracle_stream_from_pcm(dst_pcm, 12000, 1, 12000, a.sample_type)
    m.set_streams(rs, rd)
else:
    m.set_streams()
m.open_resident()

EV = [float(x) for x in a.events.split(',')]
WIN = [float(x) for x in a.windows.split(',')]
bps = 1 if a.sample_type == 'uint8' else 4
rng = np.random.default_rng(5)
rows, checks = [], []
for ev_len in EV:
    for win in WIN:
        if root:
            starts = np.sort(rng.uniform(win * 0.25, a.duration - ev_len - 2.0, a.queries))
            starts = np.round(starts * 100) / 100
            ends = starts + ev_len
            plan = m.plan(starts, ends, starts, np.full(a.queries, win))
        else:
            plan = m.plan()
        toff, tlen, lag0, nlags = plan['all']
        alg = float(np.sum(bps * tlen + bps * (nlags + tlen - 1) + 16))
        best = None
        for rep in range(a.reps + 1):
            comm.barrier()
            _native.check(lib.sb_sync())
            _native.check(lib.sb_timer_start())
            m.run_planned()
            ms = ctypes.c_float()
            _native.check(lib.sb_timer_stop(ctypes.byref(ms)))
            t = comm.max_over_ranks([ms.value])[0]
            if rep > 0:
                best = t if best is None else min(best, t)
        diff, idx = m.gather_results()
        if root:
            times = plan['t0'] + idx / 12000.0
            shift = times - starts
            ok = (ends + 1.5 < a.duration) & (np.abs(1.5) <= win)
            good = float(np.mean(np.abs(shift[ok] - 1.5) <= 1.0 / 12000 + 1e-9)) if ok.any() else float('nan')
            rows.append({'event_s': ev_len, 'window_s': win, 'queries': a.queries, 'lags': int(np.median(nlags)),
                         'ms': round(best, 4), 'events_per_s': round(a.queries / best * 1e3, 1),
                         'alg_gbs': round(alg / best / 1e6, 2), 'frac_hbm': round(alg / best / 1e6 / (peak * world), 5),
                         'shift_recovered': good})
            print(rows[-1], flush=True)
            if not a.no_oracle_check and win == WIN[-1]:
                q = a.queries // 2
                d_ref, t_ref = rd.find_substream(rs.get_substream(starts[q], ends[q]), starts[q], win)
                checks.append({'event_s': ev_len, 'window_s': win, 'query': q, 'abs_diff_err': abs(float(diff[q]) - float(d_ref)),
                               'time_err_samples': abs(times[q] - t_ref) * 12000.0,
                               'pass': bool(abs(float(diff[q]) - float(d_ref)) <= 1e-5 and abs(times[q] - t_ref) <= 1.0 / 12000 + 1e-9)})
                print('oracle check', checks[-1], flush=True)
m.close_resident()
if root:
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump({'peak_hbm_gbs_per_gpu': peak, 'n_gpus': world, 'sample_type': a.sample_type, 'duration_s': a.duration,
               'engine': lib.sb_get_engine(), 'kernel_body': lib.sb_get_epilogue(), 'scaling': 'strong (one list per cell, sharded)',
               'timing': 'CUDA events around match + all-gather, max over ranks, best of %d; streams resident' % a.reps,
               'cells': rows, 'oracle_checks': checks},
              open(os.path.join(ROOT, 'gpurun_out', a.out), 'w'), indent=1)
    print('\n| event \\ window | ' + ' | '.join('±%g s' % w for w in WIN) + ' |')
    print('|---|' + '---|' * len(WIN))
    for ev_len in EV:
        cells = [r for r in rows if r['event_s'] == ev_len]
        print('| %g s | ' % ev_len + ' | '.join('%.0f ev/s, %.0f GB/s (%.2f%%)' % (r['events_per_s'], r['alg_gbs'], 100 * r['frac_hbm']) for r in cells) + ' |')
    if checks:
        print('oracle checks passed: %d of %d' % (sum(c['pass'] for c in checks), len(checks)))
comm.barrier()
comm.close()
be.release()
