#!/usr/bin/env python3
"""Debug aid: the same batch through every engine; prints where results differ (diff values, indices)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sushi_b200 import WavStream, synth, _native   # noqa: E402

dur = float(sys.argv[1]) if len(sys.argv) > 1 else 60.0
nev = int(sys.argv[2]) if len(sys.argv) > 2 else 100
win = float(sys.argv[3]) if len(sys.argv) > 3 else 10.0
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 3
lib = _native.lib()
for stype in (sys.argv[5].split(',') if len(sys.argv) > 5 else ('uint8', 'float32')):
    src_pcm, dst_pcm = synth.make_pair(dur, 0, 1.5)
    src = WavStream.from_pcm(src_pcm, 12000, sample_type=stype)
    dst = WavStream.from_pcm(dst_pcm, 12000, sample_type=stype)
    starts, ends = synth.make_events(nev, dur, 0, 1.0, 4.0)
    res = {}
    for eng in ([int(e) for e in sys.argv[6].split(',')] if len(sys.argv) > 6 else (1, 2, 4, 5)):
        _native.check(lib.sb_set_engine(eng))
        for r in range(reps):
            d, t = dst.find_substream_batch(src, starts, ends, starts, np.full(len(starts), win))
            res[(eng, r)] = (d.copy(), t.copy())
    ref = res[(1, 0)]
    for key, (d, t) in sorted(res.items()):
        dd = np.abs(d - ref[0]); dt = np.abs(t - ref[1]) * 12000
        bad = np.nonzero((dd > 2e-6) | (dt > 0.5))[0]
        print(stype, 'engine %d rep %d: max|ddiff| %.3e max|dshift| %.2f samples, %d of %d queries differ' % (
            key[0], key[1], dd.max(), dt.max(), len(bad), len(d)), bad[:12].tolist())
_native.check(lib.sb_set_engine(2))
