#!/usr/bin/env python3
"""Numerical parity report: whole curves from the GPU against cv2.matchTemplate (the oracle's call) and
against the fp64 closed form, over template lengths and both sample types.  Prints a table.  It lives under tests/ because it calls the oracle (cv2, the fp64 closed
form): only tests/, smoke() and bench.py's CPU leg may."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv2                                              # noqa: E402  (the checker)
from sushi_b200 import WavStream, synth, _native       # noqa: E402
from oracle.ref_matcher import sqdiff_normed_fp64      # noqa: E402

dur = 240.0
src_pcm, dst_pcm = synth.make_pair(dur, 6, 1.5)
lib = _native.lib()
print('%-8s %-7s %-8s %9s %12s %12s %12s %8s' % ('type', 'event', 'window', 'lags', 'max|gpu-cv2|', 'max|gpu-f64|', 'max|cv2-f64|', 'argmin'))
for stype in ('uint8', 'float32'):
    src = WavStream.from_pcm(src_pcm, 12000, sample_type=stype)
    dst = WavStream.from_pcm(dst_pcm, 12000, sample_type=stype)
    # (engine, body variant of the packed kernels)
    variants = [(4, 3), (5, 3), (4, 1), (5, 1), (1, 1)]
    for engine, epilogue in variants:
        _native.check(lib.sb_set_engine(engine))
        _native.check(lib.sb_set_epilogue(epilogue))
        for ev_len, win in ((0.5, 10.0), (1.0, 10.0), (3.0, 10.0), (3.0, 60.0), (10.0, 10.0), (30.0, 10.0), (30.0, 60.0)):
            a = 100.0
            toff, tlen, lag0, nlags, _ = dst.plan_queries(src, [a], [a + ev_len], [a], [win])
            toff, tlen, lag0, nlags = int(toff[0]), int(tlen[0]), int(lag0[0]), int(nlags[0])
            gpu = dst.match_curve(src, toff, tlen, lag0, nlags)
            img = dst.data[:, lag0:lag0 + nlags + tlen - 1]
            tm = src.data[:, toff:toff + tlen]
            ref = cv2.matchTemplate(img, tm, cv2.TM_SQDIFF_NORMED)[0]
            f64 = sqdiff_normed_fp64(img[0], tm[0])
            print('%-8s %-7s %-8s %9d %12.3e %12.3e %12.3e %8s  engine=%s' % (
                stype, '%gs' % ev_len, '+-%gs' % win, nlags, np.abs(gpu - ref).max(), np.abs(gpu - f64).max(),
                np.abs(ref - f64).max(), 'same' if int(gpu.argmin()) == int(ref.argmin()) else 'DIFF(%d)' % (int(gpu.argmin()) - int(ref.argmin())),
                {1: 'fused', 2: 'packed', 4: 'packed_pair', 5: 'packed_single'}[engine]
                + ('/body%d' % epilogue if engine >= 2 else '')))
    _native.check(lib.sb_set_engine(2))
    _native.check(lib.sb_set_epilogue(3))
