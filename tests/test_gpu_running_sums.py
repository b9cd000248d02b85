"""The running sums of a stream (sushi_b200/csrc/sb_stream.cu) lag by lag, at tile, group and slab edges.

A constant template makes this possible through the public curve call: its centred form is exactly zero, so the
correlation the kernels compute by FFT is exactly zero and every curve value comes from the window sums
pfx[j + n] - pfx[j] of I and I^2 alone:  (sum I^2 - 2 c sum I + n c^2) / sqrt(sum I^2 * n c^2), 1 where that is not
below 1, with sum I*T = c sum I rounded to float32 as OpenCV keeps it.  The truth is that formula on exact integer
window sums (uint8) or on an fp64 cumulative sum (float32).  A wrong carry anywhere moves the value of every window
that straddles it by far more than the bar of 1e-7; on uint8 the values are bit-exact or within one float32 ulp.

* uint8: the scan works in tiles of 4096 samples and groups of 128 tiles (524 288 samples).  Streams of
  3 groups + 5 tiles + 13 samples, of exactly 2 groups, and of 300 tiles + 1 sample, with all-255 runs (the largest
  in-tile sums), random stretches and silence; whole-stream curves with templates of 1, 16, 4096 and 12 000 samples.
* float32: the tile totals are scanned in slabs of 8192 tiles (33 554 432 samples).  One stream of
  8192 x 4096 + 3 x 4096 + 7 samples; curves of about 40 000 lags across the slab edge and up to the last lag.

find must return the minimum and the first argmin of the same curve, bit for bit."""
import numpy as np
import pytest

from sushi_b200 import WavStream

pytestmark = pytest.mark.gpu

TILE, GROUP, SLAB = 4096, 128 * 4096, 8192 * 4096
BAR = 1e-7
U8_LENGTHS = (3 * GROUP + 5 * TILE + 13, 2 * GROUP, 300 * TILE + 1)
U8_TEMPLATES = (1, 16, 4096, 12000)
F32_LENGTH = SLAB + 3 * TILE + 7


def upload(arr):
    return WavStream.from_array(np.ascontiguousarray(arr).reshape(1, -1), 12000, 0, arr.size)


def u8_stream(n, seed):
    """Runs of 255, random bytes and zeros, 1 000 to 150 000 samples each; every group edge sits inside a run of 255."""
    rng = np.random.default_rng(seed)
    x = np.empty(n, np.uint8)
    at = 0
    while at < n:
        k = min(int(rng.integers(1000, 150000)), n - at)
        kind = rng.integers(0, 5)
        x[at:at + k] = 255 if kind < 2 else (0 if kind == 2 else rng.integers(0, 256, k, dtype=np.uint8))
        at += k
    for g in range(GROUP, n, GROUP):
        x[max(g - 20000, 0):g + 20000] = 255
    return x


def closed_form(s1, s2, n, c):
    """Curve of a constant template of value c from window sums s1 = sum I, s2 = sum I^2 (fp64 or exact ints)."""
    s1 = np.asarray(s1, np.float64)
    s2 = np.asarray(s2, np.float64)
    corr = (c * s1).astype(np.float32).astype(np.float64)     # OpenCV's float32 sum(I*T)
    num = np.maximum(s2 - 2.0 * corr + n * c * c, 0.0)
    den = np.sqrt(s2) * np.sqrt(n * c * c)
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.where(num < den, num / den, 1.0)


def check(img, tmpl, n, lag0, nlags, truth, max_ulps=None):
    curve = img.match_curve(tmpl, 0, n, lag0, nlags)
    err = np.abs(curve.astype(np.float64) - truth)
    worst = int(err.argmax())
    assert err[worst] <= BAR, (n, lag0, worst, float(curve[worst]), float(truth[worst]))
    if max_ulps is not None:
        ulps = np.abs(curve.view(np.int32).astype(np.int64) - truth.astype(np.float32).view(np.int32))
        assert ulps.max() <= max_ulps, (n, lag0, int(ulps.argmax()), int(ulps.max()))
    d, i = img.find_planned(tmpl, [0], [n], [lag0], [nlags])
    first = int(curve.argmin())
    assert (d[0], int(i[0])) == (curve[first], first), (n, lag0, d[0], i[0], curve[first], first)
    return float(err.max())


@pytest.mark.parametrize('length', U8_LENGTHS)
def test_u8_running_sums_every_lag(gpu_lib, length):
    x = u8_stream(length, length)
    v = x.astype(np.int64)
    p1 = np.concatenate([[0], np.cumsum(v)])
    p2 = np.concatenate([[0], np.cumsum(v * v)])
    img = upload(x)
    for n in U8_TEMPLATES:
        c = 200                                        # near the data: few lags saturate at 1
        tmpl = upload(np.full(n, c, np.uint8))
        nlags = length - n + 1
        truth = closed_form(p1[n:] - p1[:nlags], p2[n:] - p2[:nlags], n, c)
        check(img, tmpl, n, 0, nlags, truth, max_ulps=1)
        tmpl.close()
    img.close()


def test_f32_running_sums_across_the_slab_edge(gpu_lib):
    rng = np.random.default_rng(7)
    x = rng.random(F32_LENGTH, dtype=np.float32)
    x[SLAB - 3 * TILE:SLAB + 3 * TILE] = 1.0          # the largest tile totals right at the slab edge
    v = x.astype(np.float64)
    p1 = np.concatenate([[0.0], np.cumsum(v)])
    p2 = np.concatenate([[0.0], np.cumsum(v * v)])
    img = upload(x)
    for n in (1, 16, 4096, 12000):
        c = 0.5
        tmpl = upload(np.full(n, c, np.float32))
        last = F32_LENGTH - n                          # the last lag
        for lag0 in (SLAB - 20000, last - 40000 + 1):
            nlags = min(40000, last - lag0 + 1)
            j = np.arange(lag0, lag0 + nlags)
            truth = closed_form(p1[j + n] - p1[j], p2[j + n] - p2[j], n, np.float64(np.float32(c)))
            check(img, tmpl, n, lag0, nlags, truth)
        tmpl.close()
    img.close()
