"""GPU parity proper: the CUDA path, called through the C ABI, against (1) the reference's frozen
golden outputs, (2) the oracle (live cv2) on the same seeded inputs, (3) known answers and
size-independent properties at BASELINE sizes.  Tolerances are north_star's: shift within +-1
destination sample (1/12000 s), diff within 1e-5."""
import ctypes

import numpy as np
import pytest

from sushi_b200 import WavStream, SushiError, synth, _native
from tests.helpers import oracle_stream_from_pcm

pytestmark = pytest.mark.gpu

SHIFT_TOL = 1.0 / 12000 + 1e-9
DIFF_TOL = 1e-5


def gpu_stream_like(ref):
    return WavStream.from_array(ref.data, ref.sample_rate, ref.padding_size, ref.sample_count)


@pytest.fixture(scope='module')
def pair(golden_matcher):
    out = {}
    for stype in ('uint8', 'float32'):
        rs = oracle_stream_from_pcm(golden_matcher['src_pcm'], 12000, 1, 12000, stype)
        rd = oracle_stream_from_pcm(golden_matcher['dst_pcm'], 12000, 1, 12000, stype)
        out[stype] = (rs, rd, gpu_stream_like(rs), gpu_stream_like(rd))
    return out


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
def test_find_substream_matches_reference_golden(gpu_lib, golden_matcher, pair, stype):
    g = golden_matcher
    _, _, src, dst = pair[stype]
    for q, (a, b, c, w) in enumerate(g['queries']):
        d, t = dst.find_substream(src.get_substream(a, b), c, w)
        assert isinstance(d, np.float32) and isinstance(t, float)
        assert abs(float(d) - float(g['diff_' + stype][q])) <= DIFF_TOL, (q, d, g['diff_' + stype][q])
        assert abs(t - g['time_' + stype][q]) <= SHIFT_TOL, (q, t, g['time_' + stype][q])


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
def test_whole_curve_matches_reference_golden(gpu_lib, golden_matcher, pair, stype):
    g = golden_matcher
    _, _, src, dst = pair[stype]
    for qi in (0, 2):
        a, b, c, w = g['queries'][qi]
        s0, s1, stride = [int(v) for v in g['curve{0}_{1}_s0'.format(qi, stype)]]
        toff = src._get_sample_for_time(a)
        n = src._get_sample_for_time(b) - toff
        curve = dst.match_curve(src, toff, n, s0, s1 - s0 - n + 1)
        want = g['curve{0}_{1}'.format(qi, stype)]
        assert np.abs(curve[::stride] - want).max() <= DIFF_TOL
        assert abs(int(curve.argmin()) - int(want.argmin()) * stride) <= stride


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('seed', [1024, 4096, 8192, 16384], ids=lambda v: 'seed%d' % v)
def test_live_oracle_random_queries(gpu_lib, pair, stype, seed):
    """Random (event, centre, window) queries: GPU vs the oracle's cv2 call, 12 per seed."""
    rs, rd, src, dst = pair[stype]
    rng = np.random.default_rng(seed)
    for _ in range(12):
        a = float(rng.uniform(0.0, 20.0))
        ln = float(rng.choice([0.05, 0.5, 1.0, 3.0, 3.9]))
        b = min(a + ln, 24.0)
        c = float(a + rng.uniform(-3, 3))
        w = float(rng.choice([0.3, 1.5, 5.0, 10.0, 30.0]))
        pat_ref = rs.get_substream(a, b)
        d_ref, t_ref = rd.find_substream(pat_ref, c, w)
        d, t = dst.find_substream(src.get_substream(a, b), c, w)
        assert abs(float(d) - float(d_ref)) <= DIFF_TOL, (a, b, c, w)
        assert abs(t - t_ref) <= SHIFT_TOL, (a, b, c, w, t, t_ref)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('n', [11400, 40000], ids=['one_partition', 'three_partitions'])
def test_engines_agree_with_the_closed_form_and_each_other(gpu_lib, pair, stype, n):
    """Every engine is an implementation of the same formulation: each one's whole curve is within 1e-6 of the
    fp64 closed form, the engines agree with each other to float32 FFT noise, and each batch result is the
    first-index minimum of the engine's own curve -- for a template of one partition and one of three."""
    from oracle.ref_matcher import sqdiff_normed_fp64
    rs, rd, src, dst = pair[stype]
    try:
        toff = src._get_sample_for_time(6.1)
        lag0, nlags = 70000, 150001
        truth = sqdiff_normed_fp64(dst.data[0, lag0:lag0 + nlags + n - 1], src.data[0, toff:toff + n])
        curves, results = [], []
        # (engine, premac mode): the fused kernel, the fused kernel fed by the register-blocked multiply kernel
        # (premac 2 = for every query), the packed fused kernels (engine 2 picks per batch between one CTA per
        # lag block = engine 5 and one CTA per pair of lag blocks with the second product spectrum parked in
        # L2 = engine 4)
        variants = [(1, 1), (1, 2), (2, 1), (4, 1), (5, 1)]
        for engine, premac in variants:
            _native.check(gpu_lib.sb_set_engine(engine))
            _native.check(gpu_lib.sb_set_premac_mode(premac))
            curves.append(dst.match_curve(src, toff, n, lag0, nlags))
            assert np.abs(curves[-1] - truth).max() <= 1e-6, (engine, premac)
            results.append(dst.find_planned(src, [toff, toff + 5000, 100], [n, 3000, 48000],
                                            [lag0, 1000, 0], [nlags, 300000, 200000]))
            # the batch result is the first-index minimum of the variant's own curve
            d, i = dst.find_planned(src, [toff], [n], [lag0], [nlags])
            assert i[0] == int(curves[-1].argmin()) and d[0] == curves[-1].min()
        for a in range(len(variants)):
            for b in range(a + 1, len(variants)):
                assert np.abs(curves[a] - curves[b]).max() <= 2e-6, (variants[a], variants[b])
                assert np.abs(results[a][0] - results[b][0]).max() <= 2e-6, (variants[a], variants[b])
                assert np.abs(results[a][1] - results[b][1]).max() <= 1, (variants[a], variants[b])
        # pairs or single lag blocks (engines 4 / 5): the same arithmetic in the same order
        assert np.array_equal(curves[3], curves[4]) and np.array_equal(results[3][0], results[4][0])
    finally:
        _native.check(gpu_lib.sb_set_engine(2))
        _native.check(gpu_lib.sb_set_premac_mode(0))


def test_raw_ndarray_pattern_and_halves(gpu_lib, pair):
    """pattern may be any (1,n) ndarray: np.split halves (sushi.py:445) and detached copies."""
    rs, rd, src, dst = pair['uint8']
    tv = src.get_substream(6.1, 7.05)
    left, right = np.split(tv, [len(tv[0]) // 2], axis=1)
    tv_r = rs.get_substream(6.1, 7.05)
    left_r, right_r = np.split(tv_r, [len(tv_r[0]) // 2], axis=1)
    for p, pr in ((left, left_r), (right, right_r), (tv.copy(), tv_r)):
        d, t = dst.find_substream(p, 7.6, 10.0)
        d_ref, t_ref = rd.find_substream(pr, 7.6, 10.0)
        assert abs(float(d) - float(d_ref)) <= DIFF_TOL and abs(t - t_ref) <= SHIFT_TOL


def test_degenerate_inputs(gpu_lib, golden_matcher):
    """Zero-energy windows, zero template, constants, periodic ties (SURVEY.md appendix A)."""
    g = golden_matcher
    mk = lambda arr: WavStream.from_array(np.ascontiguousarray(arr), 12000, 0, arr.shape[1])
    z = mk(np.zeros((1, 64), np.uint8))
    seven = mk(np.full((1, 8), 7, np.uint8))
    nine = mk(np.full((1, 64), 9, np.uint8))
    ramp = mk((np.arange(64) % 8).astype(np.uint8)[None, :])
    assert np.array_equal(z.match_curve(seven, 0, 8, 0, 57), g['deg_zero_window'])
    assert np.array_equal(nine.match_curve(z, 0, 8, 0, 57), g['deg_zero_template'])
    assert np.abs(nine.match_curve(seven, 0, 8, 0, 57) - g['deg_const_7_vs_9']).max() <= 1e-6
    cur = ramp.match_curve(ramp, 0, 16, 0, 49)
    assert np.abs(cur - g['deg_periodic']).max() <= 1e-6
    diff, idx = ramp.find_planned(ramp, [0], [16], [0], [49])
    assert idx[0] == 0 and diff[0] == 0.0            # FIRST of the equal minima
    # exact copy -> 0 at the right place
    diff, idx = ramp.find_planned(ramp, [8], [24], [0], [41])
    assert diff[0] == 0.0 and idx[0] == 0


def test_search_span_shorter_than_pattern_swaps_like_cv2(gpu_lib, pair):
    rs, rd, src, dst = pair['uint8']
    # 12 s pattern near the end of a 24 s stream with a small window: span < pattern
    a, b, c, w = 8.0, 23.0, 33.5, 0.2
    pat_ref = rs.get_substream(a, b)
    d_ref, t_ref = rd.find_substream(pat_ref, c, w)
    d, t = dst.find_substream(src.get_substream(a, b), c, w)
    assert abs(float(d) - float(d_ref)) <= DIFF_TOL and abs(t - t_ref) <= SHIFT_TOL


def test_batch_equals_singles_and_is_order_independent(gpu_lib, pair):
    rs, rd, src, dst = pair['uint8']
    starts = np.array([1.0, 2.5, 6.0, 9.0, 12.0, 15.5, 18.0])
    ends = starts + np.array([2.0, 0.7, 3.5, 1.1, 2.2, 3.0, 1.0])
    centers = starts + 1.5
    windows = np.array([10.0, 1.5, 10.0, 30.0, 5.0, 10.0, 1.5])
    diffs, times = dst.find_substream_batch(src, starts, ends, centers, windows)
    for q in range(len(starts)):
        d, t = dst.find_substream(src.get_substream(starts[q], ends[q]), centers[q], windows[q])
        assert d == diffs[q] and t == times[q]
    perm = np.array([3, 0, 6, 2, 5, 1, 4])
    d2, t2 = dst.find_substream_batch(src, starts[perm], ends[perm], centers[perm], windows[perm])
    assert np.array_equal(d2, diffs[perm]) and np.array_equal(t2, times[perm])


def test_argument_errors_are_reported(gpu_lib, pair):
    rs, rd, src, dst = pair['uint8']
    with pytest.raises(SushiError):
        dst.find_planned(src, [0], [100], [0], [dst.data.shape[1]])        # span past the end
    with pytest.raises(SushiError):
        dst.find_planned(src, [-1], [100], [0], [10])
    with pytest.raises(SushiError):
        dst.find_planned(src, [0], [0], [0], [10])
    _, _, srcf, _ = pair['float32']
    with pytest.raises(SushiError):
        dst.find_planned(srcf, [0], [100], [0], [10])                       # dtype mismatch
    with pytest.raises(SushiError):
        dst.find_substream(srcf.get_substream(1.0, 2.0), 1.5, 1.0)


def test_config1_constant_shift_recovered(gpu_lib):
    """BASELINE config 1: 100 events, 60 s streams, +1.5 s, +-10 s: every event -> 1.5 s +- 1 sample,
    and identical to the oracle event by event."""
    src_pcm, dst_pcm = synth.make_pair(60.0, 0, 1.5)
    starts, ends = synth.make_events(100, 60.0, 0, 1.0, 4.0)
    for stype in ('uint8', 'float32'):
        rs = oracle_stream_from_pcm(src_pcm, 12000, 1, 12000, stype)
        rd = oracle_stream_from_pcm(dst_pcm, 12000, 1, 12000, stype)
        src, dst = gpu_stream_like(rs), gpu_stream_like(rd)
        diffs, times = dst.find_substream_batch(src, starts, ends, starts, np.full(len(starts), 10.0))
        ok = ends + 1.5 < 60.0
        assert np.all(np.abs((times - starts)[ok] - 1.5) <= SHIFT_TOL)
        for q in range(0, len(starts), 7):
            d_ref, t_ref = rd.find_substream(rs.get_substream(starts[q], ends[q]), starts[q], 10.0)
            assert abs(float(diffs[q]) - float(d_ref)) <= DIFF_TOL and abs(times[q] - t_ref) <= SHIFT_TOL


def test_config2_size_properties(gpu_lib):
    """BASELINE config 2 shape (2 x 30 min, +-60 s) on a reduced event count: shift recovery as a
    size-independent property, plus oracle spot checks at full window size."""
    dur = 1800.0
    src_pcm, dst_pcm = synth.make_pair(dur, 1, -7.25)
    src = WavStream.from_pcm(src_pcm, 12000)
    dst = WavStream.from_pcm(dst_pcm, 12000)
    starts, ends = synth.make_events(2000, dur, 1)
    sel = np.arange(0, 2000, 10)
    diffs, times = dst.find_substream_batch(src, starts[sel], ends[sel], starts[sel], np.full(len(sel), 60.0))
    ok = (starts[sel] - 7.25 > 0)
    assert np.all(np.abs((times - starts[sel])[ok] + 7.25) <= SHIFT_TOL)
    assert np.all(diffs[ok] < 0.2)
    from oracle.ref_matcher import RefStream
    rs = RefStream(src.data, 12000, src.padding_size, src.sample_count)
    rd = RefStream(dst.data, 12000, dst.padding_size, dst.sample_count)
    for q in (3, 77, 150):
        e = sel[q]
        d_ref, t_ref = rd.find_substream(rs.get_substream(starts[e], ends[e]), starts[e], 60.0)
        assert abs(float(diffs[q]) - float(d_ref)) <= DIFF_TOL and abs(times[q] - t_ref) <= SHIFT_TOL


def test_long_template_wide_window(gpu_lib):
    """config-5 corner: 30 s event, +-600 s span (14.4 M lags, 22 partitions)."""
    dur = 1500.0
    src_pcm, dst_pcm = synth.make_pair(dur, 2, 101.0)
    src = WavStream.from_pcm(src_pcm, 12000)
    dst = WavStream.from_pcm(dst_pcm, 12000)
    d, t = dst.find_substream(src.get_substream(700.0, 730.0), 700.0, 600.0)
    assert abs((t - 700.0) - 101.0) <= SHIFT_TOL
    from oracle.ref_matcher import RefStream
    rs = RefStream(src.data, 12000, src.padding_size, src.sample_count)
    rd = RefStream(dst.data, 12000, dst.padding_size, dst.sample_count)
    d_ref, t_ref = rd.find_substream(rs.get_substream(700.0, 730.0), 700.0, 600.0)
    assert abs(float(d) - float(d_ref)) <= DIFF_TOL and abs(t - t_ref) <= SHIFT_TOL


def test_running_sums_are_exact_for_uint8(gpu_lib):
    """A flat stream of 255s, 3 M samples: window energy must be exactly n*255^2 at every lag, far
    from the start of the running sums.  The only inexact step left is OpenCV's float32 rounding of
    sum(I*T) (3.25e9 is not a float32), so the curve is one constant below 1e-7."""
    n = 3_000_000
    s = WavStream.from_array(np.full((1, n), 255, np.uint8), 12000, 0, n)
    cur = s.match_curve(s, 1_000_000, 50_000, 2_900_000, 50_001)
    assert np.all(cur == cur[0]) and 0.0 <= cur[0] < 1e-7


# ---------------------------------------------------------------------------------------------
# GPU loader (sb_load_pcm + sb_normalise) against the reference's golden loader outputs
# ---------------------------------------------------------------------------------------------
from tests.test_oracle_golden import LOADER_CASES   # noqa: E402


@pytest.mark.parametrize('name', LOADER_CASES)
@pytest.mark.parametrize('stype', ['uint8', 'float32'])
def test_gpu_loader_matches_reference_golden(gpu_lib, golden_loader, name, stype):
    g = golden_loader
    fr, ch, sr = [int(v) for v in g[name + '_spec']]
    s = WavStream.from_pcm(g[name + '_pcm'], fr, sr, stype, channels=ch, loader='gpu')
    ref = g['{0}_{1}_data'.format(name, stype)]
    rate, count, pad = [int(v) for v in g['{0}_{1}_meta'.format(name, stype)]]
    assert (s.sample_rate, int(s.sample_count), s.padding_size) == (rate, count, pad)
    assert s.data.dtype == ref.dtype and s.data.shape == ref.shape
    assert np.array_equal(s.data, ref)                       # bit-exact, float32 included


def test_gpu_loader_equals_host_mirror_on_long_stream(gpu_lib):
    """10 minutes of stereo 44.1 kHz: the GPU loader and the NumPy mirror (itself pinned to the
    reference golden vectors) agree bit for bit, medians over ~9 M samples included."""
    fr = 44100
    base = synth.programme_audio(fr * 600, 9, rate=fr)
    pcm = np.stack([base, np.roll(base, 3) // 2], 1)
    for stype in ('uint8', 'float32'):
        a = WavStream.from_pcm(pcm, fr, 12000, stype, channels=2, loader='gpu')
        b = WavStream.from_pcm(pcm, fr, 12000, stype, channels=2, loader='host')
        assert np.array_equal(a.data, b.data)
        assert a.sample_count == b.sample_count and a.padding_size == b.padding_size
        assert abs(a.min_value - b.min_value) == 0 and abs(a.max_value - b.max_value) == 0


@pytest.mark.parametrize('name', ['stereo48k_24', 'mono44k1_24', 'six48k_24'])
@pytest.mark.parametrize('stype', ['uint8', 'float32'])
def test_gpu_loader_matches_reference_golden_int24(gpu_lib, golden_loader24, tmp_path, name, stype):
    """24-bit files through the public constructor (GPU decode of bytes 1 and 2 of every sample) against the
    reference's own WavStream.data, bit for bit."""
    g = golden_loader24
    p = str(tmp_path / 'x.wav')
    open(p, 'wb').write(g[name + '_wav'].tobytes())
    s = WavStream(p, 12000, stype)
    ref = g['{0}_{1}_data'.format(name, stype)]
    rate, count, pad = [int(v) for v in g['{0}_{1}_meta'.format(name, stype)]]
    assert (s.sample_rate, int(s.sample_count), s.padding_size) == (rate, count, pad)
    assert s.data.dtype == ref.dtype and np.array_equal(s.data, ref)
    s.close()


def test_wav_file_load_int24(gpu_lib, tmp_path):
    """RIFF file with 24-bit samples through the public constructor (GPU loader) vs the oracle."""
    import struct
    from oracle import ref_loader
    fr, ch, frames = 48000, 2, 48000 * 2
    rng = np.random.default_rng(4)
    vals = rng.integers(-2 ** 23, 2 ** 23, frames * ch, dtype=np.int64)
    payload = b''.join(int(v & 0xFFFFFF).to_bytes(3, 'little') for v in vals)
    hdr = b'RIFF' + struct.pack('<L', 36 + len(payload)) + b'WAVE' + b'fmt ' + struct.pack('<LHHLLHH', 16, 1, ch, fr, fr * ch * 3, ch * 3, 24)
    p = str(tmp_path / 'x24.wav')
    open(p, 'wb').write(hdr + b'data' + struct.pack('<L', len(payload)) + payload)
    want, count, pad = ref_loader.load_wav(p, 12000, 'uint8')
    got = WavStream(p, 12000, 'uint8')
    assert np.array_equal(got.data, want) and got.sample_count == count and got.padding_size == pad


# ---------------------------------------------------------------------------------------------
# edge cases: empty and ragged inputs, minimum sizes, batch splitting
# ---------------------------------------------------------------------------------------------
def _cv2_curve(image_row, templ_row):
    import cv2
    return cv2.matchTemplate(image_row[None, :], templ_row[None, :], cv2.TM_SQDIFF_NORMED)[0]


def test_empty_batch_is_a_no_op(gpu_lib, pair):
    rs, rd, src, dst = pair['uint8']
    d, i = dst.find_planned(src, [], [], [], [])
    assert len(d) == 0 and len(i) == 0


@pytest.mark.parametrize('engine', [1, 3, 4, 6, 7])
def test_minimum_sizes_and_ragged_edges(gpu_lib, engine):
    """n = 1 templates, single-lag searches, streams shorter than one lag block, searches that end on
    the last sample, spans that straddle exactly one block boundary."""
    rng = np.random.default_rng(engine)
    # 1 = fused kernel, 3 = blocked multiply, 4 / 6 / 7 = packed fused kernels (library engines 2 / 4 / 5)
    _native.check(gpu_lib.sb_set_engine(engine - 2 if engine >= 4 else 1))
    _native.check(gpu_lib.sb_set_premac_mode(2 if engine == 3 else 1))
    try:
        for total in (7, 1000, 16384, 16385, 40000):
            img = rng.integers(0, 256, total, dtype=np.uint8)
            tm = rng.integers(0, 256, 5000, dtype=np.uint8)
            s_img = WavStream.from_array(img[None, :], 12000, 0, total)
            s_tm = WavStream.from_array(tm[None, :], 12000, 0, len(tm))
            cases = [(0, 1, 0, total), (3, 1, total - 1, 1), (10, min(5, total), 0, total - min(5, total) + 1)]
            if total >= 1000:
                cases += [(100, 999, total - 999, 1), (0, 257, 3, total - 257 - 3 + 1)]
            if total == 16385:
                cases += [(5, 2, 16383, 1), (5, 1, 16384, 1), (0, 300, 16000, 86)]
            if total >= 40000:
                cases += [(5, 300, 16384 - 150, 151), (5, 300, 16383, 2), (7, 4000, 16000, total - 4000 - 16000 + 1)]
            for toff, n, lag0, nlags in cases:
                want = _cv2_curve(img[lag0:lag0 + nlags + n - 1], tm[toff:toff + n])
                got = s_img.match_curve(s_tm, toff, n, lag0, nlags)
                assert got.shape == want.shape
                assert np.abs(got - want).max() <= 1e-5, (total, toff, n, lag0, nlags)
                d, i = s_img.find_planned(s_tm, [toff], [n], [lag0], [nlags])
                assert abs(float(d[0]) - float(want.min())) <= 1e-5
                assert want[int(i[0])] - want.min() <= 2e-6          # a minimiser (ties on random data are rare)
    finally:
        _native.check(gpu_lib.sb_set_engine(2))
        _native.check(gpu_lib.sb_set_premac_mode(0))


def test_batch_runs_in_several_passes_of_whole_queries(gpu_lib, pair):
    """More template partitions than the resident budget: the batch runs in several passes of whole
    queries and still returns what the single-pass run returns."""
    rs, rd, src, dst = pair['uint8']
    starts = np.linspace(0.5, 19.0, 40)
    ends = starts + np.tile([0.3, 1.7, 3.2, 4.0], 10)
    centers, windows = starts + 1.0, np.full(40, 10.0)
    want = dst.find_substream_batch(src, starts, ends, centers, windows)
    # 40 templates of 1 to 4 partitions (B = 16384 samples), at most 7 partition spectra per pass
    toff, tlen = dst.plan_queries(src, starts, ends, centers, windows)[:2]
    parts = -(-np.asarray(tlen) // 16384)
    assert parts.max() <= 7 and parts.sum() > 2 * 7                  # several passes of whole queries
    _native.check(gpu_lib.sb_set_max_parts(7))
    try:
        got = dst.find_substream_batch(src, starts, ends, centers, windows)
    finally:
        _native.check(gpu_lib.sb_set_max_parts(16384))
    assert np.abs(got[0] - want[0]).max() <= 2e-6 and np.abs(got[1] - want[1]).max() <= SHIFT_TOL


def test_float32_stream_with_arbitrary_range(gpu_lib):
    """from_array accepts any float32 data, not only [0,1]: values around 1000 with a small variation
    (a hard case for the centring) still match cv2 to 1e-5."""
    rng = np.random.default_rng(3)
    img = (1000.0 + 5.0 * rng.standard_normal(60000)).astype(np.float32)
    s = WavStream.from_array(img[None, :], 12000, 0, len(img))
    want = _cv2_curve(img[2000:2000 + 30000 + 4999], img[20000:25000])
    got = s.match_curve(s, 20000, 5000, 2000, 30000)
    assert np.abs(got - want).max() <= 1e-5
    assert int(got.argmin()) == 18000 and got.min() <= 1e-6


def test_values_do_not_depend_on_the_query_range(gpu_lib, pair):
    """The property the curve cache, the sharding and the batching rest on: a lag's value depends only
    on (template, absolute position).  Any sub-range query returns exactly min / first argmin of the
    corresponding slice of one wide curve -- bit for bit, for ranges cut at arbitrary offsets."""
    rs, rd, src, dst = pair['uint8']
    toff, n = src._get_sample_for_time(9.0), 20000
    lo, count = 30000, 200000
    wide = dst.match_curve(src, toff, n, lo, count)
    rng = np.random.default_rng(8)
    a = rng.integers(0, count - 1, 40)
    b = np.minimum(a + rng.integers(1, 60000, 40), count)
    d, i = dst.find_planned(src, np.full(40, toff), np.full(40, n), lo + a, b - a)
    for q in range(40):
        part = wide[a[q]:b[q]]
        assert d[q] == part.min() and i[q] == int(part.argmin()), q
    # whole curves of sub-ranges are slices of the wide curve
    curves = dst.match_curves(src, [toff, toff], [n, n], [lo + 5, lo + 77777], [1000, 40001])
    assert np.array_equal(curves[0], wide[5:1005]) and np.array_equal(curves[1], wide[77777:77777 + 40001])


def test_mixed_batch_of_long_and_short_templates_keeps_caller_order(gpu_lib):
    """A batch mixing short templates (multiply inside the fused kernel) and very long ones (>= 12
    partitions: register-blocked multiply kernel) is processed class by class but returns results in
    the caller's order, and each query's answer equals, bit for bit, its answer when asked alone."""
    from tests.test_gpu_variants import _streams
    rs, rd, src, dst = _streams(200.0, 17)
    starts = np.array([10.0, 20.0, 45.0, 60.0, 90.0, 100.0, 120.0, 150.0])
    lens = np.array([0.5, 17.0, 1.0, 20.0, 0.2, 3.0, 24.0, 2.0])       # 17 / 20 / 24 s -> 13 / 15 / 18 partitions
    ends = starts + lens
    centers, windows = starts + 1.0, np.full(len(starts), 10.0)
    batch = dst.find_substream_batch(src, starts, ends, centers, windows)
    for q in range(len(starts)):
        d, t = dst.find_substream(src.get_substream(starts[q], ends[q]), centers[q], windows[q])
        assert d == batch[0][q] and t == batch[1][q], q
        d_ref, t_ref = rd.find_substream(rs.get_substream(starts[q], ends[q]), centers[q], windows[q])
        assert abs(float(d) - float(d_ref)) <= DIFF_TOL and abs(t - t_ref) <= SHIFT_TOL
    toff, tlen, lag0, nlags, _ = dst.plan_queries(src, starts, ends, centers, windows)
    assert (-(-np.asarray(tlen) // 16384) >= 12).sum() == 3                # three queries take the blocked route
    curves = dst.match_curves(src, toff, tlen, lag0, nlags)
    for q in range(len(starts)):
        assert len(curves[q]) == nlags[q] and curves[q].min() == batch[0][q]
