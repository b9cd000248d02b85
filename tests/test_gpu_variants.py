"""The body variants of the packed kernels on uint8 streams (sb_set_epilogue): 3 is the default since round 2 --
run-level bounds pick the few runs of 8 lags that can hold a lag block's minimum, those leave the match kernel as
records and k_finish_runs evaluates them in fp64 -- and 1 is the first version (everything inside the match kernel).
Screening of either kind only selects the lags that get the exact fp64 evaluation, so every result must agree BIT FOR
BIT -- whole curves included (the debug curve path evaluates every lag exactly under both variants) -- over pairs of
lag blocks (engine 4) and single lag blocks (engine 5).  Runs with the plain `pytest -m gpu` (no opt-in gate): a
variant that fails here is deleted, not skipped.  Dropped in round 2 after measurement: the trimmed per-lag loop over
all lags (variant 2), triples of lag blocks, 16-bit spectrum rows, the warp-specialised kernel, the Stockham FFT passes
(DESIGN.md)."""
import numpy as np
import pytest

from sushi_b200 import WavStream, synth, _native
from tests.helpers import oracle_stream_from_pcm

pytestmark = pytest.mark.gpu


@pytest.fixture()
def epilogue(gpu_lib):
    def use(variant, engine=2):
        _native.check(gpu_lib.sb_set_engine(engine))
        _native.check(gpu_lib.sb_set_epilogue(variant))
    yield use
    _native.check(gpu_lib.sb_set_engine(2))
    _native.check(gpu_lib.sb_set_epilogue(3))


def _streams(dur, seed, stype='uint8'):
    src_pcm, dst_pcm = synth.make_pair(dur, seed, 1.5)
    rs = oracle_stream_from_pcm(src_pcm, 12000, 1, 12000, stype)
    rd = oracle_stream_from_pcm(dst_pcm, 12000, 1, 12000, stype)
    mk = lambda r: WavStream.from_array(r.data, r.sample_rate, r.padding_size, r.sample_count)
    return rs, rd, mk(rs), mk(rd)


@pytest.mark.parametrize('engine', [4, 5])          # pairs of lag blocks / single lag blocks
def test_body_variants_are_bit_identical_on_batches(gpu_lib, epilogue, engine):
    rs, rd, src, dst = _streams(240.0, 11)
    starts, ends = synth.make_events(300, 240.0, 12, 0.5, 6.0)
    win = np.full(len(starts), 30.0)
    out = {}
    for variant in (1, 3):
        epilogue(variant, engine)
        assert gpu_lib.sb_get_epilogue() == variant
        out[variant] = dst.find_substream_batch(src, starts, ends, starts, win)
    for variant in (3,):
        assert np.array_equal(out[1][0], out[variant][0])
        assert np.array_equal(out[1][1], out[variant][1])
    # and they are right: the known shift comes back
    ok = (ends + 1.5 < 240.0)
    assert np.abs((out[3][1] - starts)[ok] - 1.5).max() <= 1.0 / 12000 + 1e-9


@pytest.mark.parametrize('engine', [4, 5])
def test_body_variants_curves_and_ragged_ranges(gpu_lib, epilogue, engine):
    """Whole curves (every lag evaluated exactly) and ranges that start / end inside a lag block."""
    rs, rd, src, dst = _streams(60.0, 5)
    cases = [(src._get_sample_for_time(6.1), 11400, 70000, 150001), (100, 48000, 0, 200000),
             (5000, 3000, 16383, 16386), (7, 700, 1, 5), (40000, 20000, 32768, 16384)]
    for toff, n, lag0, nlags in cases:
        got = {}
        for variant in (1, 3):
            epilogue(variant, engine)
            got[variant] = (dst.match_curve(src, toff, n, lag0, nlags), dst.find_planned(src, [toff], [n], [lag0], [nlags]))
        for variant in (3,):
            assert np.array_equal(got[1][0], got[variant][0])
            assert got[1][1][0][0] == got[variant][1][0][0] and got[1][1][1][0] == got[variant][1][1][0]
        assert got[3][1][1][0] == int(got[3][0].argmin()) and got[3][1][0][0] == got[3][0].min()


def test_third_body_degenerate_inputs(gpu_lib, epilogue, golden_matcher):
    """Silent windows, zero template, constants, ties: the blocks whose minimum is saturated must fall back to
    evaluating every lag, exactly like the clamped screening values of the first version."""
    g = golden_matcher
    mk = lambda arr: WavStream.from_array(np.ascontiguousarray(arr), 12000, 0, arr.shape[1])
    z = mk(np.zeros((1, 64), np.uint8))
    seven = mk(np.full((1, 8), 7, np.uint8))
    nine = mk(np.full((1, 64), 9, np.uint8))
    ramp = mk((np.arange(64) % 8).astype(np.uint8)[None, :])
    rng = np.random.default_rng(3)
    gap = rng.integers(0, 256, (1, 40000), dtype=np.uint8)
    gap[0, 9000:31000] = 0                                     # a long silent stretch inside programme material
    gapped = mk(gap)
    for engine, body in ((4, 3), (5, 3)):
        epilogue(body, engine)
        assert np.array_equal(z.match_curve(seven, 0, 8, 0, 57), g['deg_zero_window'])
        assert np.array_equal(nine.match_curve(z, 0, 8, 0, 57), g['deg_zero_template'])
        assert np.abs(nine.match_curve(seven, 0, 8, 0, 57) - g['deg_const_7_vs_9']).max() <= 1e-6
        assert np.abs(ramp.match_curve(ramp, 0, 16, 0, 49) - g['deg_periodic']).max() <= 1e-6
        diff, idx = ramp.find_planned(ramp, [0], [16], [0], [49])
        assert idx[0] == 0 and diff[0] == 0.0
        diff, idx = z.find_planned(seven, [0], [8], [0], [57])
        assert idx[0] == 0 and diff[0] == 1.0                   # all saturated: FIRST index
        res = {}
        for variant in (1, 3):
            epilogue(variant, engine)
            res[variant] = (gapped.match_curve(gapped, 12000, 6000, 0, 34001),
                            gapped.find_planned(gapped, [12000, 100, 33000], [6000, 5000, 5000], [0, 8000, 0], [34001, 20000, 35001]))
        for variant in (3,):
            assert np.array_equal(res[1][0], res[variant][0])
            assert np.array_equal(res[1][1][0], res[variant][1][0]) and np.array_equal(res[1][1][1], res[variant][1][1])


def test_default_is_the_third_body(gpu_lib):
    assert gpu_lib.sb_get_epilogue() == 3 and gpu_lib.sb_get_engine() == 2
    assert gpu_lib.sb_set_epilogue(2) != 0 and gpu_lib.sb_get_epilogue() == 3      # the dropped variant is refused
    assert gpu_lib.sb_set_engine(3) != 0 and gpu_lib.sb_set_engine(6) != 0      # dropped engines are refused
    assert gpu_lib.sb_get_engine() == 2
    # so are the retired cuFFT engine, lag blocks other than 16384 and hop B/2; the settings stay as they were
    assert gpu_lib.sb_set_engine(0) != 0 and gpu_lib.sb_set_block_size(8192) != 0 and gpu_lib.sb_set_hop_mode(2) != 0
    assert gpu_lib.sb_get_engine() == 2 and gpu_lib.sb_get_block_size() == 16384


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
def test_pairs_are_bit_identical_to_single_lag_blocks(gpu_lib, epilogue, stype):
    """Engine 4 against engine 5 on whole curves and batch results: ranges of 1 .. 7 lag blocks (the last pair of a
    query holds one or two), ranges that start / end inside a block, templates of 1 .. 5 partitions, and searches
    that run into the end of the stream (spectrum rows past the last block are zero)."""
    rs, rd, src, dst = _streams(60.0, 7, stype)
    n_img = dst.data.shape[1]
    cases = [(6000, 11400, 0, 16384), (6000, 11400, 5, 16384), (6000, 20000, 100, 2 * 16384), (100, 48000, 16384, 3 * 16384),
             (100, 70000, 3, 4 * 16384 + 17), (40000, 3000, 16383, 5 * 16384 + 2), (7, 700, 1, 7 * 16384),
             (30000, 36000, n_img - 36000 - 90000, 90001), (5000, 12000, n_img - 12000 - 40000, 40001)]
    for toff, n, lag0, nlags in cases:
        got = {}
        for engine in (5, 4):
            epilogue(3, engine)
            got[engine] = (dst.match_curve(src, toff, n, lag0, nlags), dst.find_planned(src, [toff], [n], [lag0], [nlags]))
        assert np.array_equal(got[5][0], got[4][0]), (toff, n, lag0, nlags)
        assert got[5][1][0][0] == got[4][1][0][0] and got[5][1][1][0] == got[4][1][1][0]
        want = rd.match_curve(rs.data[:, toff:toff + n], lag0, nlags)
        assert np.abs(got[4][0] - want).max() <= 1e-5
        # a minimiser of cv2's curve (searches that reach into the constant padding have long runs of equal values)
        assert want[int(got[4][0].argmin())] - want.min() <= 2e-6
    starts, ends = synth.make_events(120, 60.0, 8, 0.5, 5.0)
    win = np.full(len(starts), 20.0)
    res = {}
    for engine in (5, 4):
        epilogue(3, engine)
        res[engine] = dst.find_substream_batch(src, starts, ends, starts, win)
    assert np.array_equal(res[5][0], res[4][0]) and np.array_equal(res[5][1], res[4][1])


@pytest.mark.parametrize('engine', [4, 5])
def test_many_partition_templates_without_the_blocked_route(gpu_lib, epilogue, engine):
    """sb_set_premac_mode(1) sends templates of twelve and more partitions (here 30 s = 22 partitions) through the
    packed kernels, whose staging area for the self-mirrored quad holds 32 rows: those CTAs must read the quad from
    L2 instead of writing past the area (ADVICE round 1).  Same answers as the default route to FFT rounding, and
    the oracle's within the usual bar."""
    rs, rd, src, dst = _streams(200.0, 13)
    starts = np.array([20.5, 61.25, 110.0])
    ends = starts + np.array([30.0, 17.0, 24.5])         # 22, 13 and 18 partitions
    win = np.full(3, 40.0)
    epilogue(3, engine)
    want = dst.find_substream_batch(src, starts, ends, starts, win)
    _native.check(gpu_lib.sb_set_premac_mode(1))
    try:
        got = dst.find_substream_batch(src, starts, ends, starts, win)
    finally:
        _native.check(gpu_lib.sb_set_premac_mode(0))
    assert np.abs(got[0] - want[0]).max() <= 2e-6 and np.abs(got[1] - want[1]).max() <= 1.0 / 12000 + 1e-9
    for q in range(3):
        d_ref, t_ref = rd.find_substream(rs.get_substream(starts[q], ends[q]), starts[q], 40.0)
        assert abs(float(got[0][q]) - float(d_ref)) <= 1e-5 and abs(got[1][q] - t_ref) <= 1.0 / 12000 + 1e-9
