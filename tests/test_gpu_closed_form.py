"""Every match engine on an H100 against the fp64 closed form of TM_SQDIFF_NORMED (tests/closed_form_cases.py: block
edges, near-ties, flat curves, float32 streams), under every library setting that still routes somewhere.

The bars:
* curves: |GPU - fp64| <= 1e-6 at every lag, and exactly 1.0 where the fp64 value saturates at 1.0;
* find: (diff, index) equal bit for bit to the minimum and FIRST argmin of the same setting's own curve (the screening
  loses nothing), |diff - truth.min()| <= 1e-6, truth[index] - truth.min() <= 2e-6, and the planted copy's exact index
  wherever a case knows it (the exact copy of every near-tie, the first of two exact copies, degenerate blocks).

1e-6 covers every source of difference from the closed form: OpenCV's float32 rounding of sum(I*T), which the kernels
reproduce and the closed form does not, moves a value by at most 2^-24 * 2 sum(I*T) / sqrt(sum I^2 sum T^2) <= 1.2e-7
(Cauchy-Schwarz); the fp32 FFTs of centred data add about 1e-7 of the curve (DESIGN.md section 2).  That second term
depends on the template length: the rounding of a correlation value is proportional to the norm of the whole 2B-point
block times the template's norm, while the value is divided by the window's and the template's energies, so it grows
like sqrt(2B / n).  Templates of fewer than SHORT samples therefore get 1e-6 * sqrt(SHORT / n) (2.8e-6 at n = 2, where
a since retired cuFFT engine measured 1.4e-6 on white noise).  The worst error per setting and sample type is printed at the end
of the module (run with -s to see it)."""
import ctypes
import collections

import numpy as np
import pytest

from sushi_b200 import WavStream, _native
from tests import closed_form_cases as cf

pytestmark = pytest.mark.gpu

VALUE_TOL = 1e-6
SHORT = 16
ARGMIN_TOL = 2e-6

Setting = collections.namedtuple('Setting', 'name engine premac epilogue max_parts')
DEFAULTS = Setting('default', 2, 0, 3, 16384)
SETTINGS = [
    Setting('fused_hop1', 1, 0, 3, 16384),
    Setting('fused_blocked', 1, 2, 3, 16384),
    Setting('packed_epi3', 2, 0, 3, 16384),
    Setting('packed_epi1', 2, 0, 1, 16384),
    Setting('pairs_epi3', 4, 0, 3, 16384),
    Setting('pairs_epi1', 4, 0, 1, 16384),
    Setting('single_epi3', 5, 0, 3, 16384),
    Setting('single_epi1', 5, 0, 1, 16384),
    Setting('packed_passes', 2, 0, 3, 1),                        # every query in a launch pass of its own
    Setting('fused_passes', 1, 0, 3, 1),
]

CASES = cf.all_cases()
WORST = collections.defaultdict(float)          # (setting, dtype[, 'n < SHORT']) -> worst |GPU - fp64|


def apply(lib, s):
    for rc in (lib.sb_set_engine(s.engine), lib.sb_set_premac_mode(s.premac), lib.sb_set_epilogue(s.epilogue),
               lib.sb_set_max_parts(s.max_parts)):
        _native.check(rc)


@pytest.fixture()
def setting(gpu_lib):
    yield lambda s: apply(gpu_lib, s)
    apply(gpu_lib, DEFAULTS)


@pytest.fixture(scope='module')
def truths():
    """The fp64 truth of every case, once per module (the host-side cost of this file)."""
    return {c.name: c.truth() for c in CASES}


@pytest.fixture(scope='module', autouse=True)
def report_worst_errors():
    yield
    if WORST:
        print('\nworst |GPU - fp64 closed form| per setting and sample type:')
        for key, err in sorted(WORST.items()):
            print('  %-20s %-8s %-8s %.3e' % ((key + ('',))[:3] + (err,)))


def upload(arr):
    return WavStream.from_array(arr.reshape(1, -1), 12000, 0, arr.size)


def cols(queries):
    return [np.array([q[k] for q in queries], np.int64) for k in range(4)]


def value_tol(n):
    return VALUE_TOL * max(1.0, np.sqrt(SHORT / n))


def check_curve(case, q, got, truth, where):
    err = np.abs(got.astype(np.float64) - truth)
    assert err.max() <= value_tol(case.queries[q][1]), (where, case, q, case.queries[q], float(err.max()), int(err.argmax()))
    sat = truth == 1.0
    assert (got[sat] == 1.0).all(), (where, case, q, np.nonzero(sat & (got != 1.0))[0][:5])
    return float(err.max())


def check_find(case, q, d, i, curve, truth, where):
    assert np.float32(d).view(np.uint32) == curve.min().view(np.uint32) and i == int(curve.argmin()), \
        (where, case, q, case.queries[q], float(d), int(i), float(curve.min()), int(curve.argmin()))
    assert abs(float(d) - truth.min()) <= value_tol(case.queries[q][1]), (where, case, q)
    assert truth[i] - truth.min() <= ARGMIN_TOL, (where, case, q)
    if q in case.expect:
        assert i == case.expect[q], (where, case, q, int(i), case.expect[q])


@pytest.mark.parametrize('s', SETTINGS, ids=[s.name for s in SETTINGS])
def test_every_case_against_the_closed_form(gpu_lib, setting, truths, s):
    setting(s)
    for case in CASES:
        img, tm = upload(case.image), upload(case.template)
        curves = img.match_curves(tm, *cols(case.queries))
        d, i = img.find_planned(tm, *cols(case.queries))
        img.close()
        tm.close()
        for q, truth in enumerate(truths[case.name]):
            key = (s.name, np.dtype(case.dtype).name)
            err = check_curve(case, q, curves[q], truth, s.name)
            if case.queries[q][1] >= SHORT:
                WORST[key] = max(WORST[key], err)
            else:
                WORST[key + ('n < %d' % SHORT,)] = max(WORST[key + ('n < %d' % SHORT,)], err)
            check_find(case, q, d[q], int(i[q]), curves[q], truth, s.name)


def test_degenerate_blocks_agree_bit_for_bit_across_packed_engines(gpu_lib, setting, truths):
    """The emulator's degenerate cases on the hardware: a periodic stream with more minima per lag block than a CTA has
    record slots, a zero template, silent blocks, two exact copies (the first wins).  Engines 2, 4 and 5 under both
    bodies return the same answers bit for bit, and the periodic stream's winner has the residue of its first copy."""
    cases = [c for c in CASES if c.family in ('periodic', 'silence', 'mirror')]
    ref = {}
    for engine in (2, 4, 5):
        for epi in (1, 3):
            setting(DEFAULTS._replace(engine=engine, epilogue=epi))
            for c in cases:
                img, tm = upload(c.image), upload(c.template)
                d, i = img.find_planned(tm, *cols(c.queries))
                img.close()
                tm.close()
                if c.name not in ref:
                    ref[c.name] = (d, i)
                assert np.array_equal(ref[c.name][0].view(np.uint32), d.view(np.uint32)), (c, engine, epi)
                assert np.array_equal(ref[c.name][1], i), (c, engine, epi)
    d, i = ref['flat_periodic']
    assert i[0] % 1000 == 500 and i[1] % 1000 == 345 and float(d.max()) <= 1e-6
    d, i = ref['flat_silence']
    assert d[0] == 1.0 and i[0] == 0 and i[2] == 33000 and d[3] == 1.0 and i[3] == 0
    d, i = ref['ladder_mirror']
    assert float(d.max()) <= 1e-6 and list(i) == [c.expect[q] for c in cases if c.name == 'ladder_mirror' for q in range(2)]


@pytest.mark.parametrize('s', [s for s in SETTINGS if s.max_parts > 1], ids=[s.name for s in SETTINGS if s.max_parts > 1])
def test_multi_stream_calls_interleave_the_cases(gpu_lib, setting, truths, s):
    """sb_find_multi / sb_match_curves_multi over one table holding every case's streams of a sample type, the queries
    of all cases interleaved: the same bars, and the answers of the single-stream calls bit for bit."""
    setting(s)
    for dtype in (np.uint8, np.float32):
        cases = [c for c in CASES if c.dtype == dtype]
        streams, rows, back = [], [], []
        for c in cases:
            streams += [upload(c.image), upload(c.template)]
        order = sorted(((q, ci) for ci, c in enumerate(cases) for q in range(len(c.queries))))
        for q, ci in order:                                      # round robin over the cases
            rows.append((2 * ci, 2 * ci + 1) + cases[ci].queries[q])
            back.append((ci, q))
        rows = np.array(rows, np.int64)
        table = (ctypes.c_void_p * len(streams))(*[x._handle.value for x in streams])
        islot, tslot = [np.ascontiguousarray(rows[:, k], np.int32) for k in (0, 1)]
        arrs = [np.ascontiguousarray(rows[:, k], np.int64) for k in range(2, 6)]
        ptrs = [islot.ctypes.data_as(_native.c_i32p), tslot.ctypes.data_as(_native.c_i32p)] + [a.ctypes.data_as(_native.c_i64p) for a in arrs]
        diff, idx = np.empty(len(rows), np.float32), np.empty(len(rows), np.int64)
        _native.check(gpu_lib.sb_find_multi(table, len(streams), len(rows), *ptrs, diff.ctypes.data_as(_native.c_f32p),
                                            idx.ctypes.data_as(_native.c_i64p)), 'sb_find_multi')
        cur = np.empty(int(arrs[3].sum()), np.float32)
        _native.check(gpu_lib.sb_match_curves_multi(table, len(streams), len(rows), *ptrs, cur.ctypes.data_as(_native.c_f32p)),
                      'sb_match_curves_multi')
        curves = np.split(cur, np.cumsum(arrs[3])[:-1])
        single = {}
        for ci, c in enumerate(cases):
            single[ci] = streams[2 * ci].find_planned(streams[2 * ci + 1], *cols(c.queries))
        for k, (ci, q) in enumerate(back):
            c = cases[ci]
            truth = truths[c.name][q]
            check_curve(c, q, curves[k], truth, s.name + '/multi')
            check_find(c, q, diff[k], int(idx[k]), curves[k], truth, s.name + '/multi')
            assert diff[k].view(np.uint32) == single[ci][0][q].view(np.uint32) and idx[k] == single[ci][1][q], (s.name, c, q)
        for x in streams:
            x.close()


# ---------------------------------------------------------------------------------------------------------------------
# history independence: block-spectrum rows are built on demand into pool memory that is recycled between streams
# ---------------------------------------------------------------------------------------------------------------------
def _history_case():
    return [c for c in CASES if c.name == 'ladder_g4e-06'][0]


def _run(img, tm, queries):
    d, i = img.find_planned(tm, *cols(queries))
    return d, i, img.match_curves(tm, *cols(queries))


def _same(a, b):
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
    for x, y in zip(a[2], b[2]):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


def _meets_bars(case, truths, res, where):
    for q, truth in enumerate(truths[case.name]):
        check_curve(case, q, res[2][q], truth, where)
        check_find(case, q, res[0][q], int(res[1][q]), res[2][q], truth, where)


@pytest.mark.parametrize('engine', [2, 4, 5, 1])
def test_answers_do_not_depend_on_which_rows_earlier_queries_built(gpu_lib, setting, truths, engine):
    setting(DEFAULTS._replace(engine=engine))
    case = _history_case()
    Q = case.queries
    img, tm = upload(case.image), upload(case.template)
    fresh = _run(img, tm, Q)
    img.close()
    _meets_bars(case, truths, fresh, 'fresh')
    # the same content again; warm-up queries build rows out of order: the middle, the far right, the far left
    img = upload(case.image)
    L = case.image.size
    for lag0 in (L // 2, L - 2000 - 1000, 0):
        img.find_planned(tm, [0], [1000], [lag0], [2000])
    _same(fresh, _run(img, tm, Q))
    img.close()
    # a stream of the same length with other audio, its rows built, then closed: the stream under test likely inherits
    # its pool blocks
    other = upload(cf.programme(L, 99))
    other.match_curves(tm, *cols(Q))
    other.find_planned(tm, *cols(Q))
    other.close()
    img = upload(case.image)
    res = _run(img, tm, Q)
    _meets_bars(case, truths, res, 'recycled')
    _same(fresh, res)
    img.close()
    tm.close()


def test_multi_stream_answers_do_not_depend_on_prebuilt_rows(gpu_lib, setting, truths):
    """Two image streams of the same case content, only the first pre-built (part of its rows, out of order); one
    multi-stream call over both: each answers what a fresh single-stream call answers, bit for bit."""
    setting(DEFAULTS)
    case = _history_case()
    Q = case.queries
    img, tm = upload(case.image), upload(case.template)
    fresh = _run(img, tm, Q)
    img.close()
    # recycled pool blocks with other content first
    other = upload(cf.programme(case.image.size, 98))
    other.find_planned(tm, *cols(Q))
    other.close()
    a, b = upload(case.image), upload(case.image)
    a.find_planned(tm, [0], [1000], [case.image.size // 2], [2000])
    a.find_planned(tm, [0], [1000], [0], [2000])
    streams = [a, tm, b]
    rows = np.array([(0 if k % 2 else 2, 1) + q for k in range(2) for q in Q], np.int64)
    table = (ctypes.c_void_p * 3)(*[x._handle.value for x in streams])
    islot, tslot = [np.ascontiguousarray(rows[:, k], np.int32) for k in (0, 1)]
    arrs = [np.ascontiguousarray(rows[:, k], np.int64) for k in range(2, 6)]
    ptrs = [islot.ctypes.data_as(_native.c_i32p), tslot.ctypes.data_as(_native.c_i32p)] + [x.ctypes.data_as(_native.c_i64p) for x in arrs]
    diff, idx = np.empty(len(rows), np.float32), np.empty(len(rows), np.int64)
    _native.check(gpu_lib.sb_find_multi(table, 3, len(rows), *ptrs, diff.ctypes.data_as(_native.c_f32p),
                                        idx.ctypes.data_as(_native.c_i64p)), 'sb_find_multi')
    for k in range(len(rows)):
        q = k % len(Q)
        assert diff[k].view(np.uint32) == fresh[0][q].view(np.uint32) and idx[k] == fresh[1][q], (k, q)
    for x in streams:
        x.close()
