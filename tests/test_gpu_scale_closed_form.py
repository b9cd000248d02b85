"""The matcher against the fp64 closed form at BASELINE size (tests/scale_cases.py: 10 000 config-3 events on a pair
of 90-minute streams, near-tie ladders planted across every launch-level cut, a long-template batch), with the bars of
tests/test_gpu_closed_form.py.

* the k_finish_runs launches (one per record chunk) are the ones the model of run_batch predicts;
* every answer of the default run: |diff - fp64 value at the returned index| <= 1e-6, and the known index wherever the
  event kept its copy or a ladder was planted;
* about 30 chosen queries (every straddler of a record cut, super-chunk boundary or pair cut, in caller order and
  reversed; the first and last events; windows across 2^24 and 2^25; every ladder): the whole curve and find;
* batch invariance, bit for bit: reversed caller order, max_parts 997, engines 4 and 5, epilogue 1, a multi-stream
  call over two 90-minute pairs, parallel.ShardedMatcher (the path bench.py times);
* float32 copies of the image, one of them at two levels (a hard case for the whole-stream centring);
* the long-template batch: pairs chosen by engine 2 across a record cut, the blocked class across three product
  buffers.

The worst |GPU - fp64| per scenario, the launch counts and the file's wall time are printed at the end (-s)."""
import collections
import ctypes
import time

import numpy as np
import pytest

from sushi_b200 import WavStream, _native, parallel
from tests import scale_cases as sc
from tests.test_gpu_closed_form import check_curve, check_find, value_tol

pytestmark = pytest.mark.gpu

B = sc.B
WORST = collections.defaultdict(float)
REPORT = []


class View(object):
    """What check_curve / check_find read of a case: its queries and known first minima."""

    def __init__(self, name, queries, expect):
        self.name, self.queries, self.expect = name, queries, expect

    def __repr__(self):
        return 'Scale(%s)' % self.name


def configure(lib, engine=2, epilogue=3, max_parts=sc.MAX_PARTS):
    for rc in (lib.sb_set_block_size(B), lib.sb_set_hop_mode(1), lib.sb_set_premac_mode(0), lib.sb_set_engine(engine),
               lib.sb_set_epilogue(epilogue), lib.sb_set_max_parts(max_parts)):
        _native.check(rc)


def upload(arr):
    return WavStream.from_array(arr.reshape(1, -1), sc.RATE, sc.PAD, sc.COUNT)


@pytest.fixture(scope='module', autouse=True)
def report():
    t0 = time.time()
    yield
    print('\nk_finish_runs launches (predicted / observed):')
    for line in REPORT:
        print('  ' + line)
    print('worst |GPU - fp64 closed form| per scenario:')
    for key, err in sorted(WORST.items()):
        print('  %-36s %.3e' % (key, err))
    print('wall time of the module: %.1f s' % (time.time() - t0))


@pytest.fixture(scope='module')
def scale():
    return sc.build()


@pytest.fixture(scope='module')
def pair(gpu_lib, scale):
    img, tm = upload(scale.image), upload(scale.template)
    yield img, tm
    img.close()
    tm.close()
    configure(gpu_lib)


def counted(lib, img, tm, cols):
    before = lib.sb_launch_count()
    d, i = img.find_planned(tm, *cols)
    return d, i, lib.sb_launch_count() - before


@pytest.fixture(scope='module')
def default_run(gpu_lib, pair, scale):
    """The config-3 batch under the default settings, after one warm-up call that builds the block spectra."""
    img, tm = pair
    configure(gpu_lib)
    cols = scale.config3.cols()
    img.find_planned(tm, *cols)
    return counted(gpu_lib, img, tm, cols)


def same(a, b, where):
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)), (where, np.nonzero(a[0].view(np.uint32) != b[0].view(np.uint32))[0][:5])
    assert np.array_equal(a[1], b[1]), (where, np.nonzero(a[1] != b[1])[0][:5])


def chosen(scale):
    """Caller indices of the config-3 queries held to the full closed form."""
    b = scale.config3
    out = set(b.ladders)
    out |= {q + 1 for q, lad in b.ladders.items() if lad.cut}               # the query the ladder pushed off its cut
    m = b.model(2)
    for cls, qb, qe in m.superchunks:
        if cls == 0 and qe < m.n_direct:
            out |= {int(m.order[qe - 1]), int(m.order[qe])}                 # the two sides of a super-chunk boundary
    rev = b.cols()
    rm = sc.BatchModel(*[c[::-1] for c in rev[1:]], engine=2)
    rm4 = sc.BatchModel(*[c[::-1] for c in rev[1:]], engine=4)
    n = len(b.rows)
    for mm in (rm, rm4):
        out |= {n - 1 - int(mm.order[mm.owner(c)]) for c in mm.cuts}       # straddlers in reversed order
    ev = [q for q in range(n) if b.event[q] >= 0]
    out |= {ev[0], ev[-1]}
    for p in (1 << 24, 1 << 25):
        out.add(next(q for q in ev if b.rows[q][2] < p < b.rows[q][2] + b.rows[q][3]))
    return sorted(out)


def hold_to_closed_form(img, tm, image, template, view, rows, qs, d, i, scenario):
    """Whole curves of the queries qs (one match_curves call) against the closed form; find (d, i) against them."""
    cols = [np.array([rows[q][k] for q in qs], np.int64) for k in range(4)]
    curves = img.match_curves(tm, *cols)
    for k, q in enumerate(qs):
        truth = sc.closed_form(image, template, rows[q])
        err = check_curve(view, q, curves[k], truth, scenario)
        WORST[scenario + ' (curves)'] = max(WORST[scenario + ' (curves)'], err)
        check_find(view, q, d[q], int(i[q]), curves[k], truth, scenario)


def value_at_every_index(image, template, view, rows, d, i, scenario):
    worst = 0.0
    for q, row in enumerate(rows):
        v = sc.value_at(image, template, row, int(i[q]))
        err = abs(float(d[q]) - v)
        assert err <= value_tol(row[1]), (scenario, q, row, float(d[q]), v)
        if q in view.expect:
            assert int(i[q]) == view.expect[q], (scenario, q, row, int(i[q]), view.expect[q])
        worst = max(worst, err)
    WORST[scenario + ' (value at index)'] = max(WORST[scenario + ' (value at index)'], worst)


# ---------------------------------------------------------------------------------------------------------------------
# uint8, config 3
# ---------------------------------------------------------------------------------------------------------------------
def test_record_cuts_are_crossed(gpu_lib, pair, scale, default_run):
    """Each record chunk adds one k_finish_runs launch: the count under body 3 minus the count under body 1 (which writes
    no records) is the number of chunks the model predicts, for single lag blocks (engine 2) and pairs (engine 4)."""
    img, tm = pair
    cols = scale.config3.cols()
    for engine in (2, 4):
        configure(gpu_lib, engine=engine)
        img.find_planned(tm, *cols)
        r3 = default_run if engine == 2 else counted(gpu_lib, img, tm, cols)
        configure(gpu_lib, engine=engine, epilogue=1)
        r1 = counted(gpu_lib, img, tm, cols)
        m = scale.config3.model(engine)
        REPORT.append('config 3, engine %d (%s): %d / %d' % (engine, 'pairs' if m.use_pairs else 'lag blocks',
                                                              m.finish_launches, r3[2] - r1[2]))
        assert r3[2] - r1[2] == m.finish_launches
        assert m.finish_launches > len([s for s in m.superchunks if s[0] == 0])
        same(r3, default_run, 'engine %d' % engine)
        same(r1, default_run, 'engine %d, epilogue 1' % engine)
    configure(gpu_lib)


def test_every_answer_against_the_fp64_value_at_its_index(scale, default_run):
    b = scale.config3
    value_at_every_index(scale.image, scale.template, View('config3', b.queries, b.expect), b.queries,
                         default_run[0], default_run[1], 'uint8 config 3')


def test_chosen_queries_against_the_whole_closed_form(pair, scale, default_run):
    img, tm = pair
    b = scale.config3
    qs = chosen(scale)
    assert len(qs) >= 20
    hold_to_closed_form(img, tm, scale.image, scale.template, View('config3', b.queries, b.expect), b.queries, qs,
                        default_run[0], default_run[1], 'uint8 config 3')


@pytest.mark.parametrize('variant', ['reversed', 'max_parts_997', 'engine4', 'engine5', 'epilogue1'])
def test_answers_do_not_depend_on_the_batch(gpu_lib, pair, scale, default_run, variant):
    img, tm = pair
    cols = scale.config3.cols()
    if variant == 'reversed':
        configure(gpu_lib)
        d, i = img.find_planned(tm, *[c[::-1] for c in cols])
        got = (d[::-1].copy(), i[::-1].copy())
    else:
        configure(gpu_lib, **{'max_parts_997': dict(max_parts=997), 'engine4': dict(engine=4), 'engine5': dict(engine=5),
                              'epilogue1': dict(epilogue=1)}[variant])
        got = img.find_planned(tm, *cols)
    configure(gpu_lib)
    same(got, default_run, variant)


def test_multi_stream_call_over_two_90_minute_pairs(gpu_lib, pair, scale, default_run):
    """sb_find_multi over this pair and a second one with other content, queries interleaved (more than 2^19 lag
    blocks): every answer is its single-stream answer, bit for bit."""
    img, tm = pair
    configure(gpu_lib)
    rows = scale.config3.cols()
    other = sc.programme_long(sc.TOTAL, 77)
    img2, tm2 = upload(other), upload(sc.shifted_noisy_copy(other, sc.SHIFT, sc.NOISE, 78))
    single2 = img2.find_planned(tm2, *rows)
    n = len(rows[0])
    streams = [img, tm, img2, tm2]
    islot = np.tile(np.array([0, 2], np.int32), n)
    tslot = islot + 1
    arrs = [np.repeat(c, 2) for c in rows]
    assert (((arrs[2] + arrs[3] - 1) // B) - arrs[2] // B + 1).sum() > sc.RUN_CHUNK
    table = (ctypes.c_void_p * 4)(*[x._handle.value for x in streams])
    diff, idx = np.empty(2 * n, np.float32), np.empty(2 * n, np.int64)
    _native.check(gpu_lib.sb_find_multi(table, 4, 2 * n, islot.ctypes.data_as(_native.c_i32p), tslot.ctypes.data_as(_native.c_i32p),
                                        *[a.ctypes.data_as(_native.c_i64p) for a in arrs],
                                        diff.ctypes.data_as(_native.c_f32p), idx.ctypes.data_as(_native.c_i64p)), 'sb_find_multi')
    img2.close()
    tm2.close()
    same((diff[0::2], idx[0::2]), default_run, 'multi, first pair')
    same((diff[1::2], idx[1::2]), single2, 'multi, second pair')


def test_sharded_matcher_equals_the_direct_call(gpu_lib, pair, scale, default_run):
    """parallel.ShardedMatcher over SingleComm + DeviceBackend (sb_find_batch_device) on the 10 000 events."""
    img, tm = pair
    configure(gpu_lib)
    b = scale.config3
    be = parallel.DeviceBackend(gpu_lib)
    m = parallel.ShardedMatcher(parallel.SingleComm(be), be)
    try:
        m.set_streams(tm, img)
        m.find_batch(scale.starts, scale.ends, scale.starts, np.full(sc.EVENTS, sc.WINDOW))
        got = m.gather_results()
    finally:
        be.release()
    ev = np.array([q for q in range(len(b.rows)) if b.event[q] >= 0])
    assert np.array_equal(np.array(b.event)[ev], np.arange(sc.EVENTS))
    same(got, (default_run[0][ev], default_run[1][ev]), 'sharded')


# ---------------------------------------------------------------------------------------------------------------------
# float32
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('levels', [None, (0.2, 0.8)], ids=['unit', 'two_levels'])
def test_float32_at_baseline_size(gpu_lib, scale, levels):
    """The same image as float32: every answer against the fp64 value at its index (and the known index of every event
    that kept its copy), the chosen queries against the whole closed form."""
    configure(gpu_lib)
    b = scale.config3
    image = sc.to_float32(scale.image, levels)
    template = sc.to_float32(scale.template, levels, shift=sc.SHIFT)
    name = 'float32 ' + ('two levels' if levels else 'unit')
    expect = {q: v for q, v in b.expect.items() if b.event[q] >= 0}
    view = View(name, b.queries, expect)
    img, tm = upload(image), upload(template)
    try:
        d, i = img.find_planned(tm, *b.cols())
        value_at_every_index(image, template, view, b.queries, d, i, name)
        hold_to_closed_form(img, tm, image, template, view, b.queries, chosen(scale), d, i, name)
    finally:
        img.close()
        tm.close()


# ---------------------------------------------------------------------------------------------------------------------
# long templates
# ---------------------------------------------------------------------------------------------------------------------
def test_long_template_batch(gpu_lib, pair, scale):
    img, tm = pair
    lb = scale.long
    cols = lb.cols()
    m = lb.model(2)
    assert m.use_pairs and m.cuts
    configure(gpu_lib)
    img.find_planned(tm, *cols)
    r3 = counted(gpu_lib, img, tm, cols)
    configure(gpu_lib, epilogue=1)
    r1 = counted(gpu_lib, img, tm, cols)
    configure(gpu_lib)
    # engine 2 chose pairs: one finish launch per record chunk of pairs (lag blocks would need more chunks)
    items = int(m.item_base[m.n_direct])
    REPORT.append('long templates, engine 2 (pairs): %d / %d (lag blocks would take %d)'
                  % (m.finish_launches, r3[2] - r1[2], (items + sc.RUN_CHUNK - 1) // sc.RUN_CHUNK))
    assert r3[2] - r1[2] == m.finish_launches < (items + sc.RUN_CHUNK - 1) // sc.RUN_CHUNK
    same(r1, r3, 'long, epilogue 1')
    view = View('long', lb.queries, lb.expect)
    value_at_every_index(scale.image, scale.template, view, lb.queries, r3[0], r3[1], 'uint8 long templates')
    # the queries at the pair cut, and three of the blocked class, against the whole closed form
    cut = {int(m.order[m.owner(c - 1)]) for c in m.cuts} | {int(m.order[m.owner(c)]) for c in m.cuts}
    cut |= {q + 1 for q, lad in lb.ladders.items()}
    blocked = [int(m.order[p]) for p in range(m.n_direct, m.count)]
    hold_to_closed_form(img, tm, scale.image, scale.template, view, lb.queries, sorted(cut), r3[0], r3[1],
                        'uint8 long, pair cut')
    hold_to_closed_form(img, tm, scale.image, scale.template, view, lb.queries, blocked[3::4][:3], r3[0], r3[1],
                        'uint8 long, blocked class')
    # the blocked class asked one query at a time
    for q in blocked:
        d, i = img.find_planned(tm, *[[c[q]] for c in cols])
        same((d, i), (r3[0][q:q + 1], r3[1][q:q + 1]), 'blocked query %d alone' % q)
