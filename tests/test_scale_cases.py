"""The scale inputs of tests/scale_cases.py checked on the CPU: every stored gap in exact integer arithmetic, every planted
copy the first minimum of its query's fp64 truth, the model's cuts where the ladders need them, and the batch reaching
every launch-level cut it is meant to cross."""
import numpy as np
import pytest

from tests import scale_cases as sc

B = sc.B


@pytest.fixture(scope='module')
def scale():
    return sc.build()


def ladders(scale):
    for name, batch in (('config3', scale.config3), ('long', scale.long)):
        for q, lad in sorted(batch.ladders.items()):
            yield name, batch, q, lad


def test_stored_gaps_are_exact(scale):
    for name, batch, q, lad in ladders(scale):
        toff, n, lag0, _ = batch.rows[q]
        t = scale.template[toff:toff + n].astype(np.int64)
        exact = lad.p0 if lad.kind == 'rgap' else lad.p1
        assert np.array_equal(scale.image[exact:exact + n], scale.template[toff:toff + n]), (name, q)
        w0 = scale.image[lad.p0 + lad.p1 - exact:lad.p0 + lad.p1 - exact + n].astype(np.int64)
        if lad.kind == 'mirror':
            assert np.array_equal(w0, t) and batch.gap[q] == 0.0, (name, q)
            tsq = int(np.dot(t, t))
            assert tsq % 2 ** (int(np.floor(np.log2(tsq))) - 23) == 0          # sum T^2 exact in float32
            continue
        assert np.dot(w0, w0) == np.dot(t, t)
        g = batch.gap[q]
        assert g >= lad.g and abs(float(np.sum((w0 - t) ** 2)) / float(np.dot(t, t)) - g) <= 1e-12 * g, (name, q)


def test_every_planted_copy_is_the_first_minimum_of_its_truth(scale):
    for name, batch, q, lad in ladders(scale):
        truth = sc.closed_form(scale.image, scale.template, batch.rows[q])
        want = batch.expect[q]
        if lad.kind == 'mirror':
            assert list(np.nonzero(truth <= 1e-9)[0]) == [lad.p0 - lad.lag0, lad.p1 - lad.lag0] and want == lad.p0 - lad.lag0
            continue
        assert int(truth.argmin()) == want == lad.p0 + lad.p1 - lad.swapped - lad.lag0, (name, q)
        near = np.sort(truth)[:3]
        assert abs((near[1] - near[0]) - batch.gap[q]) <= 1e-12 * batch.gap[q] + 2e-15, (name, q, near)
        assert int(np.argsort(truth)[1]) == lad.swapped - lad.lag0 and near[2] > 1e-3, (name, q)


def test_known_lags_of_events_are_their_first_minimum(scale):
    """The copy construction on a sample of events, the first and last (windows clipped at the stream's ends) and the
    30 s templates of the blocked class among them."""
    b = scale.config3
    ev = [q for q in range(len(b.rows)) if b.event[q] >= 0]
    pick = [ev[0], ev[-1]] + ev[1:-1:1500]
    for batch, qs in ((b, pick), (scale.long, [0, len(scale.long.rows) - 1, len(scale.long.rows) - 7])):
        for q in qs:
            assert q in batch.expect, q
            truth = sc.closed_form(scale.image, scale.template, batch.rows[q])
            assert int(truth.argmin()) == batch.expect[q], q
            assert truth[batch.expect[q]] < 1e-3 and np.partition(truth, 1)[1] > 10 * truth.min()
    first, last = b.rows[ev[0]], b.rows[ev[-1]]
    assert first[2] == 0 and last[2] + last[3] - 1 + last[1] == sc.TOTAL


def test_value_at_matches_the_closed_form(scale):
    b = scale.config3
    for q in (0, len(b.rows) - 1):
        truth = sc.closed_form(scale.image, scale.template, b.rows[q])
        for i in (0, b.expect[q], len(truth) - 1, 12345):
            assert abs(sc.value_at(scale.image, scale.template, b.rows[q], i) - truth[i]) <= 1e-12


def test_the_model_puts_every_ladder_across_its_cut(scale):
    for name, batch, q, lad in ladders(scale):
        if lad.cut is None:
            continue
        engine, c = lad.cut
        m = batch.model(engine)
        assert c in m.cuts
        pos = int(m.pos_of[q])
        u0, u1 = m.unit_of_lag(pos, lad.p0), m.unit_of_lag(pos, lad.p1)
        assert (u0, u1) == (c - 1, c), (name, q, u0, u1, c)
        (s0, k0), (s1, k1) = m.chunk_of(u0), m.chunk_of(u1)
        assert s0 == s1 and k1 == k0 + 1, (name, q)
        if m.use_pairs:                       # the second half of the last pair of chunk c, the first of chunk c + 1
            k = int(m.k0[pos])
            assert (lad.p0 // B - k) % 2 == 1 and (lad.p1 // B - k) % 2 == 0


def test_the_batches_cross_every_launch_level_cut(scale):
    b = scale.config3
    m2, m4 = b.model(2), b.model(4)
    assert not m2.use_pairs and m4.use_pairs and len(b.rows) > sc.EVENTS
    direct = [s for s in m2.superchunks if s[0] == 0]
    assert len(direct) >= 2                                         # a super-chunk boundary
    first = [c for c in m2.cuts if c < m2.units[direct[0][2]]]
    assert len(first) >= 2                                          # two record cuts inside one super-chunk
    assert m4.cuts                                                  # a pair cut
    assert m2.finish_launches == len(m2.cuts) + len(direct)
    cut_ladders = {lad.cut for lad in b.ladders.values() if lad.cut}
    assert cut_ladders == {(2, c) for c in m2.cuts} | {(4, c) for c in m4.cuts}
    kinds = {(lad.cut[0], lad.kind) for lad in b.ladders.values() if lad.cut}
    assert {(2, 'gap'), (2, 'rgap'), (2, 'mirror'), (4, 'rgap')} <= kinds
    # ladders past 2^24 and 2^25 and one ending on the stream's last lag
    fixed = [lad for lad in b.ladders.values() if lad.cut is None]
    assert any(lad.p0 < 2 ** 24 <= lad.p1 for lad in fixed) and any(lad.p0 < 2 ** 25 <= lad.p1 for lad in fixed)
    assert any(lad.p1 == lad.lag0 + lad.nlags - 1 == sc.TOTAL - sc.LADDER_N for lad in fixed)
    # events that lost their copy to planting are few, and known
    assert sum(1 for q in b.expect if b.event[q] >= 0) > 0.99 * sc.EVENTS
    # the long-template batch: engine 2 picks pairs, more than one record chunk of them, three product-buffer chunks
    lm = scale.long.model(2)
    assert lm.use_pairs and lm.group_base[lm.n_direct] > sc.RUN_CHUNK and len(lm.cuts) >= 1
    assert lm.n_direct == len(scale.long.rows) - 12 and (lm.P[lm.n_direct:] == 22).all()
    assert len(lm.premac_chunks) == 3
    assert {lad.kind for lad in scale.long.ladders.values()} == {'gap'}
