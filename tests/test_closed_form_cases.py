"""The case generator of tests/closed_form_cases.py checked against its own truth, on the CPU: every stored gap is what
the fp64 closed form gives at the planted copies, and the first minimum of the truth is the planted copy."""
import numpy as np
import pytest

from tests import closed_form_cases as cf


@pytest.fixture(scope='module')
def ladder():
    return cf.near_tie_cases()


def test_ladder_gaps_are_exact_and_the_exact_copy_is_the_minimum(ladder):
    placed = 0
    for case in ladder:
        truth = case.truth()
        for q, want in case.expect.items():
            t = truth[q]
            if case.family == 'mirror':
                # two exact copies: both at 0 up to fp64 rounding, nothing else near
                p1 = int(np.nonzero(t <= 1e-9)[0][-1])
                assert list(np.nonzero(t <= 1e-9)[0]) == [want, p1] and p1 > want, (case, q)
                continue
            g = case.gap[q]
            assert g >= min(cf.GAPS) and int(t.argmin()) == want, (case, q)
            near = np.sort(t)[:2]
            p0 = int(np.argsort(t)[1])
            assert p0 < want, (case, q, p0, want)                      # the perturbed copy comes first
            # the gap in exact integer arithmetic: equal window energies, so the value is sum (W - T)^2 / sum T^2
            toff, n, lag0, _ = case.queries[q]
            tm = case.template[toff:toff + n].astype(np.int64)
            w = case.image[lag0 + p0:lag0 + p0 + n].astype(np.int64)
            assert np.dot(w, w) == np.dot(tm, tm)
            assert abs(float(np.sum((w - tm) ** 2)) / float(np.dot(tm, tm)) - g) <= 1e-12 * g
            # and in the fp64 closed form, whose FFT leaves ~1e-16 of absolute noise on the curve
            assert abs((near[1] - near[0]) - g) <= 1e-12 * g + 2e-15, (case, q, near, g)
            placed += 1
    assert placed == len(cf.GAPS) * len(cf.PLACEMENTS)


def test_sub_resolution_rung_values(ladder):
    """The copies of the bottom rung sit at 2 (r0 + k) / sum T^2 for the planned steps k, and nothing else comes near."""
    case = [c for c in ladder if c.family == 'fine'][0]
    t = case.truth()[0]
    tm = case.template.astype(np.int64)
    tsq = float(np.dot(tm, tm))
    low = np.sort(t)[:len(cf.FINE_STEPS)]
    r0 = round(1e-5 * tsq / 2)
    want = np.sort(2.0 * (r0 + np.array(cf.FINE_STEPS)) / tsq)
    assert np.abs(low - want).max() <= 2e-15
    assert np.sort(t)[len(cf.FINE_STEPS)] > 1e-3


def test_ladder_placements_land_where_their_names_say():
    """The geometry the placements target: lags counted from the start of the stream, runs of 8, warps of 1024, lag
    blocks of B, pairs of lag blocks counted from the query's first lag block."""
    B = cf.B
    for name, p0, p1, lag0, nlags in cf.PLACEMENTS:
        p1 = p0 + 5 if p1 is None else p1
        k0, k1 = p0 // B, p1 // B
        pair = lambda p: (p // B - lag0 // B) // 2
        if name == 'run':
            assert p0 // 8 == p1 // 8
        elif name == 'warp':
            assert p0 // 1024 == p1 // 1024 and p0 // 32 != p1 // 32
        elif name == 'warps':
            assert k0 == k1 and p0 // 1024 != p1 // 1024
        elif name == 'pair':
            assert k1 == k0 + 1 and pair(p0) == pair(p1)
        else:
            assert k1 != k0 and pair(p0) != pair(p1)
    assert (cf.LADDER_LENGTH + B - 1) // B <= 6


def test_every_case_is_well_formed_and_pins_its_known_answers():
    cases = cf.all_cases()
    names = [c.name for c in cases]
    assert len(set(names)) == len(names)
    for case in cases:
        assert case.image.dtype == case.dtype and case.template.dtype == case.dtype
        if case.family in ('ladder', 'mirror'):
            continue                                  # above
        truth = case.truth()
        for q, want in case.expect.items():
            assert int(truth[q].argmin()) == want, (case, q)
    grid = [c for c in cases if c.family == 'edge']
    lens = {q[1] for c in grid for q in c.queries}
    assert {1, 2, 11 * cf.B + 1, 21 * cf.B + 5} <= lens
    assert any(q[2] + q[3] - 1 + q[1] == c.image.size for c in grid for q in c.queries)     # ends on the last lag
