"""The near-tie ladder and the flat curves of tests/closed_form_cases.py through the CPU emulator of the packed kernels
(tests/test_kernel_emulation.py): one CTA per lag block and per pair, the first body and the third one with and without
records.  The same bars as the GPU test (tests/test_gpu_closed_form.py): every lag within 1e-6 of the fp64 closed form,
saturated lags exactly 1, the screened answer equal bit for bit to the minimum and first argmin of the kernel's own
curve, the exact copy of a near-tie found at its exact index, and every variant equal to every other bit for bit."""
import numpy as np
import pytest

from tests import closed_form_cases as cf
from tests.test_kernel_emulation import Case, emu  # noqa: F401  (the module-scoped library fixture)

VALUE_TOL = 1e-6
VARIANTS = [(kernel, epi, records) for kernel in (0, 1) for epi, records in ((1, False), (3, False), (3, True))]

CASES = {c.name: c for c in cf.near_tie_cases() + cf.flat_cases()}


def check_curves(case, cur):
    off = 0
    for q, t in enumerate(case.truth()):
        got = cur[off:off + t.size]
        off += t.size
        assert not np.isnan(got).any()
        assert np.abs(got.astype(np.float64) - t).max() <= VALUE_TOL, (case, q, np.abs(got - t).max())
        assert (got[t == 1.0] == 1.0).all(), (case, q)


@pytest.mark.parametrize('name', sorted(CASES))
def test_emulated_closed_form_cases(emu, name):  # noqa: F811
    case = CASES[name]
    c = Case(emu, case.image, case.template, case.queries, case.dtype)
    ref = None
    for kernel, epi, records in VARIANTS:
        d_c, i_c, cur = c.run(kernel, epi, curves=True)
        check_curves(case, cur)
        d, i, _ = c.run(kernel, epi, curves=False, records=records)
        off = 0
        for q, (_, _, _, nlags) in enumerate(case.queries):
            got = cur[off:off + nlags]
            off += nlags
            # the screening lost nothing: the minimum and first argmin of the kernel's own curve, bit for bit
            assert d[q].view(np.uint32) == got.min().view(np.uint32) and i[q] == int(got.argmin()), (case, q, kernel, epi, records)
        for q, want in case.expect.items():
            assert i[q] == want, (case, q, kernel, epi, records, i[q], want)
        ref = ref or (d, i, cur)
        assert np.array_equal(ref[0].view(np.uint32), d.view(np.uint32)) and np.array_equal(ref[1], i), (kernel, epi, records)
        assert np.array_equal(ref[2].view(np.uint32), cur.view(np.uint32))
        if records and case.family == 'periodic':
            assert c.last_record_counts.max() == emu.emu_run_slots()         # the record slots did overflow
    if case.family == 'mirror':
        assert float(ref[0].max()) <= 1e-6                                  # two exact copies: the first index wins (above)
    if case.family == 'periodic':
        assert ref[1][0] % 1000 == 500 and ref[1][1] % 1000 == 345
