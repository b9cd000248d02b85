"""The host mirror of the loader (DownmixedWavFile + WavStream._load) against the oracle restatement of the reference
loader on every case of tests/loader_cases.py, bit for bit: the samples, sample_count, padding_size and the two clip
values.  Where the reference raises (case.quirk), the oracle must raise too, and the mirror must equal the oracle with
the documented rule applied (DESIGN.md section 2).  No GPU."""
import numpy as np
import pytest

from sushi_b200 import wavstream
from sushi_b200.wavstream import WavStream
from tests import loader_cases as lc

CASES = lc.all_cases()
SEEN = {}


def host_load(path, case):
    f = wavstream.DownmixedWavFile(path)
    try:
        s = object.__new__(WavStream)
        s._handle = None
        s._load(f, case.sample_rate, case.sample_type)
    finally:
        f.close()
    return s


def truth(case, path):
    """The oracle's answer for this case, after checking that it raises exactly where the case says it does."""
    if case.quirk is None:
        return lc.oracle_load(case, path)
    with pytest.raises(Exception):
        lc.oracle_load(case, path)
    return lc.oracle_load(case, path, documented=True)


def same_f32(a, b):
    return np.array_equal(np.float32(a), np.float32(b), equal_nan=True)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_host_loader_matches_oracle(tmp_path, case):
    path = case.write(tmp_path)
    padded, want, count, pad, lo, hi = truth(case, path)
    SEEN[case.name] = (lc.branches(padded), lc.exact_quant_hits(padded, lo, hi))
    s = host_load(path, case)
    assert (int(s.sample_count), s.padding_size) == (count, pad) == (case.sample_count, 10 * case.framerate)
    assert s.data.shape == want.shape == (1, case.padded_length) and s.data.dtype == want.dtype
    assert np.array_equal(s.data, want, equal_nan=want.dtype == np.float32)
    assert same_f32(s.min_value, lo) and same_f32(s.max_value, hi)


def test_loader_cases_cover_every_median_branch(tmp_path):
    """Every path of the GPU median selection, and a padded array whose quantisation lands exactly on integers, is
    taken by some case (the geometry coverage is asserted by loader_cases.all_cases itself)."""
    for case in CASES:
        if case.name not in SEEN:
            path = case.write(tmp_path)
            padded, _, _, _, lo, hi = lc.oracle_load(case, path, documented=case.quirk is not None)
            SEEN[case.name] = (lc.branches(padded), lc.exact_quant_hits(padded, lo, hi))
    lc.assert_coverage(SEEN)


def test_zero_sample_last_chunk_takes_no_sample(tmp_path):
    """One leftover frame at 48 kHz resamples to no sample: the reference's cv2.resize raises; the host loader writes
    nothing for it and leaves the one-sample gap before the tail padding at zero."""
    case = lc.make_case('zero_chunk_probe', 48000, 1, 2, 48001, 'dc_pos', sample_type='float32')
    assert case.quirk == 'zero_chunk'
    path = case.write(tmp_path)
    padded, _, count, pad = lc.oracle_load(case, path, documented=True)[:4]
    assert count == 12001 and padded[0, pad + 12000] == 0 and np.all(padded[0, pad:pad + 12000] > 0)
    s = host_load(path, case)
    assert s.data.shape == padded.shape
