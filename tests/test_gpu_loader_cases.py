"""The GPU loader (sb_load_pcm + sb_normalise behind WavStream(path)) against the oracle restatement of the reference
loader and against the host mirror, bit for bit, on every case of tests/loader_cases.py: the samples, sample_count,
padding_size and the two clip values.  Where the reference raises (case.quirk) the truth is the oracle with the
documented rule applied (DESIGN.md section 2); tests/test_loader_cases.py checks that the oracle does raise there."""
import numpy as np
import pytest

from sushi_b200 import SushiError
from sushi_b200.wavstream import WavStream
from tests import loader_cases as lc
from tests.test_loader_cases import host_load, same_f32

pytestmark = pytest.mark.gpu

CASES = lc.all_cases()


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_gpu_loader_matches_oracle_and_host(gpu_lib, tmp_path, case):
    path = case.write(tmp_path)
    _, want, count, pad, lo, hi = lc.oracle_load(case, path, documented=case.quirk is not None)
    s = WavStream(path, case.sample_rate, case.sample_type)
    try:
        assert (int(s.sample_count), s.padding_size, s.sample_rate) == (count, pad, case.sample_rate)
        assert s.data.shape == want.shape and s.data.dtype == want.dtype
        nan = want.dtype == np.float32
        assert np.array_equal(s.data, want, equal_nan=nan), int(np.count_nonzero(s.data != want))
        assert same_f32(s.min_value, lo) and same_f32(s.max_value, hi), (s.min_value, lo, s.max_value, hi)
        h = host_load(path, case)
        assert np.array_equal(s.data, h.data, equal_nan=nan)
        assert same_f32(s.min_value, h.min_value) and same_f32(s.max_value, h.max_value)
    finally:
        s.close()


def test_gpu_loader_rejects_more_than_64_channels(gpu_lib, tmp_path):
    """The GPU median selection keeps a fine histogram of 32 x channels bins in shared memory, at most 2048 wide: a
    65-channel file is refused with the limit in the message.  The reference and the host mirror accept it (a
    deliberate difference, DESIGN.md section 2)."""
    case = lc.make_case('ch65', 48000, lc.MAX_CHANNELS + 1, 2, 4800, 'programme')
    path = case.write(tmp_path)
    with pytest.raises(SushiError, match='at most 64'):
        WavStream(path, 12000, 'uint8')
    want = lc.oracle_load(case, path)[1]
    assert np.array_equal(host_load(path, case).data, want)
