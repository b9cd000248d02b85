"""sb_pcm_swr on the GPU (k_swr_mix and k_swr_resample) against libswresample itself (tests/ref_swr.py, its FMA3
path), bit for bit with the output length: every case tests/test_swr_cases.py holds the CPU build of sb_swr.cuh to
(its rates, layouts, lengths and values, with its case lists and signals); input lengths chosen with the plan so that
the output ends on either side of a tile boundary at tiles of 256, 128 and 64 outputs; the narrow tiles with stereo and
8-channel layouts, at exact and inexact ratios; an input too short for any output; the integer downmix at 60 s of
48 kHz, past one pass of its grid-stride loop, in each of its three forms; 90 minutes of 44.1 kHz stereo through the
40-phase bank and through linear interpolation at an inexact ratio; and a rate pair the resampler refuses."""
import ctypes

import numpy as np
import pytest

from sushi_b200 import SushiError, _native
from tests import ref_swr
from tests.test_gpu_ffmpeg_audio import swr_device, swr_handle
from tests.test_swr_cases import IN_RATES, LAYOUTS, LENGTHS, OUT_RATES, emu, plan, signal, tiles  # noqa: F401 (emu)

pytestmark = pytest.mark.gpu


def swr_frames(pcm, mask, rate, sample_rate):
    """sb_pcm_swr's output frame count, from sb_pcm_info alone (sb_pcm_load needs at least one frame)"""
    out, frames = swr_handle(pcm, mask, rate, sample_rate)
    _native.lib().sb_pcm_destroy(out)
    return frames


def check(pcm, mask, in_rate, out_rate, chunk=4096, big=False):
    want = ref_swr.convert(pcm, mask, in_rate, out_rate, chunk=chunk)
    if not len(want):
        assert swr_frames(pcm, mask, in_rate, out_rate) == 0
        return want
    got = swr_device(pcm, mask, in_rate, out_rate, big=big)
    assert len(got) == len(want), (len(got), len(want))
    bad = np.nonzero(got != want.astype(np.float32))[0]
    assert not len(bad), (len(bad), bad[:5], got[bad[:5]], want[bad[:5]])
    return want


def frames_for(emu, rates, outputs):
    """The fewest input frames whose plan gives at least `outputs` output frames"""
    lo, hi = 1, 2 * outputs * rates[0] // rates[1] + 1000
    while lo < hi:
        mid = (lo + hi) // 2
        if plan(emu, 0x3, 2, rates[0], rates[1], mid)[0] >= outputs:
            hi = mid
        else:
            lo = mid + 1
    return lo


# the cases of tests/test_swr_cases.py, with its signals
@pytest.mark.parametrize('in_rate', IN_RATES)
@pytest.mark.parametrize('out_rate', OUT_RATES)
def test_rates(gpu_lib, in_rate, out_rate):
    out_rate = out_rate or in_rate
    check(signal('noise', in_rate + 1, 2, in_rate, in_rate ^ out_rate), 0x3, in_rate, out_rate)


@pytest.mark.parametrize('mask', LAYOUTS, ids=hex)
@pytest.mark.parametrize('rates', [(48000, 12000), (44100, 12000), (8000, 12000), (48000, 48000)], ids=str)
def test_layouts(gpu_lib, mask, rates):
    ch = bin(mask).count('1')
    check(signal('noise', rates[0] // 2 + 7, ch, rates[0], mask), mask, *rates)


@pytest.mark.parametrize('frames', LENGTHS)
@pytest.mark.parametrize('rates', [(48000, 12000), (8000, 12000), (7919, 12000), (44100, 44100)], ids=str)
def test_lengths(gpu_lib, frames, rates):
    check(signal('noise', frames, 2, rates[0], frames), 0x3, *rates)


@pytest.mark.parametrize('kind', ['silence', 'full', 'noise', 'tone'])
@pytest.mark.parametrize('mask', [0x4, 0x3, 0x60f], ids=hex)
@pytest.mark.parametrize('rates', [(48000, 12000), (44100, 12000), (22050, 24000), (7919, 12000), (48000, 48000)],
                         ids=str)
def test_values(gpu_lib, kind, mask, rates):
    check(signal(kind, 2 * rates[0] - 1, bin(mask).count('1'), rates[0], 5), mask, *rates)


# the resample kernel's tiles
@pytest.mark.parametrize('rates,outputs', [(r, n) for r in [(48000, 12000), (44100, 12000), (7919, 12000)]
                                           for n in (1, 255, 256, 257, 511, 512, 513)] +
                         [((192000, 4000), n) for n in (127, 128, 129)] +
                         [((384000, 4000), n) for n in (63, 64, 65)], ids=str)
def test_tile_boundaries(gpu_lib, emu, rates, outputs):
    """The fewest input frames that give at least `outputs` outputs, and one frame fewer: the output ends on both sides
    of the count.  Downsampling reaches each count of 255 and above exactly; the first outputs of a stream come
    several at once (17 at 48000 -> 12000), and upsampling can step over a count (7919 -> 12000 goes from 255 to 257
    and from 511 to 513)."""
    frames = frames_for(emu, rates, outputs)
    got = [len(check(signal('noise', n, 2, rates[0], n), 0x3, *rates)) for n in (frames - 1, frames)]
    assert got[0] < outputs <= got[1], got
    if rates[0] > rates[1] and outputs > 1:
        assert got[1] == outputs


@pytest.mark.parametrize('mask', [0x3, 0x63f, 0xff, 0x6cf], ids=hex)
@pytest.mark.parametrize('rates,tile', [((192000, 4000), 128), ((384000, 4000), 64), ((192001, 4001), 128),
                                        ((384001, 4001), 64)], ids=str)
def test_narrow_tiles(gpu_lib, emu, mask, rates, tile):
    assert tiles(emu, *rates)[1][0] == tile
    check(signal('noise', 2 * rates[0] + 5, bin(mask).count('1'), rates[0], mask ^ rates[0]), mask, *rates)


def test_no_output(gpu_lib, emu):
    pcm = signal('noise', 1, 2, 48000, 1)
    assert plan(emu, 0x3, 2, 48000, 12000, 1)[0] == 0
    assert len(ref_swr.convert(pcm, 0x3, 48000, 12000)) == 0
    assert swr_frames(pcm, 0x3, 48000, 12000) == 0


# past one pass of k_swr_mix's grid (sm_count * 16 CTAs of 256 threads: 540 672 frames on 132 SMs)
@pytest.mark.parametrize('mask', [0x4, 0x3, 0x3f, 0x63f], ids=hex)
def test_integer_downmix_past_one_grid_stride(gpu_lib, mask):
    channels = bin(mask).count('1')
    rng = np.random.default_rng(mask)
    pcm = rng.integers(-32768, 32768, (48000 * 60 + 17, channels)).astype(np.int16)
    # uploaded big-endian: the output may reuse the upload's staging buffer, which then never holds the mono answer
    want = check(pcm, mask, 48000, 48000, chunk=1 << 20, big=True)
    assert len(want) == len(pcm)


@pytest.mark.parametrize('rates', [(44100, 12000), (44100, 12001)], ids=str)
def test_ninety_minutes_of_44100(gpu_lib, emu, rates):
    """the 40-phase bank of 44.1 kHz, and linear interpolation where t * dst_incr is large"""
    g = plan(emu, 0x3, 2, rates[0], rates[1], 1000)
    assert (int(g[3]), int(g[4])) == ((40, 0) if rates[1] == 12000 else (1024, 1))
    frames = rates[0] * 5400
    rng = np.random.default_rng(rates[1])
    pcm = (rng.standard_normal((frames, 2), np.float32) * 6000).clip(-32768, 32767).astype(np.int16)
    check(pcm, 0x3, *rates, chunk=1 << 20)


def test_refused_pair(gpu_lib, emu):
    assert tiles(emu, 768000, 2000)[0] == -1
    lib = _native.lib()
    pcm = signal('noise', 768000, 2, 768000, 2)
    h = _native.decode(None, 'sb_pcm_from_le', pcm.ctypes.data_as(ctypes.c_void_p), len(pcm), 2, 2, 768000)
    out = ctypes.c_void_p()
    try:
        with pytest.raises(SushiError, match='sample rates 768000 -> 2000 are not supported'):
            _native.check(lib.sb_pcm_swr(h, 0x3, 2000, ctypes.byref(out)), 'sb_pcm_swr')
        assert not out.value
    finally:
        lib.sb_pcm_destroy(h)
