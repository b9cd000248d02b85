"""The --ffmpeg-audio conversion (sushi_b200/csrc/sb_swr.cuh) on the CPU, through tests/emu/emu_swr_driver.cpp compiled
with g++, against libswresample itself (tests/ref_swr.py, its FMA3 path): the mono S16 output, its length included, bit
for bit over input and output rates, layouts, lengths and values; the mono matrix row against swr_build_matrix2; the
Kaiser window's Bessel function against av_bessel_i0; the float banks against their impulse read-outs.  The resample
kernel's tiling on the CPU: sbswr::tile_shape's window against the one every output uses over about 440 rate pairs, and
k_swr_resample's tiles and staged windows (emu_swr_convert_tiled) against the untiled loop at a pair of each tile
size.  Also pinned here: libswresample's output does not depend on how the input is chunked, remixing before
resampling would give other samples, and its C, SSE and AVX paths stay within 1 LSB of the FMA3 path."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from sushi_b200 import swr
from tests import ref_swr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_swr_driver.cpp')
SOURCES = [DRIVER, os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_swr.cuh')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_swr.so')

IN_RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 88200, 96000, 192000, 7919, 12001]
OUT_RATES = [12000, 8000, 24000, 44100, None]          # None: the input rate
LAYOUTS = sorted(set(swr.DEFAULT.values()) | set(swr.FLAC.values()) | set(swr.ALAC.values()) | set(swr.TTA.values())
                 | {0x7, 0x33, 0x103, 0x603, 0x637, 0x60f, 0x3f, 0x63f})
LENGTHS = [1, 2, 33, 65, 66, 67, 131, 132, 133, 200, 47999, 48000, 48001]
SMEM_BYTES = 48 * 1024                                  # the shared memory sb_pcm_swr gives k_swr_resample's window
# the sweep's grid beyond IN_RATES x OUT_RATES: exact and inexact (prime, off-by-one) rates
GRID_IN = [1000, 2000, 4000, 7919, 8000, 11025, 12001, 16000, 22050, 24000, 32000, 44100, 44101, 48000, 64000, 88200,
           96000, 96001, 128000, 176400, 192000, 192001, 256000, 352800, 384000, 384001, 512000, 705600, 767999, 768000]
GRID_OUT = [1000, 2000, 4000, 4001, 6000, 8000, 11025, 12000, 12001, 16000, 22050, 24000, 32000, 44100, 48000]
# a pair at each tile size k_swr_resample takes, and an inexact one at each narrow tile
TILED = {(48000, 12000): 256, (44100, 12000): 256, (7919, 12000): 256, (192000, 4000): 128, (192001, 4001): 128,
         (384000, 4000): 64, (384001, 4001): 64}


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64, u64, i32, cp = ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint64, ctypes.c_int, ctypes.c_char_p
    lib.emu_swr_plan.argtypes = [u64, i32, i32, i32, i64, vp, cp, i32]
    lib.emu_swr_convert.argtypes = [vp, i64, i32, u64, i32, i32, i32, vp, cp, i32]
    lib.emu_swr_tiles.argtypes = [i32, i32, i32, i64, vp, cp, i32]
    lib.emu_swr_convert_tiled.argtypes = [vp, i64, i32, u64, i32, i32, i32, vp, cp, i32]
    lib.emu_swr_bank.argtypes = [i32, i32, vp, cp, i32]
    lib.emu_swr_row.argtypes = [u64, vp, cp, i32]
    lib.emu_swr_bessel.argtypes = [ctypes.c_double]
    lib.emu_swr_bessel.restype = ctypes.c_double
    return lib


def plan(emu, mask, channels, in_rate, out_rate, frames):
    g = np.zeros(6, np.int64)
    msg = ctypes.create_string_buffer(256)
    assert emu.emu_swr_plan(mask, channels, in_rate, out_rate, frames, g.ctypes.data, msg, 256) == 0, msg.value
    return g


def convert(emu, pcm, mask, in_rate, out_rate, mix_first=False):
    pcm = np.ascontiguousarray(pcm, np.int16)
    g = plan(emu, mask, pcm.shape[1], in_rate, out_rate, len(pcm))
    out = np.zeros(int(g[0]) + 1, np.int16)
    msg = ctypes.create_string_buffer(256)
    assert emu.emu_swr_convert(pcm.ctypes.data, len(pcm), pcm.shape[1], mask, in_rate, out_rate, int(mix_first),
                               out.ctypes.data, msg, 256) == 0, msg.value
    return out[:int(g[0])]


def tiles(emu, in_rate, out_rate, cap=1 << 26):
    """-> (return code, [tile, width, largest window used, outputs walked, period], message) of emu_swr_tiles"""
    g = np.zeros(5, np.int64)
    msg = ctypes.create_string_buffer(256)
    rc = emu.emu_swr_tiles(in_rate, out_rate, SMEM_BYTES, cap, g.ctypes.data, msg, 256)
    return rc, [int(v) for v in g], msg.value.decode()


def convert_tiled(emu, pcm, mask, in_rate, out_rate):
    pcm = np.ascontiguousarray(pcm, np.int16)
    g = plan(emu, mask, pcm.shape[1], in_rate, out_rate, len(pcm))
    out = np.zeros(int(g[0]) + 1, np.int16)
    msg = ctypes.create_string_buffer(256)
    assert emu.emu_swr_convert_tiled(pcm.ctypes.data, len(pcm), pcm.shape[1], mask, in_rate, out_rate, SMEM_BYTES,
                                     out.ctypes.data, msg, 256) == 0, msg.value
    return out[:int(g[0])]


def signal(kind, frames, channels, rate, seed):
    rng = np.random.default_rng(seed)
    if kind == 'silence':
        return np.zeros((frames, channels), np.int16)
    if kind == 'full':                                   # full-scale square waves: the filter overshoots to the clip
        period = max(2, rate // 441)
        x = np.where((np.arange(frames) // (period // 2 or 1)) % 2 == 0, 32767, -32768)
        return np.repeat(x[:, None], channels, 1).astype(np.int16)
    if kind == 'tone':                                   # near the input's Nyquist frequency
        t = np.arange(frames) / rate
        x = 30000 * np.sin(2 * np.pi * 0.49 * rate * t[:, None] + np.arange(channels))
        return np.round(x).astype(np.int16)
    return rng.integers(-32768, 32768, (frames, channels)).astype(np.int16)


def check(emu, pcm, mask, in_rate, out_rate):
    ref = ref_swr.convert(pcm, mask, in_rate, out_rate)
    got = convert(emu, pcm, mask, in_rate, out_rate)
    assert len(got) == len(ref), (len(got), len(ref))
    bad = np.nonzero(got != ref)[0]
    assert not len(bad), (len(bad), bad[:5], got[bad[:5]], ref[bad[:5]])


@pytest.mark.parametrize('in_rate', IN_RATES)
@pytest.mark.parametrize('out_rate', OUT_RATES)
def test_rates(emu, in_rate, out_rate):
    out_rate = out_rate or in_rate
    check(emu, signal('noise', in_rate + 1, 2, in_rate, in_rate ^ out_rate), 0x3, in_rate, out_rate)


@pytest.mark.parametrize('mask', LAYOUTS, ids=hex)
@pytest.mark.parametrize('rates', [(48000, 12000), (44100, 12000), (8000, 12000), (48000, 48000)], ids=str)
def test_layouts(emu, mask, rates):
    ch = bin(mask).count('1')
    check(emu, signal('noise', rates[0] // 2 + 7, ch, rates[0], mask), mask, *rates)


@pytest.mark.parametrize('frames', LENGTHS)
@pytest.mark.parametrize('rates', [(48000, 12000), (8000, 12000), (7919, 12000), (44100, 44100)], ids=str)
def test_lengths(emu, frames, rates):
    check(emu, signal('noise', frames, 2, rates[0], frames), 0x3, *rates)


@pytest.mark.parametrize('kind', ['silence', 'full', 'noise', 'tone'])
@pytest.mark.parametrize('mask', [0x4, 0x3, 0x60f], ids=hex)
@pytest.mark.parametrize('rates', [(48000, 12000), (44100, 12000), (22050, 24000), (7919, 12000), (48000, 48000)],
                         ids=str)
def test_values(emu, kind, mask, rates):
    check(emu, signal(kind, 2 * rates[0] - 1, bin(mask).count('1'), rates[0], 5), mask, *rates)


def test_tens_of_seconds(emu):
    check(emu, signal('noise', 44100 * 20 + 3, 2, 44100, 7), 0x3, 44100, 12000)
    check(emu, signal('tone', 48000 * 12, 6, 48000, 8), 0x3f, 48000, 12000)


def test_tile_windows_cover_every_output(emu):
    """sbswr::tile_shape's window against the window every output of every tile uses, for every resampling pair of
    IN_RATES x OUT_RATES and of a grid from 1 kHz to 768 kHz in and 1 kHz to 48 kHz out.  sbswr::position is walked
    over lcm(period, tile) outputs, after which both the position pattern and the tile starts repeat, so every tile
    start is seen against every phase of the pattern.  The window fits in shared memory and covers each output's taps
    with the one float to spare the header derives; tiles of 256, 128 and 64 outputs all occur, and no pair
    make_resampler accepts reaches the "too wide a filter window" refusal (the guard stays in the library)."""
    pairs = {(a, b or a) for a in IN_RATES for b in OUT_RATES} | {(a, b) for a in GRID_IN for b in GRID_OUT}
    counts, slack, refused, outputs = {}, [], 0, 0
    for a, b in sorted(p for p in pairs if p[0] != p[1]):
        rc, (tile, width, need, walked, period), msg = tiles(emu, a, b)
        if rc == -1:
            assert 'are not supported' in msg, msg
            refused += 1
            continue
        assert rc == 0, (a, b, msg)
        assert walked % period == 0 and walked % tile == 0, (a, b, walked, period, tile)
        assert need <= width and width * 4 <= SMEM_BYTES, (a, b, tile, width, need)
        counts[tile] = counts.get(tile, 0) + 1
        slack.append(width - need)
        outputs += walked
    print('pairs by tile:', counts, '; refused by make_resampler:', refused, '; outputs walked:', outputs)
    assert counts.get(256) and counts.get(128) and counts.get(64), counts
    assert min(slack) == 1, min(slack)


def test_a_refused_pair_has_no_tile(emu):
    rc, _, msg = tiles(emu, 768000, 2000)
    assert rc == -1 and 'sample rates 768000 -> 2000 are not supported' in msg


@pytest.mark.parametrize('frames', LENGTHS)
@pytest.mark.parametrize('rates', sorted(TILED), ids=str)
def test_tiled_is_untiled(emu, rates, frames):
    """emu_swr_convert_tiled (k_swr_resample's tiles, staged windows and channel order, every window read checked)
    equals emu_swr_convert bit for bit, at a pair of each tile size"""
    assert tiles(emu, *rates)[1][0] == TILED[rates]
    pcm = signal('noise', frames, 3, rates[0], frames)
    want = convert(emu, pcm, 0x7, *rates)
    assert np.array_equal(convert_tiled(emu, pcm, 0x7, *rates), want)


def test_full_scale_reaches_the_clip(emu):
    out = convert(emu, signal('full', 48000, 1, 48000, 0), 0x4, 48000, 12000)
    assert out.max() == 32767 and out.min() == -32768


@pytest.mark.parametrize('mask', LAYOUTS, ids=hex)
def test_matrix_is_swr_build_matrix2(emu, mask):
    row = np.zeros(8, np.float64)
    msg = ctypes.create_string_buffer(256)
    assert emu.emu_swr_row(mask, row.ctypes.data, msg, 256) == 0, msg.value
    f = np.float32(np.sqrt(0.5))
    ref = ref_swr.matrix(mask, center=float(f), surround=float(f))
    assert row[:len(ref)].tolist() == ref.tolist()


def test_unmixable_layouts_are_refused(emu):
    msg = ctypes.create_string_buffer(256)
    row = np.zeros(8, np.float64)
    for mask in (0x1, 0x8, 0x13, 0x800, 0x1ff | 0x200):
        assert emu.emu_swr_row(mask, row.ctypes.data, msg, 256) == -1
        assert b'cannot be mixed to mono' in msg.value


def test_bessel_is_av_bessel_i0(emu):
    from oracle import ref_flac
    util = ref_flac.libs()[2]
    util.av_bessel_i0.argtypes = [ctypes.c_double]
    util.av_bessel_i0.restype = ctypes.c_double
    xs = np.concatenate([np.linspace(0, 9, 9001), np.linspace(9, 40, 3101),
                         np.random.default_rng(3).uniform(0, 9, 3000)])
    assert all(emu.emu_swr_bessel(float(x)) == util.av_bessel_i0(float(x)) for x in xs)


@pytest.mark.parametrize('rates', [(48000, 12000), (44100, 12000), (8000, 12000), (11025, 12000), (32000, 24000),
                                   (192000, 8000)], ids=str)
def test_bank_is_the_impulse_read_out(emu, rates):
    g = plan(emu, 0x4, 1, rates[0], rates[1], 1000)
    taps, alloc, phases = int(g[1]), int(g[2]), int(g[3])
    bank = np.zeros((phases + 1) * alloc, np.float32)
    msg = ctypes.create_string_buffer(256)
    assert emu.emu_swr_bank(rates[0], rates[1], bank.ctypes.data, msg, 256) == 0
    bank = bank.reshape(phases + 1, alloc)
    ref = ref_swr.float_bank(rates[0], rates[1], taps, phases)
    assert not np.isnan(ref).any()
    assert np.array_equal(bank[:phases, :taps], ref)
    assert not bank[:phases, taps:].any()


@pytest.mark.parametrize('rates', [(48000, 12000), (44100, 12000), (8000, 12000), (7919, 12000)], ids=str)
def test_oracle_does_not_depend_on_chunking(rates):
    pcm = signal('noise', 3 * rates[0] + 11, 2, rates[0], 9)
    whole = ref_swr.convert(pcm, 0x3, *rates, chunk=None)
    for chunk in (1152, 4096):
        assert np.array_equal(ref_swr.convert(pcm, 0x3, *rates, chunk=chunk), whole)


def test_remixing_first_gives_other_samples(emu):
    pcm = signal('noise', 8000 * 3, 2, 8000, 10)
    ref = ref_swr.convert(pcm, 0x3, 8000, 12000)
    assert np.array_equal(convert(emu, pcm, 0x3, 8000, 12000), ref)
    assert (convert(emu, pcm, 0x3, 8000, 12000, mix_first=True) != ref).any()


def test_other_cpu_paths_are_within_one_lsb():
    counts = {}
    for rates in [(48000, 12000), (44100, 12000), (8000, 12000)]:
        pcm = signal('noise', 3 * rates[0] + 4, 2, rates[0], 11)
        fma3 = ref_swr.convert(pcm, 0x3, *rates).astype(np.int32)
        for path in ('c', 'sse', 'avx'):
            other = ref_swr.convert(pcm, 0x3, *rates, path=path).astype(np.int32)
            assert len(other) == len(fma3)
            assert np.abs(other - fma3).max() <= 1
            counts[rates, path] = int((other != fma3).sum())
    print('samples differing from the FMA3 path:', counts)
