"""The persistent walk of k_forward_quad on the CPU (tests/emu/emu_forward_driver.cpp, see
tests/test_kernel_emulation.py): a launch with 1, 2 or 3 CTAs, each walking the rows b, b + grid, ..., writes exactly
the rows a launch of one CTA per row writes -- across the end of the stream (MODE 0), across template boundaries of
queries with 1 to 3 partitions (MODE 1, where each row finds its query by the CTA-wide search), and across streams
(MULTI).  The MODE 1 rows are also checked against NumPy."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests.test_kernel_emulation import B, EMU, ROOT, QueryDesc, aligned, prefix_sums, quad_rows
from tests.test_kernel_emulation_multi import StreamEntry

GRIDS = (1, 2, 3)
WRITTEN = (2 * (B // 4) + 2) * 4                   # floats of a row the kernel writes (the rest is padding)
VP, I64 = ctypes.c_void_p, ctypes.c_int64


DRIVER = os.path.join(EMU, 'emu_forward_driver.cpp')


def build(out, extra=()):
    """Compiles tests/emu/emu_forward_driver.cpp into `out` unless it is newer than every source it includes."""
    deps = [DRIVER] + [os.path.join(EMU, f) for f in ('emu_multi_driver.cpp', 'emu_driver.cpp', 'emu_cuda.h', 'emu_ptx.h')] + \
           [os.path.join(ROOT, 'sushi_b200', 'csrc', f) for f in ('sb_fused2.cu', 'sb_fused_common.cuh', 'sb_fft_smem.cuh', 'sb_internal.h')]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cuda_inc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'include')
        subprocess.check_call(['g++', '-std=c++20', '-O1', '-pthread', '-DSB_EMULATE'] + list(extra) +
                              ['-I', EMU, '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-I', os.path.join(ROOT, 'include'),
                               '-I', cuda_inc, '-shared', '-fPIC', DRIVER, '-o', out])


def load(out):
    lib = ctypes.CDLL(out)
    assert lib.emu_query_desc_bytes() == ctypes.sizeof(QueryDesc)
    assert lib.emu_stream_entry_bytes() == ctypes.sizeof(StreamEntry)
    lib.emu_walk_blocks.argtypes = [ctypes.c_int, ctypes.c_int, VP, I64, VP, I64, ctypes.c_int, VP]
    lib.emu_walk_parts.argtypes = [ctypes.c_int, ctypes.c_int, VP, I64, VP, VP, ctypes.c_int, ctypes.c_int, I64, ctypes.c_int, VP]
    lib.emu_walk_blocks_multi.argtypes = [ctypes.c_int, VP, VP, ctypes.c_int]
    lib.emu_walk_parts_multi.argtypes = [ctypes.c_int, VP, VP, VP, ctypes.c_int, ctypes.c_int, I64, ctypes.c_int, VP]
    return lib


@pytest.fixture(scope='module')
def walk():
    out = os.path.join(EMU, '_build', 'libsb_emu_forward.so')
    build(out)
    return load(out)


def _ptr(a):
    return a.ctypes.data_as(VP)


def _by_grid(lib, rows, call):
    """call(grid, out) for one CTA per row (grid 0) and for GRIDS; returns {grid: rows x row floats}"""
    rf = lib.emu_quad_row_floats()
    outs = {}
    for grid in (0,) + GRIDS:
        out = aligned(rows * rf, np.float32, np.nan)
        assert call(grid, out) == 0, grid
        outs[grid] = out.reshape(rows, rf)
    assert np.isfinite(outs[0][:, :WRITTEN]).all()
    for grid in GRIDS:
        assert outs[grid].tobytes() == outs[0].tobytes(), grid
    return outs[0]


def _template_rows(x, descs, q_begin, q_end, rf):
    parts = []                                     # each row against its own template, centred like the kernel
    for q in range(q_begin, q_end):
        t = x[q][descs[q].toff:descs[q].toff + descs[q].tlen].astype(np.float64)
        for p in range(descs[q].P):
            row = np.zeros(2 * B)
            seg = t[p * B:(p + 1) * B]
            row[:seg.size] = seg - np.rint(t.sum() / t.size)
            parts.append(row)
    return quad_rows(np.array(parts), rf)[:, :WRITTEN]


def _queries(lens, toffs=None):
    """descriptors of templates of the given lengths, back to back with gaps of 123 samples unless toffs says where"""
    descs = (QueryDesc * len(lens))()
    toff = part = 0
    for q, tlen in enumerate(lens):
        descs[q].toff, descs[q].tlen, descs[q].partBase = toff if toffs is None else toffs[q], tlen, part
        descs[q].P = (tlen + B - 1) // B
        toff += tlen + 123
        part += descs[q].P
    return descs


@pytest.mark.parametrize('dtype', [np.uint8, np.float32])
def test_block_rows_do_not_depend_on_the_grid(walk, dtype):
    rng = np.random.default_rng(11)
    n = 3 * B + 5000                                    # rows 3 and 4 read past the end of the stream
    x = rng.integers(0, 256, n).astype(dtype) if dtype == np.uint8 else rng.standard_normal(n).astype(np.float32)
    src = aligned(n + 64, dtype)
    src[:n] = x
    pfx = prefix_sums(x)
    rows = 5
    _by_grid(walk, rows, lambda g, out: walk.emu_walk_blocks(g, int(dtype == np.uint8), _ptr(src), n, _ptr(pfx), 0, rows, _ptr(out)))


def test_partition_rows_do_not_depend_on_the_grid(walk):
    rng = np.random.default_rng(12)
    n = 12 * B
    x = rng.integers(0, 256, n).astype(np.uint8)
    src = aligned(n + 64, np.uint8)
    src[:n] = x
    pfx = prefix_sums(x)
    lens = [B // 3, 2 * B + 77, B, 3 * B - 5, 1000, B + 1]          # 1, 3, 1, 3, 1, 2 partitions
    descs = _queries(lens)
    rf = walk.emu_quad_row_floats()
    # the whole batch, and a launch of the rows of queries 1 .. 4 only (part_first inside the batch)
    for q_begin, q_end in ((0, len(lens)), (1, 5)):
        first = descs[q_begin].partBase
        rows = sum(descs[q].P for q in range(q_begin, q_end))
        got = _by_grid(walk, rows, lambda g, out: walk.emu_walk_parts(g, 1, _ptr(src), n, _ptr(pfx), ctypes.cast(descs, VP),
                                                                     q_begin, q_end, first, rows, _ptr(out)))
        want = _template_rows([x] * len(lens), descs, q_begin, q_end, rf)
        assert np.abs(got[:, :WRITTEN] - want).max() <= 1e-5 * np.abs(want).max()


def test_multi_stream_rows_do_not_depend_on_the_grid(walk):
    rng = np.random.default_rng(13)
    sizes = [2 * B + 300, 4 * B - 7, B + 9]
    xs = [rng.integers(0, 256, s).astype(np.uint8) for s in sizes]
    srcs, pfxs = [], []
    for x in xs:
        a = aligned(x.size + 64, np.uint8)
        a[:x.size] = x
        srcs.append(a)
        pfxs.append(prefix_sums(x))
    nblk = [(s + B - 1) // B for s in sizes]
    rf = walk.emu_quad_row_floats()
    specq = [aligned(k * rf, np.float32, np.nan) for k in nblk]
    table = (StreamEntry * len(sizes))()
    for k in range(len(sizes)):
        table[k].specq, table[k].nblk, table[k].raw, table[k].n, table[k].pfx = specq[k].ctypes.data, nblk[k], srcs[k].ctypes.data, sizes[k], pfxs[k].ctypes.data
    # block spectra: rows interleaved across the streams, written into each stream's own rows
    rows = [(k, r) for r in range(max(nblk)) for k in range(len(sizes)) if r < nblk[k]]
    row_list = np.ascontiguousarray(np.array(rows, np.int32))
    ref = None
    for grid in (0,) + GRIDS:
        for a in specq:
            a[:] = np.nan
        assert walk.emu_walk_blocks_multi(grid, ctypes.cast(table, VP), _ptr(row_list), len(rows)) == 0
        got = b''.join(a.tobytes() for a in specq)
        ref = ref or got
        assert got == ref, grid
    # template partitions of queries whose templates live in streams 2, 1, 0, 0
    tslot = [2, 1, 0, 0]
    lens = [B // 2, 3 * B - 100, 700, B + 5]
    descs = _queries(lens, toffs=[0, 11, 5000, B // 2 + 50])
    slots = np.ascontiguousarray(np.array([(0, s) for s in tslot], np.int32))
    n_rows = sum(descs[q].P for q in range(len(lens)))
    got = _by_grid(walk, n_rows, lambda g, out: walk.emu_walk_parts_multi(g, ctypes.cast(table, VP), _ptr(slots), ctypes.cast(descs, VP),
                                                                        0, len(lens), 0, n_rows, _ptr(out)))
    want = _template_rows([xs[s] for s in tslot], descs, 0, len(lens), rf)
    assert np.abs(got[:, :WRITTEN] - want).max() <= 1e-5 * np.abs(want).max()
