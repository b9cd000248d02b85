"""The multi-stream instantiations of the packed kernels (sb_find_multi: every query reads its image and template
stream from a per-call stream table) in the CPU emulation of tests/emu: three streams of different lengths, queries
interleaved across them, the image stream equal to the template stream in some.  k_match_packed, k_match_pair (also
as a persistent walk whose CTAs cross query and stream boundaries), k_finish_runs and the multi-stream forward
kernel must give, bit for bit, what the single-stream kernels give on each stream pair alone.
tests/emu/run_tsan_multi.py runs the same checks under ThreadSanitizer."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import tests.test_kernel_emulation as T

ROOT = T.ROOT
EMU = T.EMU
B = T.B


class StreamEntry(ctypes.Structure):          # sb_internal.h
    _fields_ = [('specq', ctypes.c_void_p), ('nblk', ctypes.c_int64), ('raw', ctypes.c_void_p), ('n', ctypes.c_int64),
                ('pfx', ctypes.c_void_p)]


def build_lib(out, extra=(), load=True):
    src = [os.path.join(EMU, f) for f in ('emu_multi_driver.cpp', 'emu_driver.cpp', 'emu_cuda.h', 'emu_ptx.h')] + \
          [os.path.join(ROOT, 'sushi_b200', 'csrc', f) for f in ('sb_fused2.cu', 'sb_fused_common.cuh', 'sb_fft_smem.cuh', 'sb_internal.h')]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in src):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cuda_inc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'include')
        subprocess.check_call(['g++', '-std=c++20', '-O1', '-pthread', '-DSB_EMULATE'] + list(extra) +
                              ['-I', EMU, '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-I', os.path.join(ROOT, 'include'),
                               '-I', cuda_inc, '-shared', '-fPIC', src[0], '-o', out])
    if not load:
        return None
    lib = ctypes.CDLL(out)
    assert lib.emu_query_desc_bytes() == ctypes.sizeof(T.QueryDesc)
    assert lib.emu_stream_entry_bytes() == ctypes.sizeof(StreamEntry)
    return lib


@pytest.fixture(scope='module')
def emu_multi():
    return build_lib(os.path.join(EMU, '_build', 'libsb_emu_multi.so'))


class MultiCase(object):
    """Streams (uint8) and queries (image slot, template slot, toff, n, lag0, nlags)."""

    def __init__(self, lib, streams, queries):
        self.lib, self.queries = lib, queries
        rf = lib.emu_quad_row_floats()
        self.streams = []
        for s in streams:
            img = T.aligned(s.size + 64, np.uint8)
            img[:s.size] = s
            pfx = T.prefix_sums(s)
            a = np.rint(pfx[s.size, 0] / s.size)
            nblk = (s.size + B - 1) // B
            blocks = np.zeros((nblk, 2 * B))
            for k in range(nblk):
                seg = s[k * B:k * B + 2 * B].astype(np.float64)
                blocks[k, :seg.size] = seg - a
            self.streams.append((s, img, pfx, T.quad_rows(blocks, rf), nblk))
        parts = []
        for (i, t, toff, n, lag0, nlags) in queries:
            x = streams[t][toff:toff + n].astype(np.float64)
            b = np.rint(x.sum() / n)
            for p in range((n + B - 1) // B):
                row = np.zeros(2 * B)
                seg = x[p * B:(p + 1) * B]
                row[:seg.size] = seg - b
                parts.append(row)
        self.That = T.quad_rows(np.array(parts), rf)
        self.table = (StreamEntry * len(streams))()
        for k, (s, img, pfx, xhat, nblk) in enumerate(self.streams):
            e = self.table[k]
            e.specq, e.nblk, e.raw, e.n, e.pfx = xhat.ctypes.data, nblk, img.ctypes.data, s.size, pfx.ctypes.data
        self.slots = np.ascontiguousarray(np.array([(q[0], q[1]) for q in queries], np.int32))

    def run(self, kernel, epi, curves):
        group = {0: 1, 1: 2}[kernel]
        desc = (T.QueryDesc * len(self.queries))()
        items = parts = groups = curve = 0
        cta_query = []
        for q, (i, t, toff, n, lag0, nlags) in enumerate(self.queries):
            d = desc[q]
            d.toff, d.tlen, d.lag0, d.nlags = toff, n, lag0, nlags
            d.P, d.k0 = (n + B - 1) // B, lag0 // B
            d.nk = (lag0 + nlags - 1) // B - d.k0 + 1
            d.itemBase, d.partBase, d.curveOff, d.groupBase, d.orig = items, parts, curve, groups, q
            ng = (d.nk + group - 1) // group
            cta_query += [q] * ng
            items += d.nk
            parts += d.P
            groups += ng
            curve += nlags
        cta_query = np.array(cta_query, np.int32)
        keys = np.full(len(self.queries), 0xffffffffffffffff, np.uint64)
        cur = np.full(curve, np.nan, np.float32) if curves else None
        vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        records = epi == 3 and not curves
        recs = counts = None
        if records:
            recs = np.full(len(cta_query) * self.lib.emu_run_slots() * self.lib.emu_run_record_bytes(), 0xCD, np.uint8)
            counts = np.full(len(cta_query), -1, np.int32)
        rc = self.lib.emu_run_multi(kernel, epi, 1, vp(self.That), ctypes.byref(self.table), vp(self.slots), ctypes.byref(desc),
                                    vp(cta_query), len(cta_query), vp(keys), vp(cur) if curves else None,
                                    vp(recs) if records else None, vp(counts) if records else None)
        assert rc == 0, 'emulation reported %d errors (see stderr)' % rc
        if records:
            self.lib.emu_finish_runs_multi(vp(recs), vp(counts), len(cta_query), ctypes.byref(desc), ctypes.byref(self.table),
                                           vp(self.slots), vp(keys))
        return keys, cur

    def run_alone(self, kernel, epi, curves):
        """Every query through the single-stream kernels on its own stream pair."""
        keys = np.empty(len(self.queries), np.uint64)
        cur = []
        for q, (i, t, toff, n, lag0, nlags) in enumerate(self.queries):
            c = T.Case(self.lib, self.streams[i][0], self.streams[t][0], [(toff, n, lag0, nlags)], np.uint8)
            d, idx, cv = c.run(kernel, epi, curves)
            keys[q] = (np.uint64(d.view(np.uint32)[0]) << np.uint64(32)) | np.uint64(idx[0])
            if curves:
                cur.append(cv)
        return keys, (np.concatenate(cur) if curves else None)


def three_streams():
    lengths = [5 * B - 777, 3 * B + 4321, 4 * B]
    streams = [T.programme(n, 60 + k) for k, n in enumerate(lengths)]
    rng = np.random.default_rng(61)
    # stream 1 carries a copy of part of stream 0, so one cross-stream query has a sharp match
    streams[1][2000:2000 + 20000] = np.clip(streams[0][30000:50000].astype(np.int32) + rng.integers(-4, 5, 20000), 0, 255)
    queries = [(0, 1, 2000, 20000, B + 300, 2 * B),          # image 0, template 1: match at lag 30000
               (1, 1, 100, 5000, 0, 2 * B + 100),              # image == template
               (2, 0, 40000, 9000, 500, 3 * B - 9000 - 600),   # runs to near the end of stream 2
               (0, 0, 7000, B + 1, 2 * B - 10, 20),            # image == template, two partitions, straddles a block edge
               (1, 2, 3000, 3000, 3 * B + 4321 - 3000 - 4000, 4001),   # up to the last lag of stream 1
               (2, 2, 20000, 12000, 0, 3 * B)]
    return streams, queries


def check_multi(lib, log=lambda *a: None):
    streams, queries = three_streams()
    c = MultiCase(lib, streams, queries)
    for kernel in (0, 1):
        for epi in (1, 3):
            for curves in (False, True):
                k_m, cur_m = c.run(kernel, epi, curves)
                k_a, cur_a = c.run_alone(kernel, epi, curves)
                assert np.array_equal(k_m, k_a), (kernel, epi, curves)
                if curves:
                    assert np.array_equal(cur_m.view(np.uint32), cur_a.view(np.uint32))
                log('kernel %d epilogue %d curves %d ok' % (kernel, epi, curves))
    want = c.run(1, 3, False)[0]
    assert int(want[0] & np.uint64(0xffffffff)) == 30000 - (B + 300)
    # the persistent pair kernel with fewer CTAs than pairs: every CTA's walk crosses query and stream boundaries
    try:
        for grid in (1, 2, 3):
            lib.emu_set_pair_grid(grid)
            assert np.array_equal(c.run(1, 3, False)[0], want), grid
            log('persistent pair kernel, %d CTAs ok' % grid)
    finally:
        lib.emu_set_pair_grid(0)
    # block spectra of all three streams from one multi-stream forward launch, rows interleaved across the streams
    rf = lib.emu_quad_row_floats()
    outs = [T.aligned(st[4] * rf, np.float32) for st in c.streams]
    table = (StreamEntry * len(streams))()
    for k, st in enumerate(c.streams):
        table[k].specq, table[k].nblk, table[k].raw, table[k].n, table[k].pfx = outs[k].ctypes.data, st[4], st[1].ctypes.data, st[0].size, st[2].ctypes.data
    rows = [(k, r) for r in range(max(st[4] for st in c.streams)) for k in range(len(streams)) if r < c.streams[k][4]]
    row_list = np.ascontiguousarray(np.array(rows, np.int32))
    assert lib.emu_forward_blocks_multi(ctypes.byref(table), row_list.ctypes.data_as(ctypes.c_void_p), len(rows)) == 0
    for k, st in enumerate(c.streams):
        single = T.aligned(st[4] * rf, np.float32)
        assert lib.emu_forward_blocks(1, st[1].ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(st[0].size),
                                      st[2].ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(0), st[4],
                                      single.ctypes.data_as(ctypes.c_void_p)) == 0
        assert np.array_equal(outs[k].view(np.uint32), single.view(np.uint32)), k
    log('multi-stream forward kernel ok')


def test_emulated_multi_stream_kernels_equal_per_stream_runs(emu_multi):
    check_multi(emu_multi)
