"""Many streams in one call (sb_find_multi / sb_match_curves_multi) and the lockstep solver on top of them, on an H100:
bit-for-bit equality with per-pair single-stream calls, launch counts independent of the number of streams, the error
cases, and shift_scripts / shift_events_many against their one-job-at-a-time forms."""
import ctypes
import wave

import numpy as np
import pytest

from sushi_b200 import WavStream, synth, _native
from sushi_b200.common import format_time

pytestmark = pytest.mark.gpu
B = 16384
RATE = 12000


def stream(n, seed, dtype):
    x = synth.programme_audio(n, seed).astype(np.float32)
    x = (x - x.min()) / (x.max() - x.min())
    data = (x * 255 + 0.5).astype(np.uint8) if dtype == np.uint8 else x.astype(np.float32)
    return WavStream.from_array(data.reshape(1, -1), RATE, 0, n)


def multi_call(lib, streams, q, curves=False):
    """q: rows (image slot, template slot, toff, tlen, lag0, nlags)."""
    table = (ctypes.c_void_p * len(streams))(*[s._handle.value for s in streams])
    islot = np.ascontiguousarray(q[:, 0], np.int32)
    tslot = np.ascontiguousarray(q[:, 1], np.int32)
    arrs = [np.ascontiguousarray(q[:, k], np.int64) for k in range(2, 6)]
    ptrs = [islot.ctypes.data_as(_native.c_i32p), tslot.ctypes.data_as(_native.c_i32p)] + \
           [a.ctypes.data_as(_native.c_i64p) for a in arrs]
    if curves:
        out = np.empty(int(arrs[3].sum()), np.float32)
        rc = lib.sb_match_curves_multi(table, len(streams), len(q), *ptrs, out.ctypes.data_as(_native.c_f32p))
        return rc, out
    diff = np.empty(len(q), np.float32)
    idx = np.empty(len(q), np.int64)
    rc = lib.sb_find_multi(table, len(streams), len(q), *ptrs, diff.ctypes.data_as(_native.c_f32p),
                           idx.ctypes.data_as(_native.c_i64p))
    return rc, (diff, idx)


def per_pair(streams, q, curves=False):
    """The same queries as one sb_find_batch / sb_match_curves per distinct (image, template) pair."""
    diff = np.empty(len(q), np.float32)
    idx = np.empty(len(q), np.int64)
    cur = [None] * len(q)
    for pair in sorted(set(map(tuple, q[:, :2].tolist()))):
        sel = np.nonzero((q[:, 0] == pair[0]) & (q[:, 1] == pair[1]))[0]
        img, tmpl = streams[pair[0]], streams[pair[1]]
        if curves:
            for i, c in zip(sel, img.match_curves(tmpl, *[q[sel, k] for k in range(2, 6)])):
                cur[i] = c
        else:
            d, k = img.find_planned(tmpl, *[q[sel, k] for k in range(2, 6)])
            diff[sel], idx[sel] = d, k
    return np.concatenate(cur) if curves else (diff, idx)


def queries(streams, rng, count):
    """Interleaved over the streams, image == template in some; short (P = 1), 4-6 partition and >= 12 partition
    templates, +-10 s searches."""
    rows = []
    for k in range(count):
        i = int(rng.integers(len(streams)))
        t = i if k % 3 == 0 else int(rng.integers(len(streams)))
        n = [5000, 4 * B + 3000, 12 * B + 700][k % 3]
        toff = int(rng.integers(0, streams[t].total_samples - n))
        nlags = 2 * 10 * RATE + 1
        lag0 = int(rng.integers(0, streams[i].total_samples - n - nlags))
        rows.append((i, t, toff, n, lag0, nlags))
    return np.array(rows, np.int64)


@pytest.mark.parametrize('dtype,epi', [(np.uint8, 3), (np.uint8, 1), (np.float32, 1)])
@pytest.mark.parametrize('engine', [2, 4, 5])
def test_multi_equals_per_pair_bit_for_bit(gpu_lib, dtype, epi, engine):
    lib = gpu_lib
    lengths = [180 * RATE, 150 * RATE + 777, 121 * RATE + 5]              # streams of different lengths
    streams = [stream(n, 40 + k, dtype) for k, n in enumerate(lengths)]
    q = queries(streams, np.random.default_rng(engine * 10 + epi), 18)
    old_engine, old_epi = lib.sb_get_engine(), lib.sb_get_epilogue()
    try:
        assert lib.sb_set_engine(engine) == 0 and lib.sb_set_epilogue(epi) == 0
        rc, (d, i) = multi_call(lib, streams, q)
        assert rc == 0, lib.sb_last_error()
        want_d, want_i = per_pair(streams, q)
        assert np.array_equal(d.view(np.uint32), want_d.view(np.uint32)) and np.array_equal(i, want_i)
        # curves: all three template classes (the >= 12 partition ones run per pair inside the call), then the packed
        # direct class alone (written straight into the caller's array)
        for sub in (q[:6], q[q[:, 3] < 12 * B][:6]):
            rc, cur = multi_call(lib, streams, sub, curves=True)
            assert rc == 0, lib.sb_last_error()
            assert np.array_equal(cur.view(np.uint32), per_pair(streams, sub, curves=True).view(np.uint32))
        assert (q[:6, 3] >= 12 * B).any() and (q[:6, 3] < B).any()
    finally:
        lib.sb_set_engine(old_engine)
        lib.sb_set_epilogue(old_epi)


def test_launch_count_does_not_grow_with_the_stream_count(gpu_lib):
    lib = gpu_lib
    counts = {}
    for n_streams in (1, 4, 16):
        streams = [stream(90 * RATE, 70 + k, np.uint8) for k in range(n_streams)]
        rows = []
        for k in range(16):                                    # the same 16 queries, spread over the streams
            s = k % n_streams
            rows.append((s, s, 30 * RATE + 997 * k, 2 * B + 100, 20 * RATE + 1000 * k, 20 * RATE + 1))
        q = np.array(rows, np.int64)
        got = []
        for _ in range(2):                                     # first call builds block spectra, second finds them
            before = lib.sb_launch_count()
            rc, _ = multi_call(lib, streams, q)
            assert rc == 0, lib.sb_last_error()
            got.append(lib.sb_launch_count() - before)
        counts[n_streams] = got
    assert counts[1] == counts[4] == counts[16], counts


def test_error_cases_name_the_query_or_slot(gpu_lib):
    lib = gpu_lib
    a, b = stream(40 * RATE, 3, np.uint8), stream(40 * RATE, 4, np.uint8)
    f = stream(40 * RATE, 5, np.float32)
    q = np.array([(0, 1, 1000, 5000, 2000, 10000), (1, 0, 1000, 5000, 2000, 10000)], np.int64)

    def err(streams, rows):
        rc, _ = multi_call(lib, streams, rows)
        return rc, lib.sb_last_error().decode()

    bad = q.copy(); bad[1, 1] = 2
    rc, msg = err([a, b], bad)
    assert rc == -1 and 'query 1' in msg and 'slot 2' in msg          # SB_EINVAL
    rc, msg = err([a, b], q + np.array([[0, 0, 0, 0, 0, 0], [-5, 0, 0, 0, 0, 0]]))
    assert rc == -1 and 'query 1' in msg and 'image slot -4' in msg
    rc, msg = err([a, f], q)
    assert rc == -1 and 'slot 1' in msg and 'sample type' in msg
    table = (ctypes.c_void_p * 2)(a._handle.value, None)
    islot = np.zeros(2, np.int32); tslot = np.zeros(2, np.int32)
    arrs = [np.ascontiguousarray(q[:, k], np.int64) for k in range(2, 6)]
    d = np.empty(2, np.float32); i = np.empty(2, np.int64)
    rc = lib.sb_find_multi(table, 2, 2, islot.ctypes.data_as(_native.c_i32p), tslot.ctypes.data_as(_native.c_i32p),
                           *[x.ctypes.data_as(_native.c_i64p) for x in arrs], d.ctypes.data_as(_native.c_f32p),
                           i.ctypes.data_as(_native.c_i64p))
    assert rc == -1 and 'slot 1 is NULL' in lib.sb_last_error().decode()
    # a raw sb_load_pcm stream has no running sums
    pcm = np.zeros(12000, np.int16)
    raw = ctypes.c_void_p()
    assert lib.sb_load_pcm(pcm.ctypes.data_as(ctypes.c_void_p), 12000, 1, 2, 12000, 12000, 100, 12200, ctypes.byref(raw)) == 0
    try:
        table = (ctypes.c_void_p * 2)(a._handle.value, raw.value)
        rc = lib.sb_find_multi(table, 2, 2, islot.ctypes.data_as(_native.c_i32p), tslot.ctypes.data_as(_native.c_i32p),
                               *[x.ctypes.data_as(_native.c_i64p) for x in arrs], d.ctypes.data_as(_native.c_f32p),
                               i.ctypes.data_as(_native.c_i64p))
        assert rc == -1 and 'slot 1 has no running sums' in lib.sb_last_error().decode()
    finally:
        lib.sb_stream_destroy(raw)
    # the per-query rules of sb_find_batch, checked against the query's own streams
    bad = q.copy(); bad[1, 4] = 40 * RATE
    rc, msg = err([a, b], bad)
    assert rc == -1 and 'query 1' in msg and 'outside image stream' in msg


def write_job(tmp_path, k, dur, shift):
    from sushi_b200 import AssScript
    src12, dst12 = synth.make_pair(dur, 60 + k, shift)
    paths = []
    for name, pcm in (('src%d.wav' % k, src12), ('dst%d.wav' % k, dst12)):
        with wave.open(str(tmp_path / name), 'wb') as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(12000); w.writeframes(pcm.tobytes())
        paths.append(str(tmp_path / name))
    starts, ends = synth.make_events(30, dur - 8.0, 60 + k, 0.8, 3.0, 1.5)
    lines = ['[Script Info]', 'Title: t', '', '[V4+ Styles]', AssScript.STYLES_FORMAT,
             'Style: Default,Arial,20,&H00FFFFFF,&H000000FF,&H00000000,&H00000000,0,0,0,0,100,100,0,0,1,2,2,2,10,10,10,1',
             '', '[Events]', AssScript.EVENTS_FORMAT]
    for i, (a, b) in enumerate(zip(starts, ends)):
        lines.append('Dialogue: 0,{0},{1},Default,,0,0,0,,line {2}'.format(format_time(a), format_time(b), i))
    (tmp_path / ('in%d.ass' % k)).write_text('\n'.join(lines), encoding='utf-8')
    return paths + [str(tmp_path / ('in%d.ass' % k))]


def test_shift_scripts_writes_what_shift_script_writes(gpu_lib, tmp_path):
    from sushi_b200 import shift_script, shift_scripts
    shifts = [1.5, [(0.0, 0.5), (30.0, -2.0)], [(0.0, 0.3), (25.0, 13.0)], 2.25]   # const, jump, rewind (> 10 s), const
    jobs = [write_job(tmp_path, k, 60.0, s) for k, s in enumerate(shifts)]
    for k, (src, dst, ass) in enumerate(jobs):
        shift_script(src, dst, ass, str(tmp_path / ('one%d.ass' % k)))
    shift_scripts([(src, dst, ass, str(tmp_path / ('many%d.ass' % k))) for k, (src, dst, ass) in enumerate(jobs)])
    for k in range(len(jobs)):
        assert (tmp_path / ('one%d.ass' % k)).read_bytes() == (tmp_path / ('many%d.ass' % k)).read_bytes()


def test_shift_events_many_equals_shift_events(gpu_lib):
    from sushi_b200 import shift_events, shift_events_many
    from sushi_b200.events import ScriptEvent
    jobs = []
    for k, sh in enumerate([1.5, [(0.0, 0.75), (40.0, -2.5)], [(0.0, 0.3), (35.0, 14.0)]]):
        src_pcm, dst_pcm = synth.make_pair(80.0, 90 + k, sh)
        starts, ends = synth.make_events(40, 72.0, 90 + k, 0.8, 3.0, 1.5)
        jobs.append((WavStream.from_pcm(src_pcm, RATE), WavStream.from_pcm(dst_pcm, RATE), starts, ends))
    jobs.append((jobs[0][0], jobs[1][1], jobs[0][2], jobs[0][3]))            # a destination shared with job 1

    def events(job):
        return [ScriptEvent(i, float(a), float(b)) for i, (a, b) in enumerate(zip(job[2], job[3]))]

    alone = []
    for job in jobs:
        ev = events(job)
        shift_events(ev, job[0], job[1])
        alone.append([(e.shift, e.diff, e._link.source_index if e.linked else -1) for e in ev])
    evs = [events(job) for job in jobs]
    shift_events_many([(ev, job[0], job[1]) for ev, job in zip(evs, jobs)])
    for ev, want in zip(evs, alone):
        assert [(e.shift, e.diff, e._link.source_index if e.linked else -1) for e in ev] == want
