"""MP2 (MPEG audio layer II) on the CPU: FFmpeg's fixed-point `mp2` decoder, driven through ctypes (tests/ref_mp2.py,
tests/ref_mp4.py, tests/ref_ts.py), against the writer of tests/mp2_cases.py and the CPU build of
sushi_b200/csrc/sb_mp2.cuh (tests/emu/emu_mp2_driver.cpp, compiled with g++).  Every case decodes through FFmpeg and
through the header bit for bit; the transport streams and Matroska files FFmpeg demuxes decode as their elementary
streams do, including a capture that starts mid-frame and one cut at the end; each damaged copy is refused naming the
frame and its offset; the DCT constants are recomputed from their formula."""
import ctypes
import math
import os
import re
import subprocess

import numpy as np
import pytest

from sushi_b200 import matroska as mk
from sushi_b200 import mpegts
from tests import mp2_cases as mc
from tests import ref_mp2
from tests import ref_mp4
from tests import ref_ts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_mp2_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_mp2.cuh')
SOURCES = [DRIVER, HEADER, os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_frames.h')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_mp2.so')
CASES = mc.all_cases()


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-Wno-unknown-pragmas', '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared',
                               '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.emu_mp2_decode.argtypes = [vp, i64, vp, vp, i64, vp, i64, vp, vp, ctypes.c_char_p, ctypes.c_int]
    lib.emu_mp2_decode.restype = ctypes.c_int
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, data, offsets=(0,), where=(0,)):
    """-> ((frames, channels) int16, cut) or (None, message)"""
    buf = np.frombuffer(data + bytes(16), np.uint8)
    offsets = np.ascontiguousarray(offsets, np.int64)
    where = np.ascontiguousarray(where, np.int64)
    cap = (len(data) // 20 + 4) * 1152
    pcm = np.zeros(cap * 2, np.int16)
    n = ctypes.c_int64()
    info = np.zeros(3, np.int32)
    msg = ctypes.create_string_buffer(256)
    rc = emu.emu_mp2_decode(_p(buf), len(data), _p(offsets), _p(where), len(offsets), _p(pcm), cap, ctypes.byref(n),
                            _p(info), msg, 256)
    if rc:
        return None, msg.value.decode()
    ch = int(info[0])
    return pcm[:n.value * 1152 * ch].reshape(-1, ch), int(info[2])


def test_cases_cover_the_decoder():
    mc.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_header_equals_ffmpeg_on_every_case(emu, case):
    want, mask, rate, refused = ref_mp2.decode_packets(case.frames)
    assert refused == 0 and rate == case.rate and len(want) == 1152 * len(case.frames)
    assert mask == {1: 0x4, 2: 0x3}[case.channels]
    got, cut = decode(emu, case.data)
    assert got is not None, cut
    assert np.array_equal(got, want)


def test_cases_clip_and_fall_silent():
    by = {c.name: c for c in CASES}
    loud = ref_mp2.decode_packets(by['mp2_loud_clips'].frames)[0]
    assert (loud == 32767).sum() > 100 and (loud == -32768).sum() > 100
    quiet = ref_mp2.decode_packets(by['mp2_silence'].frames)[0]
    assert not quiet[:2 * 1152].any()


@pytest.mark.parametrize('pair', mc.ts_files(CASES), ids=lambda p: p[0].name)
def test_transport_stream_decodes_as_its_elementary_stream(emu, tmp_path, pair):
    """FFmpeg lists stream types 0x03 / 0x04 as `mp3` until its parser reads a header, then `mp2`; its parser drops a
    first frame glued to the bytes before it, and its decoder decodes a last frame the file cuts with zeros"""
    ts, case = pair
    path = ts.write(tmp_path)
    assert [s.codec for s in mpegts.TransportStream(path).streams_all] == ['mp3']
    assert [s['codec'] for s in ref_ts.streams(path)] == ['mp3']
    assert [s['codec'] for s in ref_ts.streams(path, find_info=True)] == ['mp2']
    want, mask, rate = ref_mp4.decode_s16(path, 0)
    assert mask == {1: 0x4, 2: 0x3}[case.channels] and rate == case.rate
    got, cut = decode(emu, ts.es)
    assert got is not None, cut
    assert cut == (ts.name == 'ts_cut_end')
    if ts.name == 'ts_mid_frame_start':                   # the first whole frame after the cut is not decoded
        starts = np.cumsum([0] + [len(f) for f in case.frames])
        first = int(np.searchsorted(starts, 300))
        assert len(got) == 1152 * (len(case.frames) - first - 1)
    assert np.array_equal(got, want)


@pytest.mark.parametrize('pair', mc.mkv_files(CASES), ids=lambda p: p[0].name)
def test_matroska_track_decodes_as_ffmpeg_decodes_it(emu, tmp_path, pair):
    m, case = pair
    path = m.write(tmp_path)
    with mk.MatroskaFile(path) as f:
        t = f.select('audio', None)
        assert mk.audio_codec(t) == 'mp2'
        audio = f.select_audio()
        assert (audio.label, audio.fmt, audio.bits, audio.layout) == ('MP2', 'S16', 16, {1: 0x4, 2: 0x3})
        table = f.frames([t.id])[t.id]
    want, mask, rate = ref_mp4.decode_s16(path, 0)
    assert rate == case.rate
    got, cut = decode(emu, table.data, table.offset, table.block)
    assert got is not None and np.array_equal(got, want)


@pytest.mark.parametrize('damaged', mc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_frame_and_offset(emu, damaged):
    name, data, frame, offset, regex = damaged
    got, msg = decode(emu, data)
    assert got is None
    assert msg.startswith('MP2 frame %d at byte offset %d: ' % (frame, offset)), msg
    assert re.search(regex, msg), msg


def test_dct_constants_are_their_formula():
    """round(2^32 / (2 cos((2i + 1) pi / 2^(6 - j))) / 2^s), s the shift of the butterfly that uses each"""
    text = open(HEADER).read()
    shifts = {0: [1] * 11 + [2, 2, 3, 3, 5], 1: [1] * 5 + [2, 2, 4], 2: [1, 1, 1, 3], 3: [1, 2]}
    for j, s in shifts.items():
        want = [int(1 / (2 * math.cos((2 * i + 1) * math.pi / 2 ** (6 - j))) / 2 ** s[i] * 2 ** 32 + 0.5)
                for i in range(len(s))]
        body = re.search(r'kCos%d, \[\d+\], \{([^}]*)\}' % j, text).group(1)
        assert [int(x) for x in body.replace('\n', ' ').split(',') if x.strip()] == want
    assert 'kCos4 = %d;' % int(math.sqrt(0.5) / 2 * 2 ** 32 + 0.5) in text


def test_allocation_tables_match_the_writer():
    """the header's five tables, expanded, against the writer's (both from the standard's tables B.2a-d and B.1)"""
    text = open(HEADER).read()
    macros = {m.group(1): [int(x) for x in m.group(2).split(',')]
              for m in re.finditer(r'#define SBM_(\w\d) ([\d, ]+)\n', text)}

    def expand(name):
        body = re.search(r'SBM_TABLE\(uint8_t, %s, \[\], \{(.*?)\}\)' % name, text, re.S).group(1)
        return [macros[m] for m in re.findall(r'SBM_(\w\d)', body)]
    ab, cd, lsf = expand('kAllocAB'), expand('kAllocCD'), expand('kAllocLsf')
    for table, rows in ((0, ab[:27]), (1, ab[:30]), (2, cd[:8]), (3, cd[:12]), (4, lsf)):
        assert [r[1:] for r in rows] == [c for c in mc.TABLES[table]]
        assert all(len(r) == 1 << r[0] for r in rows)
