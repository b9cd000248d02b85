"""The TAK decoder (sushi_b200/csrc/sb_tak.cuh, the stages of sb_tak.cu) on the CPU, through
tests/emu/emu_tak_driver.cpp compiled with g++, fed the config of sushi_b200/tak.py: every case of tests/tak_cases.py
decodes to the writer's PCM (tests/test_tak_cases.py holds FFmpeg to the same PCM) with the file ending at an
inaccessible page, each damaged copy the GPU refuses is refused naming the frame and its file offset, and the
warp-split filter and the chunked block scans equal plain serial loops at every order and length."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from tests import tak_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_tak_driver.cpp')
SOURCES = [DRIVER, os.path.join(EMU, 'emu_guard.h'), os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_tak.cuh'),
           os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_frames.h')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_tak.so')
CASES = tc.all_cases()
BASE, DAMAGED = tc.damaged_cases()
KERNEL = [d for d in DAMAGED if d[4]]


def build():
    """the emulation library, compiled when a source is newer"""
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        tmp = LIB + '.%d' % os.getpid()
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', tmp])
        os.replace(tmp, LIB)
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    for name in ('emu_tak_decode', 'emu_tak_decode_guarded'):
        getattr(lib, name).argtypes = [vp, i64, i64, i64, vp, vp, ctypes.c_char_p, ctypes.c_int]
        getattr(lib, name).restype = ctypes.c_int
    lib.emu_tak_frames.argtypes = [vp, i64, i64, i64, vp, vp, vp, i64, vp, ctypes.c_char_p, ctypes.c_int]
    lib.emu_tak_frames.restype = ctypes.c_int
    lib.emu_tak_filter_check.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint64]
    lib.emu_tak_scan_check.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint64]
    return lib


@pytest.fixture(scope='module')
def emu():
    return build()


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, f, guarded=False, config=None):
    """-> (int16 pcm, None) or (None, message) for TakFile f"""
    config = np.ascontiguousarray(f.config if config is None else config, np.int32)
    pcm = np.zeros((f.samples + 1, f.channels), np.int16)
    msg = ctypes.create_string_buffer(256)
    buf = np.frombuffer(f.data, np.uint8)
    fn = emu.emu_tak_decode_guarded if guarded else emu.emu_tak_decode
    rc = fn(_p(buf), len(f.data), f.audio_start, f.audio_end, _p(config), _p(pcm), msg, 256)
    assert rc != -2
    if rc:
        return None, msg.value.decode()
    return pcm[:f.samples], None


def frame_table(emu, f):
    """[(start, end)] of the frames, or the message"""
    cap = 1 << 16
    start, end, n = np.zeros(cap, np.int64), np.zeros(cap, np.int64), np.zeros(1, np.int64)
    msg = ctypes.create_string_buffer(256)
    buf = np.frombuffer(f.data, np.uint8)
    rc = emu.emu_tak_frames(_p(buf), len(f.data), f.audio_start, f.audio_end, _p(f.config), _p(start), _p(end), cap,
                            _p(n), msg, 256)
    if rc:
        return msg.value.decode()
    return list(zip(start[:n[0]].tolist(), end[:n[0]].tolist()))


def _tak(tmp_path, name, data):
    from sushi_b200 import tak
    path = str(tmp_path / (name + '.tak'))
    with open(path, 'wb') as f:
        f.write(data)
    return tak.TakFile(path)


def test_cases_cover_the_decoder():
    tc.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_stream_decodes_to_the_pcm(emu, tmp_path, case):
    f = _tak(tmp_path, case.name, case.tak())
    assert (f.channels, f.rate, f.bits, f.samples, f.mask) == (case.channels, case.rate, case.bits, len(case.pcm),
                                                                case.mask)
    assert [s for s, _ in frame_table(emu, f)] == case.frame_offsets()
    pcm, err = decode(emu, f, guarded=True)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


@pytest.mark.parametrize('damaged', KERNEL, ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_frame_and_offset(emu, tmp_path, damaged):
    name, data, frame, regex, _ = damaged
    f = _tak(tmp_path, name, data)
    for guarded in (False, True):
        pcm, err = decode(emu, f, guarded)
        assert pcm is None
        if frame is not None:
            where = f.audio_start + sum(len(x) for x in _frames_of(f, frame))
            assert err.startswith('TAK frame %d at byte offset %d: ' % (frame, where)), err
        assert re.search(regex, err), err


def _frames_of(f, frame):
    """the bytes of the frames before `frame`, cut where each next header starts (every damaged copy keeps those)"""
    out, at = [], f.audio_start
    data = f.data
    for _ in range(frame):
        nxt = data.index(b'\xff\xa0', at + 1)
        out.append(data[at:nxt])
        at = nxt
    return out


@pytest.mark.parametrize('order', tc.ORDERS + (0,))
def test_warp_split_filter_equals_the_serial_loop(emu, order):
    for count in (0, 1, 31, 32, 33, 700):
        for quant in (3, 10):
            for dshift in (0, 5, 16):
                assert emu.emu_tak_filter_check(order, count, quant, dshift, order * 7919 + count) == 0, (
                    order, count, quant, dshift)


def test_block_scans_equal_the_serial_sums(emu):
    for mode in (1, 2, 3):
        for n in (1, 2, 3, 4, 15, 16, 255, 256, 257, 511, 1000, 4096, 16383, 16384):
            assert emu.emu_tak_scan_check(mode, n, mode * 100003 + n) == 0, (mode, n)


def test_config_is_refused_in_the_library_s_words(emu, tmp_path):
    f = _tak(tmp_path, BASE.name, BASE.tak())
    for index, value, text in ((0, 7, 'TAK with 7 channels is not supported (1 to 6)'),
                               (1, 8, 'TAK with 8 bits per sample is not supported (16 or 24)'),
                               (3, 3, 'TAK codec type 3 with 2 channels is not supported'),
                               (4, 12, 'sb_tak_decode_file: bad stream parameters')):
        bad = f.config.copy()
        bad[index] = value
        assert decode(emu, f, config=bad) == (None, text)


def test_long_stream_frames_decode(emu, tmp_path):
    case, data, reps = tc.long_stream(bits=16, minutes=1)
    f = _tak(tmp_path, 'long', data)
    pcm, err = decode(emu, f)
    assert err is None and np.array_equal(pcm, tc.long_pcm16(case, reps))
