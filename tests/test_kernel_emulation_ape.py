"""The APE decoder (sushi_b200/csrc/sb_ape.cuh, the four stages of sb_ape.cu) on the CPU, through
tests/emu/emu_ape_driver.cpp compiled with g++, fed the frame tables of sushi_b200/ape.py: every case of
tests/ape_cases.py decodes to the writer's PCM (tests/test_ape_cases.py holds FFmpeg to the same PCM) with the data
ending at an inaccessible page, and each damaged copy the GPU refuses is refused naming the frame and its file
offset."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from sushi_b200 import SushiError
from sushi_b200 import ape
from tests import ape_cases as ac

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_ape_driver.cpp')
SOURCES = [DRIVER, os.path.join(EMU, 'emu_guard.h'), os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_ape.cuh'),
           os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_frames.h')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_ape.so')
CASES = ac.all_cases()
BASE, DAMAGED = ac.damaged_cases()
KERNEL = [d for d in DAMAGED if d[4]]


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        tmp = LIB + '.%d' % os.getpid()
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', tmp])
        os.replace(tmp, LIB)
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    for name in ('emu_ape_decode', 'emu_ape_decode_guarded'):
        getattr(lib, name).argtypes = [vp, i64, vp, vp, i64, vp, vp, ctypes.c_char_p, ctypes.c_int]
        getattr(lib, name).restype = ctypes.c_int
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, f, guarded=False, offsets=None, config=None):
    """-> (int16 pcm, None) or (None, message) for ApeFile f"""
    offsets = np.ascontiguousarray(f.offsets if offsets is None else offsets, np.int64)
    config = np.ascontiguousarray(f.config if config is None else config, np.int32)
    channels, bpf, final = int(config[0]), int(config[4]), int(config[5])
    frames = (len(offsets) - 1) * bpf + final
    pcm = np.zeros((frames + 1, channels), np.int16)
    msg = ctypes.create_string_buffer(256)
    buf = np.frombuffer(f.data[:f.end], np.uint8)
    fn = emu.emu_ape_decode_guarded if guarded else emu.emu_ape_decode
    rc = fn(_p(buf), f.end, _p(offsets), _p(offsets), len(offsets), _p(config), _p(pcm), msg, 256)
    assert rc != -2
    if rc:
        return None, msg.value.decode()
    return pcm[:frames], None


def _ape(tmp_path, name, data):
    path = str(tmp_path / (name + '.ape'))
    with open(path, 'wb') as f:
        f.write(data)
    return ape.ApeFile(path)


def test_cases_cover_the_decoder():
    ac.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_stream_decodes_to_the_pcm(emu, tmp_path, case):
    f = _ape(tmp_path, case.name, case.ape())
    assert (f.channels, f.rate, f.bits, f.level) == (case.channels, case.rate, case.bits, case.level)
    assert list(f.offsets) == case.frame_offsets()
    pcm, err = decode(emu, f, guarded=True)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


@pytest.mark.parametrize('damaged', KERNEL, ids=lambda d: d[0])
def test_damaged_frame_is_refused_naming_frame_and_offset(emu, tmp_path, damaged):
    name, data, frame, regex, _ = damaged
    f = _ape(tmp_path, name, data)
    for guarded in (False, True):
        pcm, err = decode(emu, f, guarded)
        assert pcm is None
        assert err.startswith('APE frame %d at byte offset %d: ' % (frame, f.offsets[frame])), err
        assert re.search(regex, err), err


@pytest.mark.parametrize('damaged', [d for d in DAMAGED if not d[4]], ids=lambda d: d[0])
def test_host_refusals_come_before_the_decoder(tmp_path, damaged):
    name, data, frame, regex, _ = damaged
    with pytest.raises(SushiError, match=regex):
        _ape(tmp_path, name, data)


def test_frame_table_and_config_are_refused_in_the_library_s_words(emu, tmp_path):
    """What sb_ape_decode_frames refuses before the kernels run, through the same functions."""
    f = _ape(tmp_path, BASE.name, BASE.ape())
    outside = f.offsets.copy()
    outside[-1] = f.end
    assert decode(emu, f, offsets=outside) == (
        None, 'APE frame %d at byte offset %d: frame starts outside the buffer' % (len(outside) - 1, f.end))
    for index, value, text in ((0, 3, 'APE with 3 channels is not supported (1 or 2)'),
                               (1, 32, 'APE with 32 bits per sample is not supported (16 or 24)'),
                               (3, 6000, 'APE compression level 6000 is not supported'),
                               (5, int(f.config[4]) + 1, 'sb_ape_decode_frames: bad stream parameters')):
        bad = f.config.copy()
        bad[index] = value
        assert decode(emu, f, config=bad) == (None, text)


def test_cut_frames_read_nothing_past_their_bytes(emu, tmp_path):
    """The first frame cut at every length, last in a buffer that ends at an inaccessible page: refused, never read
    past."""
    f = _ape(tmp_path, BASE.name, BASE.ape())
    for cut in list(range(1, 40)) + list(range(40, int(f.offsets[1] - f.offsets[0]), 97)):
        f.end = int(f.offsets[1]) - cut
        pcm, err = decode(emu, f, guarded=True, offsets=f.offsets[:1])
        assert pcm is None and re.search('past the frame|CRC mismatch|invalid frame header|symbol', err), err


def test_long_stream_frames_decode(emu, tmp_path):
    case, data, reps = ac.long_stream(bits=16, minutes=1, level=2000)
    f = _ape(tmp_path, 'long', data)
    pcm, err = decode(emu, f)
    assert err is None and np.array_equal(pcm, ac.long_pcm16(case, reps))
