"""The TTA decoder (sushi_b200/csrc/sb_tta.cuh, k_tta_decode's frames) on the CPU, through
tests/emu/emu_tta_driver.cpp compiled with g++, fed the frame tables of sushi_b200/tta.py: every case of
tests/tta_cases.py decodes to the writer's PCM (tests/test_tta_cases.py holds FFmpeg to the same PCM), every A_TTA1
Matroska track decodes from its frames, and each copy the GPU refuses is refused naming the frame and its file offset,
again with the data ending at an inaccessible page."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from sushi_b200 import SushiError
from sushi_b200 import matroska as mk
from sushi_b200 import tta
from tests import mkv_tta_cases as mtc
from tests import tta_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_tta_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_tta.cuh')
LIB = os.path.join(EMU, '_build', 'libsb_emu_tta.so')
CASES = tc.all_cases()
BASE, DAMAGED = tc.damaged_cases()
KERNEL = [d for d in DAMAGED if d[4]]


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    for name in ('emu_tta_decode', 'emu_tta_decode_guarded'):
        getattr(lib, name).argtypes = [vp, i64, vp, vp, i64, vp, vp, ctypes.c_char_p, ctypes.c_int]
        getattr(lib, name).restype = ctypes.c_int
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, data, offsets, where, config, guarded=False):
    """-> (int16 pcm, None) or (None, message)"""
    offsets = np.ascontiguousarray(offsets, np.int64)
    where = np.ascontiguousarray(where, np.int64)
    config = np.ascontiguousarray(config, np.int32)
    channels, fl, last = int(config[0]), int(config[3]), int(config[4])
    frames = (len(offsets) - 1) * fl + (last or fl)
    pcm = np.zeros((frames + 1, channels), np.int16)
    msg = ctypes.create_string_buffer(256)
    buf = np.frombuffer(data, np.uint8)
    fn = emu.emu_tta_decode_guarded if guarded else emu.emu_tta_decode
    rc = fn(_p(buf), len(data), _p(offsets), _p(where), len(offsets), _p(config), _p(pcm), msg, 256)
    assert rc != -2
    if rc:
        return None, msg.value.decode()
    return pcm[:frames], None


def _tta(tmp_path, name, data):
    path = str(tmp_path / (name + '.tta'))
    with open(path, 'wb') as f:
        f.write(data)
    return tta.TTAFile(path)


def test_cases_cover_the_decoder():
    tc.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_stream_decodes_to_the_pcm(emu, tmp_path, case):
    f = _tta(tmp_path, case.name, case.tta())
    assert (f.channels, f.rate, f.bits) == (case.channels, case.rate, case.bits)
    assert list(f.where) == case.frame_offsets()
    pcm, err = decode(emu, f.audio, f.offsets, f.where, f.config, guarded=True)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


@pytest.mark.parametrize('damaged', KERNEL, ids=lambda d: d[0])
def test_damaged_frame_is_refused_naming_frame_and_offset(emu, tmp_path, damaged):
    name, data, frame, regex, _ = damaged
    f = _tta(tmp_path, name, data)
    for guarded in (False, True):
        pcm, err = decode(emu, f.audio, f.offsets, f.where, f.config, guarded)
        assert pcm is None
        assert err.startswith('TTA frame %d at byte offset %d: ' % (frame, f.where[frame])), err
        assert re.search(regex, err), err


@pytest.mark.parametrize('damaged', [d for d in DAMAGED if not d[4]], ids=lambda d: d[0])
def test_host_refusals_come_before_the_decoder(tmp_path, damaged):
    name, data, frame, regex, _ = damaged
    with pytest.raises(SushiError, match=regex) as e:
        _tta(tmp_path, name, data)
    if frame is not None:
        assert 'TTA frame %d at byte offset ' % frame in str(e.value), str(e.value)


def test_cut_frames_read_nothing_past_their_bytes(emu, tmp_path):
    """Every frame of a case cut at every length from its CRC down, last in a buffer that ends at an inaccessible page:
    the decoder refuses it without reading past it."""
    case = [c for c in CASES if c.name == 'three24'][0]
    f = _tta(tmp_path, case.name, case.tta())
    body = f.audio[:int(f.offsets[1])]
    for cut in list(range(1, 40)) + list(range(40, len(body), 997)):
        pcm, err = decode(emu, body[:len(body) - cut], f.offsets[:1], f.where[:1], f.config, guarded=True)
        assert pcm is None and re.search('reads past the frame|does not end on its CRC|CRC mismatch|shorter', err), err


@pytest.mark.parametrize('mkv', mtc.cases(), ids=lambda m: m[0].name)
def test_matroska_track_decodes_from_its_frames(emu, tmp_path, mkv):
    spec, case, outcome = mkv
    with mk.MatroskaFile(spec.write(tmp_path)) as m:
        t = m.select('audio', None)
        assert mk.audio_codec(t) == 'tta'
        frames = m.frames([t.id])[t.id]
        config = tta.matroska_config(t, m.timestamp_scale, m.duration)
    pcm, err = decode(emu, frames.data, frames.offset, frames.block, config)
    if outcome == 'decoded':
        assert err is None, err
        assert np.array_equal(pcm, case.pcm16)
    else:
        last = len(frames) - 1
        assert err.startswith('TTA frame %d at byte offset %d: ' % (last, frames.block[last])), err


def test_long_stream_frames_decode(emu, tmp_path):
    case, data, reps = tc.long_stream(bits=24, minutes=1)
    f = _tta(tmp_path, 'long', data)
    pcm, err = decode(emu, f.audio, f.offsets, f.where, f.config)
    assert err is None and np.array_equal(pcm, tc.long_pcm16(case, reps))
