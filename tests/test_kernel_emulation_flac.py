"""The FLAC decoder of sushi_b200/csrc/sb_flac.cuh on the CPU (tests/emu/emu_flac_driver.cpp, compiled with g++): every
case of tests/flac_cases.py decodes bit for bit to the int16 samples the WAV loader reads of the same PCM, and every
damaged file fails with the message that names its frame and byte offset."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from sushi_b200.wavstream import FlacFile
from tests import flac_cases as fc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_flac_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_flac.cuh')
CASES = fc.all_cases()
BASE, CORRUPT = fc.corrupt_cases()


def build(out, extra=()):
    """Compiles the driver into `out` unless it is newer than the driver and the header."""
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)) or extra:
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function'] + list(extra) +
                              ['-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', out])


def load(out):
    lib = ctypes.CDLL(out)
    vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.emu_flac_index.argtypes = [vp, i64, i64, ci, ci, ci, ctypes.c_char_p, ci]
    lib.emu_flac_index.restype = i64
    lib.emu_flac_decode.argtypes = [vp, i64, i64, ci, ci, ci, vp, ctypes.c_char_p, ci]
    lib.emu_flac_decode.restype = ci
    return lib


@pytest.fixture(scope='module')
def emu():
    out = os.path.join(EMU, '_build', 'libsb_emu_flac.so')
    build(out)
    return load(out)


def emu_decode(lib, path):
    """-> (int16 samples (frames, channels), None) or (None, message)."""
    info = FlacFile(path)
    data = np.frombuffer(info.data, np.uint8)
    msg = ctypes.create_string_buffer(256)
    args = (data.ctypes.data_as(ctypes.c_void_p), len(data), info.frame_offset, info.channels_count,
            info.bits_per_sample, info.framerate)
    n = lib.emu_flac_index(*args, msg, 256)
    if n < 0:
        return None, msg.value.decode()
    out = np.zeros((n, info.channels_count), np.int16)
    if lib.emu_flac_decode(*args, out.ctypes.data_as(ctypes.c_void_p), msg, 256) != 0:
        return None, msg.value.decode()
    if info.total_samples and info.total_samples != n:
        return None, 'FLAC STREAMINFO says {0} samples, the frames hold {1}'.format(info.total_samples, n)
    return out, None


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_emulated_decoder_matches_the_pcm(emu, tmp_path, case):
    got, err = emu_decode(emu, case.write(tmp_path))
    assert err is None, err
    assert np.array_equal(got, case.pcm16())


@pytest.mark.parametrize('case', CORRUPT, ids=lambda c: c.name)
def test_emulated_decoder_names_the_corrupt_frame(emu, tmp_path, case):
    got, err = emu_decode(emu, case.write(tmp_path))
    assert got is None and err is not None
    assert re.search(case.corrupt[3], err), err


def test_emulated_decoder_decodes_the_undamaged_base(emu, tmp_path):
    got, err = emu_decode(emu, BASE.write(tmp_path))
    assert err is None and np.array_equal(got, BASE.pcm16())
