"""The WavPack decoder (sushi_b200/csrc/sb_wavpack.cuh, k_wavpack_decode's blocks) on the CPU, through
tests/emu/emu_wavpack_driver.cpp compiled with g++, fed the block tables of sushi_b200/wavpack.py: every case of
tests/wavpack_cases.py decodes to the writer's PCM (tests/test_wavpack_cases.py holds FFmpeg to the same PCM), every
A_WAVPACK4 Matroska track decodes from its frame table, and each copy the GPU refuses is refused naming the block and its
file offset, again with the padding ending at an inaccessible page."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError
from sushi_b200 import matroska as mk
from sushi_b200 import wavpack as wp
from tests import mkv_wavpack_cases as mwc
from tests import wavpack_cases as wc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_wavpack_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_wavpack.cuh')
LIB = os.path.join(EMU, '_build', 'libsb_emu_wavpack.so')
CASES = wc.all_cases()
BASE, DAMAGED = wc.damaged_cases()
KERNEL = [d for d in DAMAGED if d[4]]


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    for name in ('emu_wavpack_decode', 'emu_wavpack_decode_guarded'):
        getattr(lib, name).argtypes = [vp, i64, vp, i64, ctypes.c_int, i64, vp, ctypes.c_char_p, ctypes.c_int]
        getattr(lib, name).restype = ctypes.c_int
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, data, table, channels, guarded=False):
    """-> (int16 pcm, None) or (None, message)"""
    table = np.ascontiguousarray(table, np.int64)
    frames = int((table[:, 5] + table[:, 2]).max())
    pcm = np.zeros((frames + 1, channels), np.int16)
    msg = ctypes.create_string_buffer(256)
    if guarded:
        buf = np.frombuffer(data, np.uint8)
        rc = emu.emu_wavpack_decode_guarded(_p(buf), len(data), _p(table), len(table), channels, frames, _p(pcm), msg,
                                            256)
    else:
        buf = np.frombuffer(data + bytes(16), np.uint8)
        rc = emu.emu_wavpack_decode(_p(buf), len(data), _p(table), len(table), channels, frames, _p(pcm), msg, 256)
    if rc:
        return None, msg.value.decode()
    return pcm[:frames], None


def _wv(tmp_path, name, data):
    path = str(tmp_path / (name + '.wv'))
    with open(path, 'wb') as f:
        f.write(data)
    return wp.WavPackFile(path)


def test_cases_cover_the_decoder():
    wc.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_stream_decodes_to_the_pcm(emu, tmp_path, case):
    f = _wv(tmp_path, case.name, case.wv())
    assert (f.stream.channels, f.stream.rate, f.stream.bits_per_sample) == (case.channels, case.rate, case.bits)
    pcm, err = decode(emu, f.data, f.table, case.channels)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


@pytest.mark.parametrize('damaged', KERNEL, ids=lambda d: d[0])
def test_damaged_block_is_refused_naming_block_and_offset(emu, tmp_path, damaged):
    name, data, block, regex, _ = damaged
    f = _wv(tmp_path, name, data)
    pcm, err = decode(emu, f.data, f.table, f.stream.channels)
    assert pcm is None
    assert err.startswith('WavPack block %d at byte offset %d: ' % (block, f.where[block])), err
    assert re.search(regex, err), err


@pytest.mark.parametrize('damaged', [d for d in DAMAGED if not d[4]], ids=lambda d: d[0])
def test_host_refusals_come_before_the_decoder(tmp_path, damaged):
    name, data, block, regex, _ = damaged
    with pytest.raises(SushiError, match=regex) as e:
        _wv(tmp_path, name, data)
    if block is not None and 'is WavPack (' not in str(e.value):
        assert 'WavPack block %d at byte offset ' % block in str(e.value), str(e.value)


def test_damaged_blocks_read_nothing_past_the_padding(emu, tmp_path):
    """Every case and every copy the GPU refuses again, with the 8 bytes of padding the library guarantees ending at an
    inaccessible page: a read further past the last block would kill the test process."""
    for case in CASES:
        f = _wv(tmp_path, case.name, case.wv())
        pcm, err = decode(emu, f.data, f.table, case.channels, guarded=True)
        assert err is None and np.array_equal(pcm, case.pcm16), case.name
    for name, data, block, regex, _ in KERNEL:
        f = _wv(tmp_path, name, data)
        for cut in (0, 1):                     # the damaged block last in the buffer
            keep = f.table[:block + 1]
            end = int(keep[-1, 0] + keep[-1, 1]) if cut else len(f.data)
            pcm, err = decode(emu, f.data[:end], keep, f.stream.channels, guarded=True)
            assert pcm is None and re.search(regex, err), (name, err)


@pytest.mark.parametrize('mkv', mwc.cases(), ids=lambda m: m[0].name)
def test_matroska_track_decodes_from_its_frames(emu, tmp_path, mkv):
    spec, case = mkv
    with mk.MatroskaFile(spec.write(tmp_path)) as f:
        t = f.select('audio', None)
        assert mk.audio_codec(t) == 'wavpack'
        frames = f.frames([t.id])[t.id]
    table, stream = wp.matroska_table(frames, t.codec_private, t.id, t.channels)
    pcm, err = decode(emu, frames.data, table, stream.channels)
    assert err is None, err
    n = min(len(pcm), len(case.pcm16))
    assert len(pcm) == (n if spec.name.endswith('_cut') else len(case.pcm16))
    assert np.array_equal(pcm, case.pcm16[:n])


def test_long_stream_blocks_decode(emu, tmp_path):
    case, data, reps = wc.long_stream(bits=24, minutes=1, block=4800)
    f = _wv(tmp_path, 'long', data)
    pcm, err = decode(emu, f.data, f.table, 2)
    assert err is None and np.array_equal(pcm, np.tile(case.pcm16, (reps, 1)))
