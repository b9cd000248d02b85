"""The TrueHD decoder (sushi_b200/csrc/sb_truehd.cuh: k_truehd_sync's candidates, the host chain, k_truehd_decode's
segments and the joined checks) on the CPU, through tests/emu/emu_truehd_driver.cpp compiled with g++: every case of
tests/truehd_cases.py decodes to the PCM FFmpeg gives (tests/test_truehd_cases.py holds FFmpeg to the same PCM), every
Matroska track of tests/mkv_truehd_cases.py decodes from its frame table, and each damaged copy is refused naming the
access unit and its byte offset.  A 90-minute 24-bit 7.1 stream (about 1.2 GB, byte offsets past 2^32 bits)
decodes to its PCM."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from sushi_b200 import matroska as mk
from tests import mkv_truehd_cases as mtc
from tests import truehd_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_truehd_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_truehd.cuh')
BASE, DAMAGED = tc.damaged_cases()


@pytest.fixture(scope='module')
def emu():
    out = os.path.join(EMU, '_build', 'libsb_emu_truehd.so')
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-fopenmp', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', out])
    lib = ctypes.CDLL(out)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.emu_truehd_decode.argtypes = [vp, i64, vp, vp, i64, vp, i64, vp, ctypes.c_char_p, ctypes.c_int, vp, i64, vp]
    lib.emu_truehd_decode.restype = i64
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, data, blocks, where):
    """-> (int16 pcm, None) or (None, message)"""
    buf = np.frombuffer(data + b'\0', np.uint8)
    blocks = np.ascontiguousarray(blocks, np.int64)
    where = np.ascontiguousarray(where, np.int64)
    info = np.zeros(2, np.int32)
    msg = ctypes.create_string_buffer(256)
    n = emu.emu_truehd_decode(_p(buf), len(data), _p(blocks), _p(where), len(blocks), None, 0, _p(info), msg, 256,
                              None, 0, None)
    if n < 0:
        return None, msg.value.decode()
    pcm = np.zeros((n + 1, int(info[0])), np.int16)
    assert emu.emu_truehd_decode(_p(buf), len(data), _p(blocks), _p(where), len(blocks), _p(pcm), n, _p(info), msg,
                                 256, None, 0, None) == n
    return pcm[:n], None


@pytest.mark.parametrize('case', tc.all_cases() + [BASE], ids=lambda c: c.name)
def test_stream_decodes_to_the_pcm(emu, case):
    pcm, err = decode(emu, case.data, [0], [-1])
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


@pytest.mark.parametrize('case', DAMAGED, ids=lambda c: c.name)
def test_damaged_stream_is_refused_naming_the_access_unit(emu, case):
    pcm, err = decode(emu, case.data, [0], [-1])
    assert pcm is None and re.search(case.damage[3], err), err


@pytest.mark.parametrize('pair', mtc.cases(), ids=lambda p: p[0].name)
def test_matroska_track_decodes_from_its_frames(emu, tmp_path, pair):
    mkv, case = pair
    with mk.MatroskaFile(mkv.write(tmp_path)) as f:
        t = f.select('audio', None)
        assert mk.audio_codec(t) == 'truehd'
        table = f.frames([t.id])[t.id]
    pcm, err = decode(emu, table.data, table.offset, table.block)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)
    # an AU that runs past its lace is named by the file offset of its block
    cut = bytearray(table.data)
    k = len(table.offset) // 2
    end = int(table.offset[k + 1]) if k + 1 < len(table.offset) else len(cut)
    del cut[end - 2:end]
    offs = np.array([o if o < end else o - 2 for o in table.offset], np.int64)
    pcm, err = decode(emu, bytes(cut), offs, table.block)
    assert pcm is None and 'byte offset %d:' % table.block[k] in err, err


def test_ninety_minute_stream_decodes_to_its_pcm(emu):
    seg, pcm, reps = tc.long_stream()
    buf = np.zeros(len(seg) * reps + 1, np.uint8)
    buf[:-1] = np.tile(np.frombuffer(seg, np.uint8), reps)
    assert (len(buf) - 1) * 8 > 2 ** 32
    blocks, where = np.zeros(1, np.int64), np.full(1, -1, np.int64)
    info = np.zeros(2, np.int32)
    msg = ctypes.create_string_buffer(256)
    bad = np.zeros(1, np.int64)
    expect = np.ascontiguousarray(pcm)
    n = emu.emu_truehd_decode(_p(buf), len(buf) - 1, _p(blocks), _p(where), 1, None, 0, _p(info), msg, 256, _p(expect),
                              len(pcm), _p(bad))
    assert n == len(pcm) * reps == 90 * 60 * 48000, msg.value
    assert tuple(info) == (8, 48000) and bad[0] == 0
