"""The ALAC decoder (sushi_b200/csrc/sb_alac.cuh: k_alac_frames' first element, k_alac_decode's frames) on the CPU,
through tests/emu/emu_alac_driver.cpp compiled with g++: every case of tests/alac_cases.py decodes to the writer's
PCM (tests/test_alac_cases.py holds FFmpeg to the same PCM), every A_ALAC Matroska track decodes from its frame table,
and each damaged copy is refused naming the frame and its file offset."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import matroska as mk
from tests import alac_cases as ac
from tests import mkv_alac_cases as mac

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_alac_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_alac.cuh')
CASES = ac.all_cases()
BASE, DAMAGED = ac.damaged_cases()


@pytest.fixture(scope='module')
def emu():
    out = os.path.join(EMU, '_build', 'libsb_emu_alac.so')
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', out])
    lib = ctypes.CDLL(out)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.emu_alac_decode.argtypes = [vp, i64, vp, vp, i64, vp, vp, i64, ctypes.c_char_p, ctypes.c_int]
    lib.emu_alac_decode.restype = i64
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode(emu, data, offsets, where, cfg):
    """-> (int16 pcm, None) or (None, message)"""
    buf = np.frombuffer(data + bytes(16), np.uint8)
    offsets = np.ascontiguousarray(offsets, np.int64)
    where = np.ascontiguousarray(where, np.int64)
    config = cfg.array()
    msg = ctypes.create_string_buffer(256)
    n = emu.emu_alac_decode(_p(buf), len(data), _p(offsets), _p(where), len(offsets), _p(config), None, 0, msg, 256)
    if n < 0:
        return None, msg.value.decode()
    pcm = np.zeros((n + 1, cfg.channels), np.int16)
    assert emu.emu_alac_decode(_p(buf), len(data), _p(offsets), _p(where), len(offsets), _p(config), _p(pcm), n, msg,
                               256) == n
    return pcm[:n], None


def test_cases_cover_the_decoder():
    ac.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES + [BASE], ids=lambda c: c.name)
def test_stream_decodes_to_the_pcm(emu, case):
    pcm, err = decode(emu, case.data, case.offsets, case.offsets + 1000, case.cfg)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


@pytest.mark.parametrize('damaged', DAMAGED, ids=lambda d: d[0])
def test_damaged_frame_is_refused_naming_frame_and_offset(emu, damaged):
    name, cfg, frames, f, regex = damaged
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in frames])[:-1]]).astype(np.int64)
    where = offsets * 3 + 77
    pcm, err = decode(emu, b''.join(frames), offsets, where, cfg)
    assert pcm is None
    assert err.startswith('ALAC frame %d at byte offset %d: ' % (f, where[f])), err
    assert re.search(regex, err), err


GUARDED = r"""
import ctypes, sys
import numpy as np
sys.path.insert(0, {root!r})
from tests import alac_cases as ac
lib = ctypes.CDLL({lib!r})
vp = ctypes.c_void_p
lib.emu_alac_decode_guarded.argtypes = [vp, ctypes.c_int64, vp, vp, ctypes.c_int64, vp, ctypes.c_char_p, ctypes.c_int]
lib.emu_alac_decode_guarded.restype = ctypes.c_int64
for name, cfg, frames, f, regex in ac.damaged_cases()[1]:
    data = np.frombuffer(b''.join(frames), np.uint8)
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in frames])[:-1]]).astype(np.int64)
    config = cfg.array()
    msg = ctypes.create_string_buffer(256)
    p = lambda a: a.ctypes.data_as(vp)
    n = lib.emu_alac_decode_guarded(p(data), len(data), p(offsets), p(offsets), len(offsets), p(config), msg, 256)
    print(name, n, msg.value.decode())
"""


def test_damaged_frames_read_nothing_past_the_padding(emu):
    """Every damaged copy again, with the 8 bytes of padding the library guarantees ending at an inaccessible page, in a
    child process: a read further past the last frame would kill it."""
    code = GUARDED.format(root=ROOT, lib=os.path.join(EMU, '_build', 'libsb_emu_alac.so'))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stdout.splitlines()
    assert len(lines) == len(DAMAGED)
    for line, (name, _, _, f, regex) in zip(lines, DAMAGED):
        assert line.startswith(name + ' -1 ALAC frame %d at byte offset' % f) and re.search(regex, line), line


@pytest.mark.parametrize('pair', mac.cases()[::4], ids=lambda p: p[0].name)
def test_matroska_track_decodes_from_its_frames(emu, tmp_path, pair):
    mkv, case = pair
    with mk.MatroskaFile(mkv.write(tmp_path)) as f:
        t = f.select('audio', None)
        assert mk.audio_codec(t) == 'alac'
        table = f.frames([t.id])[t.id]
    cfg = ac.Config(*[int(v) for v in _config(t.codec_private)])
    pcm, err = decode(emu, table.data, table.offset, table.block, cfg)
    assert err is None, err
    assert np.array_equal(pcm, case.pcm16)


def _config(cookie):
    import struct
    fl, _, depth, pb, mb, kb, ch, _, _, _, rate = struct.unpack('>IBBBBBBHIII', cookie[:24])
    return fl, depth, pb, mb, kb, ch, rate


def test_escape_stream_and_long_stream_frames_decode(emu):
    rng = np.random.default_rng(3)
    pcm = rng.integers(-32768, 32768, (10000, 2))
    case = ac.escape_stream(pcm, ac.Config(frame_length=4096, bit_depth=16, channels=2))
    got, err = decode(emu, case.data, case.offsets, case.offsets, case.cfg)
    assert err is None and np.array_equal(got, case.pcm16)
    cfg, frames, pcm, _ = ac.long_stream()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in frames])[:-1]])
    got, err = decode(emu, b''.join(frames), offsets, offsets, cfg)
    assert err is None and np.array_equal(got, ac.to16(pcm, 24))
