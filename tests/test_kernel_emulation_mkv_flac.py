"""The listed-frame path of the FLAC decoder (k_flac_frames' per-frame logic and the table sb_flac_decode_frames builds,
from sushi_b200/csrc/sb_flac.cuh) on the CPU, through tests/emu/emu_flac_frames_driver.cpp compiled with g++:

* listing every frame of every uncut FLAC case of tests/flac_cases.py at its offset builds the same frame table as the
  sync-code chain of sb_flac_decode_file;
* every FLAC track of tests/mkv_cases.py decodes bit for bit to its PCM, the cut track (frame numbers from 5, a stale
  STREAMINFO total) included;
* a frame with a bad CRC-8 or CRC-16 is named with the file offset of the block holding it."""
import ctypes
import os
import re

import numpy as np
import pytest

from sushi_b200 import matroska as mk
from sushi_b200.wavstream import FlacFile
from tests import flac_cases as fc
from tests import mkv_cases as mc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_flac_frames_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_flac.cuh')
MKV = [c for c in mc.all_cases() if any(s.codec == 'A_FLAC' for s in c.specs) and c.refused is None
       and (c.damage is None or c.damage[0] in ('crc8', 'crc16'))]


@pytest.fixture(scope='module')
def emu():
    out = os.path.join(EMU, '_build', 'libsb_emu_flac_frames.so')
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)):
        import subprocess
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-I',
                               os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', out])
    lib = ctypes.CDLL(out)
    vp, i64, ci, cs = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_char_p
    lib.emu_flac_frames.argtypes = [vp, i64, vp, vp, i64, ci, ci, ci, vp, cs, ci]
    lib.emu_flac_frames.restype = i64
    lib.emu_flac_chain_table.argtypes = [vp, i64, i64, ci, ci, ci, vp, i64, cs, ci]
    lib.emu_flac_chain_table.restype = i64
    lib.emu_flac_frames_decode.argtypes = [vp, i64, vp, vp, i64, ci, ci, ci, vp, cs, ci]
    lib.emu_flac_frames_decode.restype = ci
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize('case', fc.all_cases(), ids=lambda c: c.name)
def test_listed_frames_build_the_chained_table(emu, case):
    info = FlacFile.from_bytes(case.flac, case.name)
    buf = np.frombuffer(case.flac, np.uint8)
    offsets = np.ascontiguousarray(case.offsets[:-1], np.int64)
    n = len(offsets)
    msg = ctypes.create_string_buffer(256)
    chained = np.zeros((max(n, 1), 5), np.int64)
    assert emu.emu_flac_chain_table(_p(buf), len(buf), info.frame_offset, info.channels_count, info.bits_per_sample,
                                    info.framerate, _p(chained), n, msg, 256) == n, msg.value
    listed = np.zeros((max(n, 1), 5), np.int64)
    samples = emu.emu_flac_frames(_p(buf), len(buf), _p(offsets), _p(offsets), n, info.channels_count,
                                  info.bits_per_sample, info.framerate, _p(listed), msg, 256)
    assert samples == len(case.pcm), msg.value
    assert np.array_equal(listed[:n], chained[:n])


def _track(path, case):
    with mk.MatroskaFile(path) as f:
        t = [t for t in f.tracks if t.codec_id == 'A_FLAC'][0]
        info = FlacFile.from_bytes(t.codec_private, case.name)
        return t, info, f.frames([t.id])[t.id]


def _decode(emu, info, table):
    buf = np.frombuffer(table.data + b'\0', np.uint8)
    offsets = np.ascontiguousarray(table.offset, np.int64)
    where = np.ascontiguousarray(table.block, np.int64)
    msg = ctypes.create_string_buffer(256)
    tab = np.zeros((max(len(offsets), 1), 5), np.int64)
    n = emu.emu_flac_frames(_p(buf), len(table.data), _p(offsets), _p(where), len(offsets), info.channels_count,
                            info.bits_per_sample, info.framerate, _p(tab), msg, 256)
    if n < 0:
        return None, msg.value.decode()
    pcm = np.zeros((n, info.channels_count), np.int16)
    if emu.emu_flac_frames_decode(_p(buf), len(table.data), _p(offsets), _p(where), len(offsets), info.channels_count,
                                  info.bits_per_sample, info.framerate, _p(pcm), msg, 256) != 0:
        return None, msg.value.decode()
    return pcm, None


@pytest.mark.parametrize('case', [c for c in MKV if c.damage is None], ids=lambda c: c.name)
def test_matroska_flac_tracks_decode_to_the_pcm(emu, tmp_path, case):
    t, info, table = _track(case.write(tmp_path), case)
    pcm, err = _decode(emu, info, table)
    assert err is None, err
    spec = case.specs[t.id]
    assert np.array_equal(pcm, (spec.pcm >> (spec.bits - 16)).astype(np.int16))
    if case.name == 'cut':
        assert info.total_samples > len(pcm)                       # the stale STREAMINFO total is not checked
        assert table.frame(0)[4] != 0                              # and the first frame number is not 0


@pytest.mark.parametrize('case', [c for c in MKV if c.damage], ids=lambda c: c.name)
def test_damaged_frame_is_named_by_its_block(emu, tmp_path, case):
    _, info, table = _track(case.write(tmp_path), case)
    pcm, err = _decode(emu, info, table)
    assert pcm is None and re.search(case.damage[2], err), err
