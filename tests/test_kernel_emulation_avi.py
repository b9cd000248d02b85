"""The CPU build of sushi_b200/csrc/sb_avi.cuh (tests/emu/emu_avi_driver.cpp, compiled with g++), driven as sb_avi.cu
drives it, against FFmpeg's `avi` demuxer (tests/ref_avi.py):
  - the elementary stream of every audio stream of every case equals FFmpeg's packets concatenated, with the file fed
    in 1-byte chunks, in chunks that cut chunk headers, and in one 64 MB chunk; each chunk's file offset is named;
  - every damaged copy is refused naming the expected offset, where FFmpeg resyncs and demuxes on;
  - PCM chunks that are not whole sample frames are refused by name, where FFmpeg's decoder drops the partial frame;
  - a cut copy keeps the bytes of the chunk the file cuts and says it was cut."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from sushi_b200 import avi
from tests import avi_cases as ac
from tests import ref_avi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_avi_driver.cpp')
SOURCES = [DRIVER, os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_avi.cuh')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_avi.so')
GOOD = ac.good_cases()
CHUNKS = (64 << 20, 4099, 777, 13, 12, 9, 5)


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-I',
                               os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.emu_avi_demux.argtypes = [vp, i64, ctypes.c_uint32, i64, vp, i64, i64, vp, i64, vp, i64, vp, ctypes.c_char_p,
                                  ctypes.c_int]
    lib.emu_avi_demux.restype = i64
    return lib


def demux(emu, data, extents, sid, chunk, frame_bytes=0):
    """-> (elementary stream bytes, chunk file offsets, cut) or (None, message)"""
    buf = np.frombuffer(data, np.uint8)
    ext = np.array(extents or [(0, 0)], np.int64).reshape(-1)
    es = np.zeros(len(data) + 1, np.uint8)
    offs = np.zeros(len(data) // 8 + 1, np.int64)
    info = np.zeros(2, np.int64)
    msg = ctypes.create_string_buffer(256)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    tag = int.from_bytes(b'%02dwb' % sid, 'little')
    n = emu.emu_avi_demux(p(buf), len(data), tag, frame_bytes, p(ext), len(extents), chunk, p(es), len(es), p(offs),
                          len(offs), p(info), msg, 256)
    if n < 0:
        return None, msg.value.decode()
    return es[:n].tobytes(), [int(x) for x in offs[:info[0]]], int(info[1])


def frame_bytes(s):
    return s.channels * s.bits // 8 if s.codec == 'pcm' else 0


@pytest.mark.parametrize('case', GOOD, ids=repr)
def test_emulation_gives_ffmpegs_stream_bytes(emu, tmp_path, case):
    path = case.write(tmp_path)
    f = avi.AviFile(path)
    for sid, s in case.audio():
        want = b''.join(ref_avi.packets(path, sid))
        assert want == s.es
        kept = [o for o, c in zip(s.offsets, (s.chunks[k] for i, k in case.order if i == sid)) if c]
        for chunk in CHUNKS + (1,):
            es, offs, cut = demux(emu, case.data, f.movi, sid, chunk, frame_bytes(s))
            assert es == want, chunk
            assert offs == kept and cut == 0


def test_chunk_sizes_cut_chunk_headers():
    """the small feed sizes put feed boundaries inside chunk headers and LIST rec headers of the audio"""
    for case in GOOD:
        heads = [o for _, s in case.audio() for o in s.offsets]
        cuts = [sum(o < c < o + 8 for o in heads for c in range(chunk, len(case.data), chunk)) for chunk in CHUNKS]
        assert sum(cuts) >= 3, (case, cuts)


@pytest.mark.parametrize('damaged', ac.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_the_offset(emu, tmp_path, damaged):
    name, data, offset, regex = damaged
    base = ac.damaged_cases()[0]
    path = base.write(tmp_path, data, '_' + name + '.avi')
    f = avi.AviFile(path)
    for chunk in (64 << 20, 1000, 33, 7):
        got, msg = demux(emu, data, f.movi, 1, chunk, 4)[:2]
        assert got is None
        assert msg.startswith('AVI chunk at byte offset %d: ' % offset), msg
        assert regex in msg
    # FFmpeg resyncs by scanning for the next chunk header (and takes `01w\x01` for a chunk of stream 1) and demuxes on
    got = b''.join(ref_avi.packets(path, 1))
    assert len(got) >= len(base.streams[1].es) // 2


def test_partial_pcm_frames_are_refused(emu, tmp_path):
    case, sid, offset = ac.partial_frame_case()
    path = case.write(tmp_path)
    f = avi.AviFile(path)
    for chunk in (64 << 20, 100, 3):
        got, msg = demux(emu, case.data, f.movi, sid, chunk, 4)[:2]
        assert got is None and msg == 'AVI chunk at byte offset %d: PCM chunk is not a whole number of sample ' \
                                       'frames' % offset
    # FFmpeg's decoder drops the partial frame of the packet
    pcm, _ = ref_avi.decode_pcm(path, sid, 2, 16)
    assert len(pcm) == len(case.streams[sid].es) // 4


def test_cut_copy_keeps_the_cut_chunk(emu, tmp_path):
    base, data, before = ac.cut_case()
    path = base.write(tmp_path, data, '_cut.avi')
    f = avi.AviFile(path)
    want = b''.join(ref_avi.packets(path, 1))
    assert base.streams[1].es.startswith(want) and len(want) < len(base.streams[1].es)
    for chunk in (64 << 20, 999, 40):
        es, offs, cut = demux(emu, data, f.movi, 1, chunk, 4)
        assert es == want and cut == 1 and len(offs) == before + 1
