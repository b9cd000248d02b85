"""MPEG program streams on the CPU: the writer of tests/ps_cases.py, sushi_b200.mpegps and the CPU build of
sushi_b200/csrc/sb_ps.cuh (tests/emu/emu_ps_driver.cpp, compiled with g++) against FFmpeg's `mpeg` demuxer
(tests/ref_ps.py):
  - the stream list mpegps.py reads (order, FFmpeg's ids, kinds, codec names) equals FFmpeg's on every case;
  - the emulation driver gives the chosen stream's bytes FFmpeg's demuxer returns, at chunk sizes that split start
    codes, pack headers and PES packets, and names each PES's file offset;
  - every damaged copy is refused naming the expected offset, where FFmpeg resyncs and demuxes on;
  - a cut copy keeps the bytes of the PES the file cuts;
  - selection and the refusals by codec name."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from sushi_b200 import mpegps
from sushi_b200.common import SushiError
from tests import ps_cases as pc
from tests import ref_ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_ps_driver.cpp')
SOURCES = [DRIVER, os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_ps.cuh')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_ps.so')
GOOD = pc.good_cases()
CHUNKS = (1 << 20, 4096, 2051, 777, 37, 17, 6)


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-I',
                               os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.emu_ps_demux.argtypes = [vp, i64, ctypes.c_int, i64, vp, i64, vp, i64, vp, ctypes.c_char_p, ctypes.c_int]
    lib.emu_ps_demux.restype = i64
    return lib


def demux(emu, data, stream_id, chunk):
    """-> (elementary stream bytes, PES file offsets, cut) or (None, message)"""
    buf = np.frombuffer(data, np.uint8)
    es = np.zeros(len(data) + 1, np.uint8)
    pes = np.zeros(len(data) // 6 + 1, np.int64)
    info = np.zeros(2, np.int64)
    msg = ctypes.create_string_buffer(256)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    n = emu.emu_ps_demux(p(buf), len(data), stream_id, chunk, p(es), len(es), p(pes), len(pes), p(info), msg, 256)
    if n < 0:
        return None, msg.value.decode()
    return es[:n].tobytes(), [int(x) for x in pes[:info[0]]], int(info[1])


@pytest.mark.parametrize('case', GOOD + list(pc.refused_cases()), ids=lambda c: c.name)
def test_stream_list_equals_ffmpeg(tmp_path, case):
    path = case.write(tmp_path)
    ps = mpegps.ProgramStream(path)
    mine = [dict(id=s.stream_id, kind=s.kind, codec=s.codec) for s in ps.streams_all]
    assert [s.id for s in ps.streams_all] == list(range(len(mine)))
    assert mine == ref_ps.streams(path)


@pytest.mark.parametrize('case', GOOD, ids=lambda c: c.name)
def test_emulation_gives_ffmpegs_stream_bytes(emu, tmp_path, case):
    path = case.write(tmp_path)
    ps = mpegps.ProgramStream(path)
    for e in case.audio():
        s = next(t for t in ps.streams_all if t.stream_id == 0x100 | e.sid)
        want = b''.join(ref_ps.packets(path, s.id))
        assert want == e.es
        for chunk in CHUNKS:
            es, pes, cut = demux(emu, case.data, e.sid, chunk)
            assert es == want, (chunk, pes)
            assert pes == e.pes_offsets and cut == 0


def test_cases_split_where_they_should():
    """chunk boundaries of CHUNKS fall inside start codes, pack headers and PES packets of the audio"""
    data = GOOD[1].data
    a = GOOD[1].audio()[0]
    codes = [i for i in range(len(data) - 3) if data[i:i + 3] == b'\x00\x00\x01' and data[i + 3] >= 0xB9]
    cuts = [range(chunk, len(data), chunk) for chunk in CHUNKS[2:]]
    assert sum(any(o < c < o + 20 for c in cs for o in a.pes_offsets) for cs in cuts) >= 3   # inside a PES header
    assert sum(any(x < c < x + 4 for c in cs for x in codes) for cs in cuts) >= 3          # inside a start code


@pytest.mark.parametrize('damaged', pc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_the_offset(emu, tmp_path, damaged):
    name, data, offset, regex = damaged
    for chunk in (1 << 20, 1000, 33):
        got, msg = demux(emu, data, pc.AUDIO, chunk)[:2]
        assert got is None
        assert msg.startswith('%s at byte offset %d: ' % (
            'PES packet' if 'PES header' in regex else 'program stream packet', offset)), msg
        assert regex in msg
    # FFmpeg resyncs by scanning for the next start code: it still lists the stream and demuxes it, less what it
    # skipped
    base = pc.damaged_cases()[0]
    path = base.write(tmp_path, data, '_' + name + '.vob')
    streams = ref_ps.streams(path)
    sid = next(i for i, s in enumerate(streams) if s['id'] == 0x1C0)
    got = b''.join(ref_ps.packets(path, sid))
    want = base.audio()[0].es
    if name == 'broken_start_code':                       # that PES is lost
        assert len(got) < len(want)
    elif name == 'bad_pes_header':                        # that PES is skipped
        assert len(got) < len(want)
    else:                                                 # the packets after the fault are found again
        assert len(got) >= len(want) - 2100 and got != b''


def test_cut_copy_keeps_the_cut_pes(emu, tmp_path):
    base, data, before = pc.cut_case()
    a = base.audio()[0]
    path = base.write(tmp_path, data, '_cut.mpg')
    sid = next(s.id for s in mpegps.ProgramStream(path).streams_all if s.stream_id == 0x1C0)
    want = b''.join(ref_ps.packets(path, sid))
    assert a.es.startswith(want) and len(want) < len(a.es)
    for chunk in (1 << 20, 999, 40):
        es, pes, cut = demux(emu, data, pc.AUDIO, chunk)
        assert es == want and cut == 1 and len(pes) == before + 1


def test_selection_and_refusals(tmp_path):
    two = mpegps.ProgramStream(next(c for c in GOOD if c.name == 'two_audio').write(tmp_path))
    with pytest.raises(SushiError, match='More than one audio stream found'):
        two.select('audio', None)
    assert two.select('audio', 0).stream_id == 0x1C1 and two.select('audio', 2).stream_id == 0x1C0
    with pytest.raises(SushiError, match="Stream with index 1 doesn't exist"):
        two.select('audio', 1)
    assert two.select_audio(0).label == 'MP2' and two.chapters == []
    dvd = mpegps.ProgramStream(next(c for c in GOOD if c.name == 'dvd_joint').write(tmp_path))
    assert dvd.select('subtitles', None).script_type == 'dvd_subtitle'
    for sid, codec in ((1, 'pcm_dvd'), (3, 'ac3')):
        with pytest.raises(SushiError, match=r'^Audio track {0} is {1}, which cannot be decoded here'.format(sid, codec)):
            dvd.select_audio(sid)
    l3, lossy = pc.refused_cases()
    with pytest.raises(SushiError, match=r'^Audio track 0 is MPEG audio layer III \(MP3\), which cannot be decoded'):
        mpegps.ProgramStream(l3.write(tmp_path)).select_audio()
    with pytest.raises(SushiError, match=r'^Audio track 2 is dts, which cannot be decoded here'):
        mpegps.ProgramStream(lossy.write(tmp_path)).select_audio(2)
    bad = tmp_path / 'x.mpg'
    bad.write_bytes(b'\x00\x00\x01\xb3' + bytes(100))
    with pytest.raises(SushiError, match='not a program stream'):
        mpegps.ProgramStream(str(bad))
    assert mpegps.is_program_stream('A.VOB') and mpegps.is_program_stream('b.m2p') and \
        not mpegps.is_program_stream('c.ts')
