"""The transport stream demuxer and BD-LPCM decoder (sushi_b200/csrc/sb_ts.cuh: k_ts_scan's packet checks, the
compaction, k_ts_cc's continuity check, k_pes_index and k_bdlpcm_decode) on the CPU, through tests/emu/emu_ts_driver.cpp
compiled with g++.  Every case of tests/ts_cases.py, fed in chunks of several sizes (PES packets split across chunk
edges), decodes to the writer's PCM (a TrueHD stream to the writer's .thd bytes, which the TrueHD emulation decodes);
each damaged copy is refused naming its byte offset; a cut copy keeps what FFmpeg keeps."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from tests import ts_cases as tsc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_ts_driver.cpp')
HEADER = os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_ts.cuh')
CHUNKS = (7, 64, 1000)                 # packets per feed


@pytest.fixture(scope='module')
def emu():
    out = os.path.join(EMU, '_build', 'libsb_emu_ts.so')
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(DRIVER), os.path.getmtime(HEADER)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-Wno-format-security',
                               '-I', os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', out])
    lib = ctypes.CDLL(out)
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.emu_ts_decode.argtypes = [vp, i64, i32, i32, i32, i64, vp, i64, vp, ctypes.c_char_p, i32]
    lib.emu_ts_decode.restype = i64
    return lib


def decode(emu, data, psize, pid, codec, chunk_packets):
    """-> (int16 pcm or bytes, info, None) or (None, None, message)"""
    buf = np.frombuffer(bytes(data) + b'\0', np.uint8)
    info = np.zeros(4, np.int32)
    msg = ctypes.create_string_buffer(256)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    n = emu.emu_ts_decode(p(buf), len(data), psize, pid, codec, chunk_packets * psize, None, 0, p(info), msg, 256)
    if n < 0:
        return None, None, msg.value.decode()
    out = np.zeros((n + 1) * (8 if codec == 0 else 1), np.int16 if codec == 0 else np.uint8)
    assert emu.emu_ts_decode(p(buf), len(data), psize, pid, codec, chunk_packets * psize, p(out), n, p(info), msg,
                             256) == n
    if codec == 1:
        return out[:n].tobytes(), info, None
    return out[:n * info[0]].reshape(n, info[0]), info, None


DECODED = [(c, s) for c in tsc.all_cases() if c.hdmv and not c.refused and c.name != 'bd_stereo20_48k'
           for s in c.audio()]


@pytest.mark.parametrize('pair', DECODED, ids=lambda p: '%s-%x' % (p[0].name, p[1].pid))
@pytest.mark.parametrize('chunk', CHUNKS)
def test_every_stream_decodes_to_its_pcm(emu, pair, chunk):
    case, s = pair
    got, info, err = decode(emu, case.data, case.psize, s.pid, 1 if s.kind == 'truehd' else 0, chunk)
    assert err is None, err
    if s.kind == 'truehd':
        thd = b''.join(p[s.header_len:] for p, f in zip(s.pes, s.pes_frames) if f is not None)
        assert got == thd
        return
    assert tuple(info) == (s.channels, s.rate, s.bits, 0)
    assert np.array_equal(got, s.pcm)


def test_twenty_bit_lpcm_is_refused(emu):
    c = tsc.case('bd_stereo20_48k')
    _, _, err = decode(emu, c.data, c.psize, tsc.AUDIO_PID, 0, 64)
    assert re.search(r'PES packet at byte offset %d: 20-bit BD-LPCM' % c.pes_offset(tsc.AUDIO_PID, 0), err), err


@pytest.mark.parametrize('case', [c for c in tsc.damaged_cases() if not c.name.endswith(('_pat_crc', '_pmt_crc'))],
                         ids=lambda c: c.name)
@pytest.mark.parametrize('chunk', (5, 1000))
def test_damaged_copy_is_refused_naming_its_offset(emu, case, chunk):
    _, _, err = decode(emu, case.data, case.psize, tsc.AUDIO_PID, 0, chunk)
    regex, offset = case.damage
    assert err is not None and re.search(regex, err) and 'byte offset %d:' % offset in err, err


@pytest.mark.parametrize('case', tsc.cut_cases(), ids=lambda c: c.name)
def test_cut_copy_keeps_the_whole_frames_ffmpeg_keeps(emu, case):
    s = next(x for x in case.streams if x.kind == 'lpcm')
    got, info, err = decode(emu, case.data, case.psize, s.pid, 0, 64)
    assert err is None, err
    assert info[3] == 1 and np.array_equal(got, case.expected(s))
