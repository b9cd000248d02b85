"""WavStream(path, ffmpeg_audio=True) on the GPU: an input that is not a WAV file loads bit for bit as WavStream loads
the mono pcm_s16le WAV the reference's ffmpeg call writes for it, that WAV made here by libswresample itself
(tests/ref_swr.py, FMA3 path) from the writer's PCM.  Raw FLAC, Matroska FLAC and 16-bit little-endian PCM, raw
TTA and WavPack; stereo, 5.1 and mono; downsampling, upsampling, an inexact ratio and equal rates (the integer path);
90 minutes of stereo and of 5.1 through sb_pcm_swr; the refusals; and the command line with --ffmpeg-audio against the
run on the two WAVs."""
import ctypes
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, WavStream, _native, swr
from tests import flac_cases as fc
from tests import mkv_cases as mc
from tests import ref_swr
from tests import tta_cases as tc
from tests import wavpack_cases as wc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def wav_bytes(mono, rate):
    data = np.ascontiguousarray(mono, '<i2').tobytes()
    return (b'RIFF' + struct.pack('<I', 36 + len(data)) + b'WAVEfmt ' +
            struct.pack('<IHHIIHH', 16, 1, 1, rate, rate * 2, 2, 16) + b'data' + struct.pack('<I', len(data)) + data)


def ffmpeg_wav(tmp_path, pcm, mask, rate, sample_rate, name='ref.wav'):
    path = tmp_path / name
    path.write_bytes(wav_bytes(ref_swr.convert(pcm, mask, rate, sample_rate), sample_rate))
    return str(path)


def assert_same(got, want):
    assert got.data.shape == want.data.shape
    assert np.array_equal(got.data, want.data)
    assert (got.sample_rate, got.sample_count, got.padding_size) == (want.sample_rate, want.sample_count,
                                                                      want.padding_size)


def flac_file(tmp_path, channels, rate, frames, seed, bits=16):
    plan = fc.stereo_plan(['lpc', 'fixed'], order=8, porder=3) if channels == 2 else \
        fc.uniform_plan(channels, kind='auto', order=8)
    case = fc.make('swr', 'programme', frames, channels, bits, rate, fc.fixed_blocks(frames, 4096), plan, seed)
    path = tmp_path / 'in.flac'
    path.write_bytes(case.flac)
    return str(path), case.pcm.astype(np.int16)


def mkv_file(tmp_path, spec, rate):
    a = mc._timed(spec, 1000.0 / rate)
    blocks = mc._blocks_for(0, a, lambda j: ('none', 1, False, None))
    ts, clusters = mc.arrange([a], 1000, [blocks])
    path = tmp_path / 'in.mka'
    path.write_bytes(mc.build('swr', [a], clusters, ts).data)
    return str(path)


@pytest.mark.parametrize('channels,rate,sample_rate', [(2, 48000, 12000), (6, 48000, 12000), (1, 44100, 12000),
                                                      (2, 8000, 12000), (2, 7919, 12000), (6, 44100, 24000),
                                                      (2, 48000, 48000), (6, 48000, 48000), (1, 48000, 48000)])
def test_flac(tmp_path, channels, rate, sample_rate):
    path, pcm = flac_file(tmp_path, channels, rate, 3 * rate + 123, channels * rate)
    want = WavStream(ffmpeg_wav(tmp_path, pcm, swr.FLAC[channels], rate, sample_rate), sample_rate=sample_rate)
    assert_same(WavStream(path, sample_rate=sample_rate, ffmpeg_audio=True), want)


@pytest.mark.parametrize('sample_type', ['uint8', 'float32'])
def test_both_sample_types(tmp_path, sample_type):
    path, pcm = flac_file(tmp_path, 2, 44100, 44100 * 4, 3)
    want = WavStream(ffmpeg_wav(tmp_path, pcm, 0x3, 44100, 12000), sample_type=sample_type)
    assert_same(WavStream(path, sample_type=sample_type, ffmpeg_audio=True), want)


@pytest.mark.parametrize('channels', [1, 2, 6])
def test_matroska_pcm(tmp_path, channels):
    spec = mc.pcm_track(48000 * 3 + 480, channels, 16, 48000, 480, channels)
    path = mkv_file(tmp_path, spec, 48000)
    want = WavStream(ffmpeg_wav(tmp_path, spec.pcm.astype(np.int16), swr.DEFAULT[channels], 48000, 12000))
    assert_same(WavStream(path, ffmpeg_audio=True), want)


def test_matroska_flac(tmp_path):
    spec = mc.flac_track(4096 * 10 + 77, 2, 16, 44100, 4096, 4)
    path = mkv_file(tmp_path, spec, 44100)
    want = WavStream(ffmpeg_wav(tmp_path, spec.pcm.astype(np.int16), 0x3, 44100, 12000))
    assert_same(WavStream(path, ffmpeg_audio=True), want)


def test_tta(tmp_path):
    case = next(c for c in tc.all_cases() if c.bits == 16 and c.pcm.shape[1] == 2)
    path = tmp_path / 'in.tta'
    path.write_bytes(case.tta())
    want = WavStream(ffmpeg_wav(tmp_path, case.pcm16, 0x3, case.rate, 12000))
    assert_same(WavStream(str(path), ffmpeg_audio=True), want)


def test_wavpack(tmp_path):
    case = next(c for c in wc.all_cases() if c.name == 'mono16')
    path = tmp_path / 'in.wv'
    path.write_bytes(case.wv())
    want = WavStream(ffmpeg_wav(tmp_path, case.pcm16, 0x4, case.rate, 12000))
    assert_same(WavStream(str(path), ffmpeg_audio=True), want)


def test_wav_input_loads_as_before(tmp_path):
    rng = np.random.default_rng(5)
    path = tmp_path / 'in.wav'
    pcm = rng.integers(-32768, 32768, (48000 * 2, 1)).astype(np.int16)
    path.write_bytes(wav_bytes(pcm[:, 0], 48000))
    assert_same(WavStream(str(path), ffmpeg_audio=True), WavStream(str(path)))


def swr_device(pcm, mask, rate, sample_rate):
    """sb_pcm_from_le then sb_pcm_swr; the mono samples read back through sb_pcm_load at their own rate with no
    padding (a mono stream at its own rate loads as its int16 values in float32)"""
    lib = _native.lib()
    buf = np.ascontiguousarray(pcm, '<i2')
    h = _native.decode(None, 'sb_pcm_from_le', buf.ctypes.data_as(ctypes.c_void_p), len(pcm), pcm.shape[1], 2, rate)
    out = ctypes.c_void_p()
    try:
        _native.check(lib.sb_pcm_swr(h, mask, sample_rate, ctypes.byref(out)), 'sb_pcm_swr')
    finally:
        lib.sb_pcm_destroy(h)
    raw = ctypes.c_void_p()
    try:
        frames, channels, r = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
        _native.check(lib.sb_pcm_info(out, ctypes.byref(frames), ctypes.byref(channels), ctypes.byref(r)), 'info')
        assert (channels.value, r.value) == (1, sample_rate)
        _native.check(lib.sb_pcm_load(out, sample_rate, 0, frames.value, ctypes.byref(raw)), 'sb_pcm_load')
        host = np.zeros(frames.value, np.float32)
        _native.check(lib.sb_stream_read(raw, 0, frames.value, host.ctypes.data_as(ctypes.c_void_p)), 'read')
        return host
    finally:
        if raw:
            lib.sb_stream_destroy(raw)
        lib.sb_pcm_destroy(out)


@pytest.mark.parametrize('mask', [0x3, 0x3f], ids=hex)
def test_ninety_minutes(mask):
    channels = bin(mask).count('1')
    frames = 48000 * 5400
    rng = np.random.default_rng(mask)
    pcm = (rng.standard_normal((frames, channels), np.float32) * 6000).clip(-32768, 32767).astype(np.int16)
    want = ref_swr.convert(pcm, mask, 48000, 12000, chunk=1 << 20)
    got = swr_device(pcm, mask, 48000, 12000)
    assert len(got) == len(want)
    assert np.array_equal(got, want.astype(np.float32))


def test_s32_sources_are_refused_before_the_gpu(tmp_path):
    path, _ = flac_file(tmp_path, 2, 48000, 48000, 6, bits=24)
    with pytest.raises(SushiError, match=r'FLAC stream of 24 bits decodes to S32'):
        WavStream(path, ffmpeg_audio=True)
    spec = mc.pcm_track(48000, 2, 24, 48000, 480, 7)
    with pytest.raises(SushiError, match=r'track 0: .*PCM stream of 24 bits decodes to S32'):
        WavStream(mkv_file(tmp_path, spec, 48000), ffmpeg_audio=True)


def test_host_loader_is_refused(tmp_path):
    path, _ = flac_file(tmp_path, 2, 48000, 48000, 8)
    with pytest.raises(SushiError, match="needs loader='gpu'"):
        WavStream(path, ffmpeg_audio=True, loader='host')


def test_command_line(tmp_path):
    """a Matroska FLAC source and a raw FLAC destination 0.125 s later: the script --ffmpeg-audio writes is the one the
    run on the two WAVs the reference's ffmpeg call would write gives"""
    spec = mc.flac_track(4096 * 40, 2, 16, 48000, 4096, 11)
    src = mkv_file(tmp_path, spec, 48000)
    dst_pcm = np.concatenate([np.zeros((6000, 2), np.int64), spec.pcm])[:len(spec.pcm)]
    plan = fc.stereo_plan(['lpc', 'fixed'], order=8, porder=3)
    flac, _, _ = fc.encode(dst_pcm, 48000, 16, fc.fixed_blocks(len(dst_pcm), 4096), plan, np.random.default_rng(13))
    dst = tmp_path / 'b.flac'
    dst.write_bytes(flac)
    script = tmp_path / 's.srt'
    script.write_text('1\n00:00:00,500 --> 00:00:01,500\nOne\n\n2\n00:00:01,800 --> 00:00:02,700\nTwo\n\n')
    a = ffmpeg_wav(tmp_path, spec.pcm.astype(np.int16), 0x3, 48000, 12000, 'a.wav')
    b = ffmpeg_wav(tmp_path, dst_pcm.astype(np.int16), 0x3, 48000, 12000, 'b.wav')

    def run(src, dst, out, *extra):
        subprocess.check_call([sys.executable, '-m', 'sushi_b200', '--src', src, '--dst', dst, '--script',
                               str(script), '-o', str(tmp_path / out)] + list(extra), cwd=ROOT)
        return (tmp_path / out).read_text()
    shifted = run(src, str(dst), 'x.srt', '--ffmpeg-audio')
    assert shifted == run(a, b, 'y.srt')
    assert '00:00:00,625' in shifted
