"""WavStream(path, ffmpeg_audio=True) on the GPU: an input that is not a WAV file loads bit for bit as WavStream loads
the mono pcm_s16le WAV the reference's ffmpeg call writes for it, that WAV made here by libswresample itself
(tests/ref_swr.py, FMA3 path) from the writer's PCM.  Raw FLAC, Matroska FLAC and 16-bit little-endian PCM, raw
TTA and WavPack; stereo, 5.1 and mono; downsampling, upsampling, an inexact ratio and equal rates (the integer path);
90 minutes of stereo and of 5.1 through sb_pcm_swr; the refusals; and the command line with --ffmpeg-audio against the
run on the two WAVs.  Then against an oracle that owes nothing to this project's decoders or layout tables: FFmpeg
decodes the file and reports its channel layout, and libswresample converts that.  The 16-bit audio tracks of the MP4
and QuickTime cases (ALAC mono, stereo and 8 channels; twos, sowt, 3-channel lpcm and ipcm PCM; FLAC), Matroska ALAC
and TTA, raw FLAC of 3, 4, 5, 7 and 8 channels, raw TTA of 6 and 8 channels, and FLAC inputs around the filter length;
and the refusals of Matroska WavPack, BD-LPCM, WavPack of more than two channels and big-endian Matroska PCM."""
import ctypes
import functools
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, WavStream, _native, inputs, swr
from tests import flac_cases as fc
from tests import mkv_alac_cases, mkv_tta_cases, mkv_wavpack_cases, mp4_cases, ts_cases
from tests import mkv_cases as mc
from tests import ref_mp4, ref_swr
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


def flac_file(tmp_path, channels, rate, frames, seed, bits=16, **kw):
    plan = fc.stereo_plan(['lpc', 'fixed'], order=8, porder=3) if channels == 2 else \
        fc.uniform_plan(channels, kind='auto', order=8)
    case = fc.make('swr', 'programme', frames, channels, bits, rate, fc.fixed_blocks(frames, 4096), plan, seed, **kw)
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


def swr_handle(pcm, mask, rate, sample_rate, big=False):
    """sb_pcm_from_le (big: sb_pcm_from_be) then sb_pcm_swr -> (the mono output handle, which the caller destroys, and
    its frame count from sb_pcm_info)"""
    lib = _native.lib()
    buf = np.ascontiguousarray(pcm, '>i2' if big else '<i2')
    h = _native.decode(None, 'sb_pcm_from_be' if big else 'sb_pcm_from_le', buf.ctypes.data_as(ctypes.c_void_p),
                       len(pcm), pcm.shape[1], 2, rate)
    out = ctypes.c_void_p()
    try:
        _native.check(lib.sb_pcm_swr(h, mask, sample_rate, ctypes.byref(out)), 'sb_pcm_swr')
    finally:
        lib.sb_pcm_destroy(h)
    try:
        frames, channels, r = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
        _native.check(lib.sb_pcm_info(out, ctypes.byref(frames), ctypes.byref(channels), ctypes.byref(r)), 'info')
        assert (channels.value, r.value) == (1, sample_rate)
    except BaseException:
        lib.sb_pcm_destroy(out)
        raise
    return out, frames.value


def swr_device(pcm, mask, rate, sample_rate, big=False):
    """swr_handle's mono samples read back through sb_pcm_load at their own rate with no padding (a mono stream at its
    own rate loads as its int16 values in float32)"""
    lib = _native.lib()
    out, frames = swr_handle(pcm, mask, rate, sample_rate, big)
    raw = ctypes.c_void_p()
    try:
        _native.check(lib.sb_pcm_load(out, sample_rate, 0, frames, ctypes.byref(raw)), 'sb_pcm_load')
        host = np.zeros(frames, np.float32)
        _native.check(lib.sb_stream_read(raw, 0, frames, host.ctypes.data_as(ctypes.c_void_p)), 'read')
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


# ---- against FFmpeg's own decode ------------------------------------------------------------------------------------
# The oracle below owes nothing to this project's decoders or layout tables: libavformat and libavcodec decode the
# stream (tests/ref_mp4.decode_s16), the decoder reports its channel layout and rate, and libswresample converts that.

def ffmpeg_decoded(tmp_path, path, sid=0, sample_rate=12000):
    pcm, mask, rate = ref_mp4.decode_s16(path, sid)
    return WavStream(ffmpeg_wav(tmp_path, pcm, mask, rate, sample_rate), sample_rate=sample_rate)


def write(tmp_path, name, data):
    path = tmp_path / name
    path.write_bytes(data)
    return str(path)


# the 16-bit audio tracks of mp4_cases.good_cases(): (case, stream id, FFmpeg's codec)
MP4_TRACKS = [('m4a_alac', 0, 'alac'), ('mov_alac_last', 0, 'alac'), ('mp4_aac', 1, 'alac'),
              ('mov_master', 1, 'pcm_s16be'), ('mov_master', 2, 'pcm_s16le'), ('mov_lpcm', 1, 'pcm_s16le'),
              ('mp4_ipcm', 0, 'pcm_s16be'), ('mp4_flac', 0, 'flac')]


@functools.lru_cache(maxsize=None)
def mp4_by_name():
    return {c.name: c for c in mp4_cases.good_cases()}


@functools.lru_cache(maxsize=None)
def matroska_by_name():
    """the 16-bit A_ALAC cases and the decoded 16-bit A_TTA1 cases"""
    out = {m.name: m for m, c in mkv_alac_cases.cases() if c.bits == 16}
    out.update((m.name, m) for m, c, how in mkv_tta_cases.cases() if how == 'decoded' and c.bits == 16)
    return out


def test_every_16_bit_mp4_track_is_listed():
    got = sorted((c.name, sid, t.codec) for c in mp4_by_name().values() for sid, t in enumerate(c.traks)
                 if t.kind == 'audio' and t.bits == 16 and t.codec != 'aac')
    assert got == sorted(MP4_TRACKS)


@pytest.mark.parametrize('name,sid,codec', MP4_TRACKS, ids=lambda v: str(v))
def test_mp4_against_ffmpeg(tmp_path, name, sid, codec):
    """ALAC (stereo, mono, 8 channels in layout 0xff), twos / sowt / lpcm (3 channels) / ipcm PCM, FLAC"""
    case = mp4_by_name()[name]
    path = case.write(tmp_path)
    assert ref_mp4.demux(path, packets=False).streams[sid][1] == codec
    if codec.startswith('pcm'):                          # twos and ipcm take sb_pcm_from_be, sowt and lpcm the LE path
        reader, _ = inputs.open_input(path)
        try:
            assert reader.select_audio(sid).pcm()[5] == codec.endswith('be')
        finally:
            reader.close()
    assert_same(WavStream(path, track=sid, ffmpeg_audio=True), ffmpeg_decoded(tmp_path, path, sid))


@pytest.mark.parametrize('name', ['mka_' + n for n in ('mono16', 'stereo16', 'stereo16_pt15', 'full16', 'orders',
                                                     'silence16', 'layout3', 'layout4', 'layout5', 'layout6',
                                                     'layout7', 'layout8', 'apple')] +
                         ['mka_tta_' + n for n in ('laced', 'six16', 'rate192000')])
def test_matroska_against_ffmpeg(tmp_path, name):
    path = write(tmp_path, name + '.mka', matroska_by_name()[name].data)
    assert_same(WavStream(path, ffmpeg_audio=True), ffmpeg_decoded(tmp_path, path))


def test_matroska_cases_are_listed():
    assert len(matroska_by_name()) == 16


def test_matroska_big_endian_pcm_is_refused(tmp_path):
    """A_PCM/INT/BIG is not read from Matroska, with or without --ffmpeg-audio (big-endian PCM reaches sb_pcm_from_be
    through the MP4 twos and ipcm tracks above)"""
    spec = mc.pcm_track(44100, 2, 16, 44100, 441, 20, codec='A_PCM/INT/BIG')
    path = mkv_file(tmp_path, spec, 44100)
    with pytest.raises(SushiError, match='Audio track 0 is A_PCM/INT/BIG at 16 bits, which cannot be decoded here'):
        WavStream(path, ffmpeg_audio=True)


@pytest.mark.parametrize('channels', [3, 4, 5, 7, 8])
def test_flac_channels_against_ffmpeg(tmp_path, channels):
    path, _ = flac_file(tmp_path, channels, 44100, 44100 + 999, 30 + channels)
    assert_same(WavStream(path, ffmpeg_audio=True), ffmpeg_decoded(tmp_path, path))


@pytest.mark.parametrize('name', ['six16', 'eight16_extreme'])
def test_tta_channels_against_ffmpeg(tmp_path, name):
    case = next(c for c in tc.all_cases() if c.name == name)
    path = write(tmp_path, name + '.tta', case.tta())
    assert_same(WavStream(path, ffmpeg_audio=True), ffmpeg_decoded(tmp_path, path))


def load_outcome(load):
    try:
        return load()
    except SushiError as e:
        return str(e)


# L = 132 taps at 48000 -> 12000: 1 and 66 frames give no output at all, 132 and 133 give 33 frames.  STREAMINFO
# gives the encoder's block size of 4096, as an encoder writes it for a stream shorter than one block (FFmpeg refuses
# a FLAC stream whose largest block is under 16 samples).
@pytest.mark.parametrize('frames', [1, 66, 132, 133])
def test_short_flac_against_ffmpeg(tmp_path, frames):
    path, _ = flac_file(tmp_path, 2, 48000, frames, 40 + frames, min_block=4096, max_block=4096)
    got = load_outcome(lambda: WavStream(path, ffmpeg_audio=True))
    want = load_outcome(lambda: ffmpeg_decoded(tmp_path, path))
    assert not isinstance(got, str) and not isinstance(want, str), (got, want)
    assert_same(got, want)
    assert want.sample_count == (0 if frames < 132 else 33)


def test_matroska_wavpack_is_refused(tmp_path):
    mkv, _ = mkv_wavpack_cases.cases()[0]
    path = write(tmp_path, 'in.mka', mkv.data)
    with pytest.raises(SushiError, match='cannot tell which sample format FFmpeg decodes this WavPack stream'):
        WavStream(path, ffmpeg_audio=True)


def test_bd_lpcm_is_refused(tmp_path):
    case = next(c for c in ts_cases.all_cases() if c.name == 'bd_stereo16_48k')
    with pytest.raises(SushiError, match='cannot tell which sample format FFmpeg decodes this .*LPCM.* stream'):
        WavStream(case.write(tmp_path), ffmpeg_audio=True)


def test_wavpack_of_more_than_two_channels_is_refused(tmp_path):
    """refused after the GPU decode, once the channel count is known"""
    case = next(c for c in wc.all_cases() if c.name == 'six16')
    path = write(tmp_path, 'in.wv', case.wv())
    with pytest.raises(SushiError, match="does not know FFmpeg's channel layout of this 6-channel WavPack stream"):
        WavStream(path, ffmpeg_audio=True)
