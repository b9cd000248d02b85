"""Every GPU decoder's output, every frame of it: the sb_pcm handle a file decodes to (through the product's own reader,
inputs.open_input -> select_audio -> decode, or sb_pcm_from_be / sb_pcm_from_le for container PCM) is loaded at its own
rate with no padding (sb_pcm_load), which skips the resample, and read back with sb_stream_read.  Each read-back sample
is then the reference loader's readframes of one frame of the decoded int16 PCM -- the float32 mean of its channels,
from which the integer channel sum is recovered exactly for 1 to 8 channels -- and is compared bit for bit with
readframes of FFmpeg's decode (the int16 PCM each format's GPU test builds its WAV from; sources wider than 16 bits by
their top 16 bits).

Loading at 12 kHz reads only every 4th frame of a 48 kHz stream (every 16th at 192 kHz) and quantises to uint8; here no
frame and no bit is hidden.  The cases are every decodable good case of every format, and sizes that reach the
structures only the GPU has: the MP2 output-rounding carry across 1024-tile passes of k_mp2_tiles, ALAC's launches of
2^25 / frameLength frames, the 90-minute stream of every decoder, and demuxer chunks whose per-CTA totals take
k_scan_totals past one 1024-entry pass."""
import ctypes
import functools

import numpy as np
import pytest

from oracle import ref_loader
from sushi_b200 import _native, inputs, mpegps, mpegts, ogg
from tests import alac_cases as ac
from tests import flac_cases as fc
from tests import mkv_alac_cases as mac
from tests import mkv_cases as mkc
from tests import mkv_truehd_cases as mthd
from tests import mkv_tta_cases as mtta
from tests import mkv_wavpack_cases as mwc
from tests import mp2_cases as mp2c
from tests import mp4_cases as m4c
from tests import mpa_cases
from tests import ogg_cases as oc
from tests import ps_cases as pc
from tests import ref_mp2, ref_mp4
from tests import truehd_cases as thc
from tests import ts_cases as tsc
from tests import tta_cases as ttc
from tests import wavpack_cases as wc

SLICE = 1 << 24                     # samples per sb_stream_read


class Periodic(object):
    """The int16 PCM (frames, channels) of `reps` repetitions of `period`, then `tail`, cut to `frames` frames: rows
    are built per slice, so a 90-minute expectation never exists whole in host memory."""

    def __init__(self, period, reps, tail=None, frames=None):
        self.period = np.ascontiguousarray(period, np.int16)
        self.tail = np.zeros((0, self.period.shape[1]), np.int16) if tail is None else np.asarray(tail, np.int16)
        self.body = len(self.period) * reps
        self.n = self.body + len(self.tail) if frames is None else frames
        self.shape = (self.n, self.period.shape[1])

    def __len__(self):
        return self.n

    def __getitem__(self, s):
        k = np.arange(s.start, min(s.stop, self.n))
        inside = k < self.body
        out = np.empty((len(k), self.shape[1]), np.int16)
        out[inside] = self.period[k[inside] % len(self.period)]
        out[~inside] = self.tail[k[~inside] - self.body]
        return out


def decoded_handle(source, track=None):
    """The sb_pcm handle of `source`'s audio as the product makes it: a codec's decode(device) (then its check of the
    frame count), or container PCM uploaded by sb_pcm_from_be / sb_pcm_from_le.  The caller destroys it."""
    reader, _ = inputs.open_input(source)
    try:
        audio = reader.select_audio(track)
        if audio.label is None:
            data, frames, channels, width, rate, big = audio.pcm()
            buf = np.frombuffer(data, dtype=np.uint8)
            return _native.decode(None, 'sb_pcm_from_be' if big else 'sb_pcm_from_le',
                                  buf.ctypes.data_as(ctypes.c_void_p), frames, channels, width, rate), None
        return audio.decode(None), audio.check
    finally:
        if reader is not source and hasattr(reader, 'close'):
            reader.close()


def where(f, frame_len):
    """frame f inside the decoder's unit: frame_len is its length, or the sorted start frames of variable units"""
    if frame_len is None:
        return 'frame %d' % f
    if np.ndim(frame_len) == 0:
        return 'frame %d (sample %d of unit %d of %d)' % (f, f % frame_len, f // frame_len, frame_len)
    u = int(np.searchsorted(frame_len, f, 'right')) - 1
    return 'frame %d (sample %d of unit %d)' % (f, f - int(frame_len[u]), u)


def assert_decodes_to(source, want, rate, frame_len, track=None):
    """The handle `source` decodes to holds `want` ((frames, channels) int16, or a Periodic) at `rate`: its shape by
    sb_pcm_info, every frame by sb_pcm_load at its own rate read back bit for bit against readframes of `want`."""
    lib = _native.lib()
    h, check = decoded_handle(source, track)
    raw = ctypes.c_void_p()
    try:
        frames, channels, r = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
        _native.check(lib.sb_pcm_info(h, ctypes.byref(frames), ctypes.byref(channels), ctypes.byref(r)), 'sb_pcm_info')
        if check is not None:
            check(frames.value)
        n, ch = frames.value, channels.value
        assert (n, ch, r.value) == (len(want), want.shape[1], rate)
        assert 1 <= ch <= 8
        if n == 0:
            return
        _native.check(lib.sb_pcm_load(h, rate, 0, n, ctypes.byref(raw)), 'sb_pcm_load')
        first, bad, worst = None, 0, 0
        for a in range(0, n, SLICE):
            b = min(n, a + SLICE)
            got = np.empty(b - a, np.float32)
            _native.check(lib.sb_stream_read(raw, a, b - a, got.ctypes.data_as(ctypes.c_void_p)), 'sb_stream_read')
            exp = ref_loader.readframes(np.ascontiguousarray(want[a:b], '<i2').tobytes(), 2, ch)
            diff = np.flatnonzero(got.view(np.uint32) != exp.view(np.uint32))
            if len(diff):
                first = a + int(diff[0]) if first is None else first
                bad += len(diff)
                lsb = np.abs(np.rint(got[diff].astype(np.float64) * ch) - np.rint(exp[diff].astype(np.float64) * ch))
                worst = max(worst, int(np.nan_to_num(lsb, nan=2 ** 31).max()))
        assert bad == 0, '%d of %d frames differ; the first at %s; the largest by %d LSB of the channel sum' % (
            bad, n, where(first, frame_len), worst)
    finally:
        if raw:
            lib.sb_stream_destroy(raw)
        lib.sb_pcm_destroy(h)


def write(tmp_path, name, data):
    path = tmp_path / name
    path.write_bytes(data)
    return str(path)


def flac_starts(case):
    return np.cumsum([0] + [f['block_size'] for f in case.frames])[:-1]


def ffmpeg_s16(path, sid):
    pcm, _, rate = ref_mp4.decode_s16(path, sid)
    return pcm, rate


# ---- the CPU contract the read-back rests on -----------------------------------------------------------------------

@pytest.mark.parametrize('channels', [1, 2, 6, 8])
@pytest.mark.parametrize('rate', [7919, 44100, 192000])
@pytest.mark.parametrize('seconds', [None, 2.37])
def test_own_rate_load_is_readframes(channels, rate, seconds):
    """At sample_rate == framerate the reference loader's content region is readframes of the whole PCM (one frame,
    and a partial last second), and the integer channel sum is recovered exactly from it"""
    rng = np.random.default_rng([channels, rate])
    frames = 1 if seconds is None else int(seconds * rate)
    pcm = rng.integers(-32768, 32768, (frames, channels)).astype(np.int16)
    pcm[:min(frames, 3)] = [[-32768] * channels, [32767] * channels, [-32768, 32767] * (channels // 2) +
                            [1] * (channels % 2)][:min(frames, 3)]
    raw = pcm.astype('<i2').tobytes()
    at = [0]

    def read(n):
        out = raw[at[0]:at[0] + n * channels * 2]
        at[0] += n * channels * 2
        return out
    data, count, padding = ref_loader.pad_stream(read, frames, rate, 2, channels, sample_rate=rate)
    assert (count, padding) == (frames, 10 * rate)
    whole = ref_loader.readframes(raw, 2, channels)
    assert np.array_equal(data[0, padding:padding + frames].view(np.uint32), whole.view(np.uint32))
    assert np.array_equal(np.rint(whole.astype(np.float64) * channels).astype(np.int64), pcm.astype(np.int64).sum(1))


# ---- every good case of every format --------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', fc.all_cases(), ids=lambda c: c.name)
def test_flac(gpu_lib, tmp_path, case):
    assert_decodes_to(case.write(tmp_path), case.pcm16(), case.rate, flac_starts(case))


MKV_TRACKS = [(c, sid) for c in mkc.all_cases() if c.damage is None and c.refused is None for sid in c.audio_ids()]


@pytest.mark.gpu
@pytest.mark.parametrize('case,sid', MKV_TRACKS, ids=lambda x: x.name if hasattr(x, 'name') else str(x))
def test_matroska_flac_and_pcm(gpu_lib, tmp_path, case, sid):
    s = case.specs[sid]
    assert_decodes_to(case.write(tmp_path), (s.pcm >> (s.pcm_bits - 16)).astype(np.int16), s.rate, None, track=sid)


@pytest.mark.gpu
@pytest.mark.parametrize('case', thc.all_cases(), ids=lambda c: c.name)
def test_truehd(gpu_lib, tmp_path, case):
    assert_decodes_to(case.write(tmp_path), case.pcm16, case.rate, case.spa)


@pytest.mark.gpu
@pytest.mark.parametrize('pair', mthd.cases(), ids=lambda p: p[0].name)
def test_matroska_truehd(gpu_lib, tmp_path, pair):
    mkv, case = pair
    assert_decodes_to(mkv.write(tmp_path), case.pcm16, case.rate, case.spa)


TS_STREAMS = [(c, s) for c in tsc.all_cases() if c.hdmv and not c.refused and c.name != 'bd_stereo20_48k'
              for s in c.audio()]


@pytest.mark.gpu
@pytest.mark.parametrize('packets', [None, 7, 61])
@pytest.mark.parametrize('pair', TS_STREAMS, ids=lambda p: '%s-%x' % (p[0].name, p[1].pid))
def test_transport_stream(gpu_lib, tmp_path, monkeypatch, pair, packets):
    """BD-LPCM 16/24-bit and TrueHD, at the default chunk and at chunks that split PES packets"""
    case, s = pair
    path = case.write(tmp_path)
    sid = next(t.id for t in mpegts.TransportStream(path).streams_all
               if t.pid == s.pid and t.codec == ('truehd' if s.kind == 'truehd' else 'pcm_bluray'))
    if packets:
        monkeypatch.setattr(mpegts, 'CHUNK_BYTES', packets * case.psize)
    unit = s.rate // 1200 if s.kind == 'truehd' else s.rate // 200
    assert_decodes_to(path, s.pcm, s.rate, unit, track=sid)


def alac_m4a(tmp_path, case, per_chunk=(3, 3, 2)):
    return write(tmp_path, case.name + '.m4a', m4c.build(case.name, [m4c.alac_trak(case, per_chunk=per_chunk,
                                                                                    edits=None)], ftyp=b'M4A '))


@pytest.mark.gpu
@pytest.mark.parametrize('case', ac.all_cases(), ids=lambda c: c.name)
def test_alac_in_mp4(gpu_lib, tmp_path, case):
    assert_decodes_to(alac_m4a(tmp_path, case), case.pcm16, case.rate, case.cfg.frame_length)


@pytest.mark.gpu
@pytest.mark.parametrize('pair', mac.cases(), ids=lambda p: p[0].name)
def test_alac_in_matroska(gpu_lib, tmp_path, pair):
    mkv, case = pair
    assert_decodes_to(mkv.write(tmp_path), case.pcm16, case.rate, case.cfg.frame_length)


MP4_TRACKS = [(c, sid) for c in m4c.good_cases() for sid in c.audio_ids()]


@pytest.mark.gpu
@pytest.mark.parametrize('pair', MP4_TRACKS, ids=lambda p: '%s-%d' % (p[0].name, p[1]))
def test_mp4_track(gpu_lib, tmp_path, pair):
    """the ALAC, FLAC and PCM tracks of mp4_cases, big-endian twos / in24 by sb_pcm_from_be"""
    case, sid = pair
    t = case.traks[sid]
    assert_decodes_to(case.write(tmp_path), ac.to16(t.pcm, t.bits), t.rate, None, track=sid)


@pytest.mark.gpu
@pytest.mark.parametrize('case', wc.all_cases(), ids=lambda c: c.name)
def test_wavpack(gpu_lib, tmp_path, case):
    path = write(tmp_path, case.name + '.wv', case.wv())
    assert_decodes_to(path, case.pcm16, case.rate, np.cumsum((0,) + tuple(case.counts))[:-1])


@pytest.mark.gpu
@pytest.mark.parametrize('pair', mwc.cases(), ids=lambda p: p[0].name)
def test_matroska_wavpack(gpu_lib, tmp_path, pair):
    mkv, case = pair
    assert_decodes_to(mkv.write(tmp_path), case.pcm16[:mwc.kept_samples(mkv, case)], case.rate,
                      np.cumsum((0,) + tuple(case.counts))[:-1])


@pytest.mark.gpu
@pytest.mark.parametrize('case', ttc.all_cases(), ids=lambda c: c.name)
def test_tta(gpu_lib, tmp_path, case):
    path = write(tmp_path, case.name + '.tta', case.tta())
    assert_decodes_to(path, case.pcm16, case.rate, case.frame_length)


@pytest.mark.gpu
@pytest.mark.parametrize('triple', [t for t in mtta.cases() if t[2] != 'refused'], ids=lambda t: t[0].name)
def test_matroska_tta(gpu_lib, tmp_path, triple):
    mkv, case, _ = triple
    assert_decodes_to(mkv.write(tmp_path), case.pcm16, case.rate, case.frame_length)


MP2_CASES = mp2c.all_cases()


@pytest.mark.gpu
@pytest.mark.parametrize('packets', [None, 1, 7, 61])
@pytest.mark.parametrize('pair', mp2c.ts_files(MP2_CASES), ids=lambda p: p[0].name)
def test_mp2_in_transport_stream(gpu_lib, tmp_path, monkeypatch, pair, packets):
    """at the default chunk and at chunks of 1, 7 and 61 packets, which split PES packets"""
    path = pair[0].write(tmp_path)
    pcm, rate = ffmpeg_s16(path, 0)
    if packets:
        monkeypatch.setattr(mpegts, 'CHUNK_BYTES', packets * 188)
    assert_decodes_to(path, pcm, rate, 1152)


@pytest.mark.gpu
@pytest.mark.parametrize('pair', mp2c.mkv_files(MP2_CASES), ids=lambda p: p[0].name)
def test_mp2_in_matroska(gpu_lib, tmp_path, pair):
    path = pair[0].write(tmp_path)
    pcm, rate = ffmpeg_s16(path, 0)
    assert_decodes_to(path, pcm, rate, 1152)


@pytest.mark.gpu
@pytest.mark.parametrize('case', mpa_cases.all_cases(), ids=lambda c: c[0])
def test_raw_mp2(gpu_lib, tmp_path, case):
    path = write(tmp_path, case[0] + '.mp2', case[1])
    pcm, rate = ffmpeg_s16(path, 0)
    assert_decodes_to(path, pcm, rate, 1152)


PS_STREAMS = [(c, 0x100 | e.sid) for c in pc.good_cases() for e in c.audio()]


@pytest.mark.gpu
@pytest.mark.parametrize('chunk', [None, 17, 777])
@pytest.mark.parametrize('pair', PS_STREAMS, ids=lambda p: '%s_%x' % (p[0].name, p[1]))
def test_mp2_in_program_stream(gpu_lib, tmp_path, monkeypatch, pair, chunk):
    case, stream_id = pair
    path = case.write(tmp_path)
    sid = next(s.id for s in mpegps.ProgramStream(path).streams_all if s.stream_id == stream_id)
    pcm, rate = ffmpeg_s16(path, sid)
    if chunk:
        monkeypatch.setattr(mpegps, 'CHUNK_BYTES', chunk)
    assert_decodes_to(path, pcm, rate, 1152, track=sid)


OGG_STREAMS = [(c, k) for c in oc.good_cases() for k in range(len(c.streams))]


@pytest.mark.gpu
@pytest.mark.parametrize('chunk', [None, 28, 777])
@pytest.mark.parametrize('pair', OGG_STREAMS, ids=lambda p: '%s_%d' % (p[0].name, p[1]))
def test_ogg_flac(gpu_lib, tmp_path, monkeypatch, pair, chunk):
    case, k = pair
    path = case.write(tmp_path)
    if chunk:
        monkeypatch.setattr(ogg, 'CHUNK_BYTES', chunk)
    flac = case.streams[k].case
    assert_decodes_to(path, flac.pcm16(), flac.rate, flac_starts(flac), track=k)


# ---- sizes that reach the GPU-only structures -----------------------------------------------------------------------

# (frames, channels): 1024 and 1025 (frame, channel) tiles, one pass of k_mp2_tiles and one tile into the second; about
# 1100 mono and 600 stereo frames
MP2_TILES = [(1024, 1), (1025, 1), (512, 2), (513, 2), (1100, 1), (600, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize('lsf', [0, 1], ids=['mpeg1_48000', 'lsf_24000'])
@pytest.mark.parametrize('frames,channels', MP2_TILES, ids=lambda v: str(v))
def test_mp2_tile_scan(gpu_lib, tmp_path, frames, channels, lsf):
    """the output-rounding remainder carried across the 1024-tile passes of k_mp2_tiles"""
    base = mp2c.stream('tiles', 500 + 10 * lsf + channels, 37, lsf=lsf, rate_index=1, bitrate_index=8 if lsf else 10,
                       mode=3 if channels == 1 else [0, 1, 2], mode_ext=[0, 3])
    seq = [base.frames[k % len(base.frames)] for k in range(frames)]
    # in Matroska, one frame per block: every frame reaches the decoder (a raw file's first frames go to the probe)
    path = mp2c.mkv_file('tiles', mp2c.Case('tiles', seq, base.specs[:1])).write(tmp_path)
    pcm, _, rate, refused = ref_mp2.decode_packets(seq)
    assert refused == 0 and pcm.shape == (frames * 1152, channels)
    assert_decodes_to(path, pcm, rate, 1152)


@pytest.mark.gpu
def test_mp2_ninety_minutes(gpu_lib, tmp_path):
    """about 562 000 tiles, as test_gpu_mp2 builds them: one Matroska block per 100 frames"""
    frames, _ = mp2c.long_stream(90.0)
    pcm = ref_mp2.decode_packets(frames)[0]
    sizes = [len(f) for f in frames]
    pieces = [sum(sizes[k:k + 100]) for k in range(0, len(sizes), 100)]
    path = mp2c.mkv_file('long', mp2c.Case('long', frames, [mp2c.FrameSpec(mode=0, rate=48000)]),
                         pieces).write(tmp_path)
    del frames
    assert_decodes_to(path, pcm, 48000, 1152)


ALAC_LAUNCH_LENGTH = 32768
ALAC_PER_LAUNCH = 2 ** 25 // ALAC_LAUNCH_LENGTH         # kScratchBytes / (8 * frameLength) frames per launch


@functools.lru_cache(maxsize=None)
def alac_launch_period():
    return ac.long_stream(bits=16, minutes=1, frame_length=ALAC_LAUNCH_LENGTH, seed=11, n_unique=3)[:3]


@pytest.mark.gpu
@pytest.mark.parametrize('n', [ALAC_PER_LAUNCH, ALAC_PER_LAUNCH + 1, 2 * ALAC_PER_LAUNCH + 77])
def test_alac_launches(gpu_lib, tmp_path, n):
    """a stream of one launch's worth of frames, one more, and more than two launches"""
    cfg, period, pcm = alac_launch_period()
    frames = [period[k % len(period)] for k in range(n)]
    case = ac.AlacCase('launches', cfg, frames, pcm[:1], set())          # pcm: a stand-in, not what it decodes to
    path = alac_m4a(tmp_path, case, per_chunk=(64,))
    want = Periodic(ac.to16(pcm, 16), -(-n // len(period)), frames=n * ALAC_LAUNCH_LENGTH)
    assert_decodes_to(path, want, 48000, ALAC_LAUNCH_LENGTH)


@pytest.mark.gpu
def test_alac_ninety_minutes(gpu_lib, tmp_path):
    cfg, frames, pcm, reps = ac.long_stream()
    case = ac.AlacCase('long', cfg, frames * reps, pcm, set())
    path = str(tmp_path / 'long.m4a')
    with open(path, 'wb') as f:
        f.write(m4c.build('long', [m4c.alac_trak(case, per_chunk=(64,), edits=None)], ftyp=b'M4A '))
    del case.data
    assert_decodes_to(path, Periodic(case.pcm16, reps), 48000, cfg.frame_length)


@pytest.mark.gpu
def test_flac_baseline(gpu_lib, tmp_path):
    """90 minutes, 225 001 frames: bit positions past 2^32"""
    data, pcm = fc.baseline_file()
    path = write(tmp_path, 'baseline.flac', data)
    del data
    assert_decodes_to(path, pcm, fc.BASELINE_RATE, fc.BASELINE_BLOCK)


@pytest.mark.gpu
def test_truehd_ninety_minutes_71(gpu_lib, tmp_path):
    seg, pcm, reps = thc.long_stream()
    path = str(tmp_path / 'long.thd')
    with open(path, 'wb') as f:
        for _ in range(reps):
            f.write(seg)
    assert_decodes_to(path, Periodic(pcm, reps), 48000, 40)


@pytest.mark.gpu
def test_wavpack_ninety_minutes(gpu_lib, tmp_path):
    case, data, reps = wc.long_stream(bits=24, minutes=90)
    path = write(tmp_path, 'long.wv', data)
    del data
    assert_decodes_to(path, Periodic(case.pcm16, reps), 48000, case.counts[0])


@pytest.mark.gpu
def test_tta_ninety_minutes(gpu_lib, tmp_path):
    case, data, reps = ttc.long_stream(bits=24, minutes=90)
    path = write(tmp_path, 'long.tta', data)
    del data
    fl = case.frame_length
    assert_decodes_to(path, Periodic(case.pcm16[:fl], reps, case.pcm16[fl:]), 48000, fl)


@pytest.mark.gpu
def test_bd_lpcm_ninety_minutes(gpu_lib, tmp_path):
    path = str(tmp_path / 'long.m2ts')
    pcm, reps = tsc.long_m2ts(path)
    assert_decodes_to(path, Periodic(pcm, reps), 48000, 240)


# Demuxer chunks whose per-CTA totals need a second 1024-entry pass of k_scan_totals, all in one default chunk:
# transport stream: 256 packets per CTA, so more than 262 144 packets; program stream and Ogg: 16 bytes per thread,
# 256 threads per CTA, so more than 4 MB; Ogg again: one thread per page candidate, so more than 262 144 pages.

@pytest.mark.gpu
def test_transport_stream_chunk_of_more_than_1024_ctas(gpu_lib, tmp_path):
    path = str(tmp_path / 'three_minutes.m2ts')
    pcm, reps = tsc.long_m2ts(path, minutes=3.0)
    size = (tmp_path / 'three_minutes.m2ts').stat().st_size
    assert 1024 * 256 < size // 192 and size <= mpegts.CHUNK_BYTES // 192 * 192     # whole packets per chunk
    assert_decodes_to(path, Periodic(pcm, reps), 48000, 240)


def padded_program_stream(data, seed, pads=40):
    """An MPEG-2 program stream of the MP2 stream `data`: packs of one audio PES of 500 to 1500 payload bytes, each
    followed by `pads` empty padding packets (6 bytes each), so start codes -- the candidates k_ps_link, k_ps_pes and
    k_ps_place run a thread for -- are dense all through the stream.  Returns (file bytes, candidate count)."""
    rng = np.random.default_rng([seed])
    out = bytearray(pc.pack_header(0, True) + pc.system_header([pc.AUDIO]))
    at = k = 0
    while at < len(data):
        n = int(rng.integers(500, 1501))
        if k:
            out += pc.pack_header(1800 * k, True)
        out += pc.pes2(pc.AUDIO, data[at:at + n], 90000 + 3600 * k) + pc.padding(0) * pads
        at += n
        k += 1
    out += b'\x00\x00\x01\xb9'
    return bytes(out), k * (2 + pads) + 2


@pytest.mark.gpu
def test_program_stream_chunk_of_more_than_1024_ctas(gpu_lib, tmp_path):
    """5 minutes of MP2 (about 9 MB) with more than 262 144 start codes: more than 1024 CTAs of bytes and of
    candidates in one chunk, the audio's PES spread across all of them"""
    frames, data = mp2c.long_stream(5.0, distinct=40, seed=12)
    ps, candidates = padded_program_stream(data, 22)
    assert 1024 * 256 < candidates and 1024 * 256 * 16 < len(ps) <= mpegps.CHUNK_BYTES
    path = write(tmp_path, 'big.mpg', ps)
    sid = next(s.id for s in mpegps.ProgramStream(path).streams_all if s.kind == 'audio')
    pcm, rate = ffmpeg_s16(path, sid)
    assert np.array_equal(pcm, ref_mp2.decode_packets(frames)[0])
    assert_decodes_to(path, pcm, rate, 1152, track=sid)


@pytest.mark.gpu
def test_ogg_chunk_of_more_than_1024_ctas(gpu_lib, tmp_path):
    """a 5 MB stream whose header packets are followed by 300 000 pages without segments: more than 1024 CTAs of
    bytes and of page candidates in one chunk"""
    rng = np.random.default_rng([oc.SEED, 70])
    frames = 48000 * 20
    pcm = fc.make_pcm('programme', frames, 2, 16, 48000, rng)
    flac, infos, offsets = fc.encode(pcm, 48000, 16, fc.fixed_blocks(frames, 4096),
                                     fc.uniform_plan(2, kind='fixed', order=2), rng)
    flac_case = fc.FlacCase('big', flac, pcm, 48000, 16, infos, offsets, 12000, 'uint8')
    case = oc.make('big', [(0x70, flac_case, [], None, 17, lambda i, rng: 300000 if i == 1 else 0)], 70)
    assert sum(1 for i in case.pages if not i['segs']) == 300000
    assert 1024 * 256 < len(case.pages) and 1024 * 256 * 16 < len(case.data) <= ogg.CHUNK_BYTES
    assert_decodes_to(case.write(tmp_path), flac_case.pcm16(), 48000, flac_starts(flac_case))
