"""Transport stream inputs on the GPU (sb_ts_*): a BD-LPCM or TrueHD stream of an .m2ts or .ts file loads bit for bit as
the plain PCM WAV of the samples FFmpeg's decoder returns (tests/test_ts_cases.py holds FFmpeg to the writer's PCM),
whatever the chunk size the file is fed in; damage is refused naming its byte offset; a cut copy keeps what FFmpeg
keeps; the command line on transport streams writes what it writes on the WAVs."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, mpegts, synth
from sushi_b200.common import py2_round
from sushi_b200.wavstream import WavStream
from tests import flac_cases as fc
from tests import mkv_cases as mc
from tests import ts_cases as tsc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STREAMS = [(c, s) for c in tsc.all_cases() if c.hdmv and not c.refused and c.name != 'bd_stereo20_48k'
           for s in c.audio()]


def _sid(path, pid, codec):
    return next(s.id for s in mpegts.TransportStream(path).streams_all if s.pid == pid and s.codec == codec)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', STREAMS, ids=lambda p: '%s-%x' % (p[0].name, p[1].pid))
def test_stream_loads_as_the_wav_of_its_pcm(gpu_lib, tmp_path, monkeypatch, pair, stype):
    case, s = pair
    path = case.write(tmp_path)
    sid = _sid(path, s.pid, 'truehd' if s.kind == 'truehd' else 'pcm_bluray')
    want = WavStream(tsc.write_wav(tmp_path / 'w.wav', s.pcm, s.rate), 12000, stype)
    for packets in (None, 7, 61):                       # the default chunk, and chunks that split PES packets
        if packets:
            monkeypatch.setattr(mpegts, 'CHUNK_BYTES', packets * case.psize)
        got = WavStream(path, 12000, stype, track=sid)
        assert_same_stream(got, want)
        got.close()


def test_truehd_stream_loads_as_its_thd(gpu_lib, tmp_path):
    case = tsc.case('bd_truehd')
    s = next(x for x in case.streams if x.kind == 'truehd')
    thd = tmp_path / 'a.thd'
    thd.write_bytes(b''.join(p[s.header_len:] for p, f in zip(s.pes, s.pes_frames) if f is not None))
    path = case.write(tmp_path)
    assert_same_stream(WavStream(path, 12000, 'float32', track=1), WavStream(str(thd), 12000, 'float32'))


def test_opened_transport_stream_and_host_loader(gpu_lib, tmp_path):
    case = tsc.case('bd_8ch24_48k')
    s = case.audio()[0]
    ts = mpegts.TransportStream(case.write(tmp_path))
    assert_same_stream(WavStream(ts, 8000, 'uint8'), WavStream(tsc.write_wav(tmp_path / 'w.wav', s.pcm, s.rate), 8000))
    with pytest.raises(SushiError, match="needs loader='gpu'"):
        WavStream(ts, loader='host')


@pytest.mark.parametrize('case', tsc.damaged_cases(), ids=lambda c: c.name)
def test_damaged_copy_is_refused_naming_its_offset(gpu_lib, tmp_path, monkeypatch, case):
    monkeypatch.setattr(mpegts, 'CHUNK_BYTES', 50 * case.psize)
    with pytest.raises(SushiError, match=case.damage[0]) as e:
        WavStream(case.write(tmp_path), 12000, 'uint8', track=1)
    assert 'byte offset %d:' % case.damage[1] in str(e.value), str(e.value)


def test_twenty_bit_lpcm_is_refused(gpu_lib, tmp_path):
    with pytest.raises(SushiError, match='20-bit BD-LPCM'):
        WavStream(tsc.case('bd_stereo20_48k').write(tmp_path))


@pytest.mark.parametrize('case', tsc.cut_cases(), ids=lambda c: c.name)
def test_cut_copy_keeps_what_ffmpeg_keeps(gpu_lib, tmp_path, case):
    s = next(x for x in case.streams if x.kind == 'lpcm')
    got = WavStream(case.write(tmp_path), 12000, 'float32', track=_sid(case.write(tmp_path), s.pid, 'pcm_bluray'))
    assert_same_stream(got, WavStream(tsc.write_wav(tmp_path / 'w.wav', case.expected(s), s.rate), 12000, 'float32'))


def test_ninety_minutes_of_24_bit_stereo_equals_from_pcm(gpu_lib, tmp_path):
    path = str(tmp_path / 'long.m2ts')
    pcm, reps = tsc.long_m2ts(path)
    assert os.path.getsize(path) > 10 ** 9
    got = WavStream(path, 12000, 'uint8')
    want = WavStream.from_pcm(np.tile(pcm, (reps, 1)), 48000, 12000, 'uint8', channels=2)
    assert_same_stream(got, want)


def test_command_line_on_transport_stream_equals_wav(gpu_lib, tmp_path):
    from sushi_b200.common import format_time
    dur, seed = 40.0, 5
    src12, dst12 = synth.make_pair(dur, seed, -1.5)
    rng = np.random.default_rng(seed)
    starts, ends = synth.make_events(24, dur - 8.0, seed, 0.8, 3.0, 1.5)
    head = mc.ass_script(seed)[0]
    lines = list(head) + ['Dialogue: 0,%s,%s,Default,,0,0,0,,line %d' % (
        format_time(py2_round(a * 100) / 100.0), format_time(py2_round(b * 100) / 100.0), i)
        for i, (a, b) in enumerate(zip(starts, ends))]
    (tmp_path / 'in.ass').write_text('\n'.join(lines) + '\n', encoding='utf-8')
    up = np.repeat(src12, 4).astype(np.int64)
    src = tsc.TsCase('src', 192, True, [tsc.blob_stream(tsc.VIDEO_PID, 0x1B, 'video', 20, 20000, rng),
                                        tsc.lpcm_stream(tsc.AUDIO_PID, 2, 16, 48000, 0, rng, pcm=np.stack([up, up // 2], 1)),
                                        tsc.blob_stream(tsc.PGS_PID, 0x90, 'pgs', 3, 300, rng)], rng)
    src_ts = src.write(tmp_path)
    src_wav = tsc.write_wav(tmp_path / 'src.wav', src.streams[1].pcm, 48000)
    up = np.repeat(dst12, 4).astype(np.int64)
    st = np.stack([up, up // 2], 1)
    flac, infos, offsets = fc.encode(st, 48000, 16, fc.fixed_blocks(len(st), 4096),
                                     fc.stereo_plan(['lpc'], assignments=(10, 0, 8, 9), order=10, porder=6), rng)
    dst_flac = tmp_path / 'dst.flac'
    dst_flac.write_bytes(flac)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', st.astype(np.int16), 48000)
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    outs = []
    for a, b, name in ((src_ts, str(dst_flac), 'ts.ass'), (src_wav, dst_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', b, '-o', outs[-1]], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
    # the empty chapter file is written at the reference's path and removed
    assert not os.path.exists(src_ts + '.sushi.chapters.txt')
