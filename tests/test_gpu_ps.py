"""MPEG program streams and raw MPEG audio on the GPU: every good case of tests/ps_cases.py and every raw file of
tests/mpa_cases.py loads bit for bit as the plain PCM WAV of FFmpeg's decode, in both sample types and (program streams)
with chunks small enough to split start codes, pack headers and PES packets; --ffmpeg-audio equals libswresample on
FFmpeg's decode; damaged copies are refused with the CPU build's message; a cut copy loads as FFmpeg decodes it; the
command line on a .mpg pair writes what it writes for the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, mpegps
from sushi_b200.wavstream import WavStream
from tests import mp2_cases as mc
from tests import mpa_cases
from tests import ps_cases as pc
from tests import ref_mp4
from tests import ref_swr
from tests import ts_cases as tsc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOOD = pc.good_cases()


def _ffmpeg_wav(tmp_path, path, sid=None, name='ffmpeg.wav'):
    if sid is None:
        sid = next(i for i, s in enumerate(mpegps.ProgramStream(path).streams_all) if s.kind == 'audio')
    pcm, _, rate = ref_mp4.decode_s16(path, sid)
    return tsc.write_wav(tmp_path / name, pcm, rate)


def _pairs():
    """(case, stream index) of every MPEG audio stream of the good cases"""
    out = []
    for c in GOOD:
        for e in c.audio():
            out.append((c, 0x100 | e.sid))
    return out


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', _pairs(), ids=lambda p: '%s_%x' % (p[0].name, p[1]))
def test_program_stream_loads_as_ffmpegs_decode(gpu_lib, tmp_path, pair, stype):
    case, stream_id = pair
    path = case.write(tmp_path)
    ps = mpegps.ProgramStream(path)
    sid = next(s.id for s in ps.streams_all if s.stream_id == stream_id)
    want = WavStream(_ffmpeg_wav(tmp_path, path, sid), 12000, stype)
    assert_same_stream(WavStream(ps, 12000, stype, track=sid), want)


def test_small_chunks_split_packets(gpu_lib, tmp_path, monkeypatch):
    case = next(c for c in GOOD if c.name == 'dvd_joint')
    path = case.write(tmp_path)
    want = WavStream(_ffmpeg_wav(tmp_path, path, 5), 12000, 'uint8')
    for chunk in (6, 17, 777, 4096):
        monkeypatch.setattr(mpegps, 'CHUNK_BYTES', chunk)
        assert_same_stream(WavStream(path, 12000, 'uint8', track=5), want)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', mpa_cases.all_cases(), ids=lambda c: c[0])
def test_raw_mpeg_audio_loads_as_ffmpegs_decode(gpu_lib, tmp_path, case, stype):
    name, data = case[:2]
    path = tmp_path / (name + '.mp2')
    path.write_bytes(data)
    want = WavStream(_ffmpeg_wav(tmp_path, str(path), 0), 12000, stype)
    assert_same_stream(WavStream(str(path), 12000, stype), want)


@pytest.mark.parametrize('which', ['vcd_stereo', 'dvb_mono_psm', 'mpa'])
def test_ffmpeg_audio_equals_libswresample_on_ffmpegs_decode(gpu_lib, tmp_path, which):
    if which == 'mpa':
        path = str(tmp_path / 'a.mp2')
        open(path, 'wb').write(mpa_cases.all_cases()[1][1])
        sid = 0
    else:
        path = next(c for c in GOOD if c.name == which).write(tmp_path)
        sid = next(s.id for s in mpegps.ProgramStream(path).streams_all if s.kind == 'audio')
    pcm, mask, rate = ref_mp4.decode_s16(path, sid)
    mono = ref_swr.convert(pcm, mask, rate, 12000)
    want = WavStream(tsc.write_wav(tmp_path / 'swr.wav', mono.reshape(-1, 1), 12000), 12000, 'float32')
    assert_same_stream(WavStream(path, 12000, 'float32', ffmpeg_audio=True), want)


@pytest.mark.parametrize('damaged', pc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_with_the_cpu_builds_message(gpu_lib, tmp_path, damaged):
    name, data, offset, regex = damaged
    path = pc.damaged_cases()[0].write(tmp_path, data, '_' + name + '.vob')
    kind = 'PES packet' if 'PES header' in regex else 'program stream packet'
    ps = mpegps.ProgramStream(path)
    sid = next(s.id for s in ps.streams_all if s.stream_id == 0x1C0)
    with pytest.raises(SushiError, match='%s at byte offset %d: %s' % (kind, offset, regex)):
        WavStream(ps, 12000, 'uint8', track=sid)


def test_cut_copy_loads_as_ffmpeg_decodes_it(gpu_lib, tmp_path):
    base, data, _ = pc.cut_case()
    path = base.write(tmp_path, data, '_cut.mpg')
    assert_same_stream(WavStream(mpegps.ProgramStream(path), 12000, 'uint8', track=0),
                       WavStream(_ffmpeg_wav(tmp_path, path, 0), 12000, 'uint8'))


def test_command_line_on_a_program_stream_equals_wav(gpu_lib, tmp_path):
    from sushi_b200 import synth
    from sushi_b200.common import format_time, py2_round
    from tests import mkv_cases as mkc
    dur, seed = 30.0, 8
    starts, ends = synth.make_events(12, dur - 8.0, seed, 0.8, 3.0, 1.5)
    head = mkc.ass_script(seed)[0]
    lines = list(head) + ['Dialogue: 0,%s,%s,Default,,0,0,0,,line %d' % (
        format_time(py2_round(a * 100) / 100.0), format_time(py2_round(b * 100) / 100.0), i)
        for i, (a, b) in enumerate(zip(starts, ends))]
    (tmp_path / 'in.ass').write_text('\n'.join(lines) + '\n', encoding='utf-8')
    frames, data = mc.long_stream(dur / 60.0, distinct=40, seed=seed)
    case = mc.Case('capture', frames, [mc.FrameSpec(mode=0, rate=48000)])
    ps = pc.PsCase('capture', True, [pc.Elem(pc.VIDEO, 'video', pc.video_blob(np.random.default_rng([9]), 30000, True)),
                                     pc.Elem(pc.AUDIO, 'mp2', data, case=case)], 21, nav=True, pad=True)
    src_ps = ps.write(tmp_path)
    dst_wav = _ffmpeg_wav(tmp_path, src_ps, name='dst.wav')
    src_wav = _ffmpeg_wav(tmp_path, src_ps, name='src.wav')
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    outs = []
    for a, name in ((src_ps, 'ps.ass'), (src_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', dst_wav, '-o', outs[-1]], cwd=ROOT, capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
