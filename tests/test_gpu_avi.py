"""AVI files on the GPU: every audio stream of every good case of tests/avi_cases.py loads bit for bit as the plain PCM
WAV of FFmpeg's decode, in both sample types and with feeds small enough to split chunk headers and payloads;
--ffmpeg-audio equals libswresample on FFmpeg's decode and layout for 16-bit PCM and MP2; damaged copies and partial
PCM frames are refused with the CPU build's message; a cut copy loads as FFmpeg decodes it; a 90-minute 24-bit stereo
OpenDML file over 1 GiB loads as WavStream.from_pcm of its samples; the command line on an .avi equals the command line
on its WAV."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, avi
from sushi_b200.wavstream import WavStream
from tests import avi_cases as ac
from tests import ref_mp4
from tests import ref_swr
from tests import ts_cases as tsc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOOD = ac.good_cases()


def _ffmpeg_wav(tmp_path, path, sid, name='ffmpeg.wav'):
    """the plain 16-bit WAV of FFmpeg's decode of stream `sid` (24-bit PCM by its top 16 bits; packets the decoder
    refuses skipped, as the ffmpeg command line skips them)"""
    out, sfmt, _, _, rate = ref_mp4._decode(path, sid, None)
    if sfmt in (2, 7):
        out = out >> 16
    return tsc.write_wav(tmp_path / name, out.astype(np.int16), rate)


def _pairs():
    return [(c, i) for c in GOOD for i, _ in c.audio()]


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', _pairs(), ids=lambda p: '%s_%d' % (p[0].name, p[1]))
def test_avi_loads_as_ffmpegs_decode(gpu_lib, tmp_path, pair, stype):
    case, sid = pair
    path = case.write(tmp_path)
    want = WavStream(_ffmpeg_wav(tmp_path, path, sid), 12000, stype)
    assert_same_stream(WavStream(avi.AviFile(path), 12000, stype, track=sid), want)


@pytest.mark.parametrize('name', ['pcm16_mono_rec', 'mp2_vbr_odml'])
def test_small_feeds_split_chunks(gpu_lib, tmp_path, monkeypatch, name):
    case = next(c for c in GOOD if c.name == name)
    path = case.write(tmp_path)
    want = WavStream(_ffmpeg_wav(tmp_path, path, 1), 12000, 'uint8')
    for feed in (5, 13, 777, 4096):
        monkeypatch.setattr(avi, 'CHUNK_BYTES', feed)
        assert_same_stream(WavStream(path, 12000, 'uint8', track=1), want)


@pytest.mark.parametrize('name', ['pcm16_every_frame', 'two_audio_preload', 'pcm16_mono_rec', 'mp2_cbr_subs',
                                  'mp2_vbr_odml'])
def test_ffmpeg_audio_equals_libswresample_on_ffmpegs_decode(gpu_lib, tmp_path, name):
    case = next(c for c in GOOD if c.name == name)
    path = case.write(tmp_path)
    sid = next(i for i, s in case.audio() if s.codec == 'mp2' or s.bits == 16)
    pcm, mask, rate = ref_mp4.decode_s16(path, sid)
    mono = ref_swr.convert(pcm, mask, rate, 12000)
    want = WavStream(tsc.write_wav(tmp_path / 'swr.wav', mono.reshape(-1, 1), 12000), 12000, 'float32')
    assert_same_stream(WavStream(path, 12000, 'float32', track=sid, ffmpeg_audio=True), want)


@pytest.mark.parametrize('damaged', ac.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_with_the_cpu_builds_message(gpu_lib, tmp_path, damaged):
    name, data, offset, regex = damaged
    path = ac.damaged_cases()[0].write(tmp_path, data, '_' + name + '.avi')
    with pytest.raises(SushiError, match='AVI chunk at byte offset %d: .*%s' % (offset, regex)):
        WavStream(path, 12000, 'uint8', track=1)


def test_partial_pcm_frames_are_refused(gpu_lib, tmp_path):
    case, sid, offset = ac.partial_frame_case()
    with pytest.raises(SushiError, match='AVI chunk at byte offset %d: PCM chunk is not a whole number of sample '
                                         'frames' % offset):
        WavStream(case.write(tmp_path), 12000, 'uint8', track=sid)


def test_cut_copy_loads_as_ffmpeg_decodes_it(gpu_lib, tmp_path):
    base, data, _ = ac.cut_case()
    path = base.write(tmp_path, data, '_cut.avi')
    assert_same_stream(WavStream(path, 12000, 'uint8', track=1),
                       WavStream(_ffmpeg_wav(tmp_path, path, 1), 12000, 'uint8'))


def test_long_opendml_file_loads_as_its_samples(gpu_lib, tmp_path):
    path = str(tmp_path / 'long.avi')
    pcm = ac.long_file(path, 90.0, 24)
    assert os.path.getsize(path) > 1 << 30 and len(avi.AviFile(path).movi) == 2
    want = WavStream.from_pcm(pcm, 48000, 12000, 'uint8', channels=2)
    del pcm
    assert_same_stream(WavStream(path, 12000, 'uint8'), want)


def test_command_line_on_an_avi_equals_wav(gpu_lib, tmp_path):
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
    rng = np.random.default_rng([seed])
    v = ac.video_stream(rng, 60)
    a = ac.pcm_stream(rng, 2, 16, 48000, 24000, chunk_frames=60)
    t = np.arange(24000 * 60) / 48000.0
    tone = (8000 * np.sin(2 * np.pi * (220 + 40 * np.sin(t)) * t) * (1 + np.sin(t * 3))).astype('<i2')
    pcm = np.stack([tone, tone[::-1]], 1)
    a.chunks = [pcm[k * 24000:(k + 1) * 24000].tobytes() for k in range(60)]
    a.es = b''.join(a.chunks)
    case = ac.AviCase('capture', [v, a], ac.interleave([v, a], rng, per=[12, 1]), segments=2, junk=4)
    src_avi = case.write(tmp_path)
    dst_wav = _ffmpeg_wav(tmp_path, src_avi, 1, 'dst.wav')
    src_wav = _ffmpeg_wav(tmp_path, src_avi, 1, 'src.wav')
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    outs = []
    for src, name in ((src_avi, 'avi.ass'), (src_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', src, '--dst', dst_wav, '-o', outs[-1]], cwd=ROOT, capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
