"""MP2 inputs on the GPU: every transport stream and Matroska case of tests/mp2_cases.py loads bit for bit as the plain
PCM WAV of the samples FFmpeg's `mp2` decoder returns for it, in both sample types and with transport stream chunks
that split PES packets; 90 minutes of 48 kHz stereo equal WavStream.from_pcm of FFmpeg's decode; --ffmpeg-audio
equals libswresample on FFmpeg's decode; every damaged copy is refused with the CPU build's message; a track whose
frames straddle Matroska blocks is refused; the command line on a capture writes what it writes for the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, mpegts
from sushi_b200 import matroska as mk
from sushi_b200.wavstream import WavStream
from tests import mp2_cases as mc
from tests import ref_mp2
from tests import ref_mp4
from tests import ref_swr
from tests import ts_cases as tsc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = mc.all_cases()


def _ffmpeg_wav(tmp_path, path):
    pcm, _, rate = ref_mp4.decode_s16(path, 0)
    return tsc.write_wav(tmp_path / 'ffmpeg.wav', pcm, rate)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', mc.ts_files(CASES), ids=lambda p: p[0].name)
def test_transport_stream_loads_as_ffmpegs_decode(gpu_lib, tmp_path, pair, stype):
    ts, _ = pair
    path = ts.write(tmp_path)
    got = WavStream(path, 12000, stype)
    assert_same_stream(got, WavStream(_ffmpeg_wav(tmp_path, path), 12000, stype))


def test_transport_stream_chunks_that_split_pes_packets(gpu_lib, tmp_path, monkeypatch):
    ts, _ = mc.ts_files(CASES)[3]
    path = ts.write(tmp_path)
    want = WavStream(_ffmpeg_wav(tmp_path, path), 12000, 'uint8')
    for chunk in (188, 188 * 7, 188 * 61):
        monkeypatch.setattr(mpegts, 'CHUNK_BYTES', chunk)
        assert_same_stream(WavStream(path, 12000, 'uint8'), want)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', mc.mkv_files(CASES), ids=lambda p: p[0].name)
def test_matroska_track_loads_as_ffmpegs_decode(gpu_lib, tmp_path, pair, stype):
    m, _ = pair
    path = m.write(tmp_path)
    assert_same_stream(WavStream(path, 12000, stype), WavStream(_ffmpeg_wav(tmp_path, path), 12000, stype))


def test_matroska_frames_straddling_blocks_are_refused(gpu_lib, tmp_path):
    m, _ = mc.mkv_straddling(CASES)
    with pytest.raises(SushiError, match='the block does not start with a frame header|the frame runs past its block'):
        WavStream(m.write(tmp_path), 12000, 'uint8')


def test_ninety_minutes_of_stereo_equals_from_pcm(gpu_lib, tmp_path):
    frames, data = mc.long_stream(90.0)
    pcm = ref_mp2.decode_packets(frames)[0]
    # one Matroska block per 100 frames: the whole stream through sb_mp2_decode_frames
    sizes = [len(f) for f in frames]
    pieces = [sum(sizes[k:k + 100]) for k in range(0, len(sizes), 100)]
    path = mc.mkv_file('long', mc.Case('long', frames, [mc.FrameSpec(mode=0, rate=48000)]), pieces).write(tmp_path)
    got = WavStream(path, 12000, 'uint8')
    want = WavStream.from_pcm(pcm, 48000, 12000, 'uint8', channels=2)
    assert got.sample_count == want.sample_count == len(frames) * 1152 // 4
    assert_same_stream(got, want)


@pytest.mark.parametrize('pair', mc.ts_files(CASES)[:2] + mc.mkv_files(CASES)[:1], ids=lambda p: p[0].name)
def test_ffmpeg_audio_equals_libswresample_on_ffmpegs_decode(gpu_lib, tmp_path, pair):
    f, _ = pair
    path = f.write(tmp_path)
    pcm, mask, rate = ref_mp4.decode_s16(path, 0)
    mono = ref_swr.convert(pcm, mask, rate, 12000)
    want = WavStream(tsc.write_wav(tmp_path / 'swr.wav', mono.reshape(-1, 1), 12000), 12000, 'float32')
    assert_same_stream(WavStream(path, 12000, 'float32', ffmpeg_audio=True), want)


@pytest.mark.parametrize('damaged', mc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_with_the_cpu_builds_message(gpu_lib, tmp_path, damaged):
    name, data, frame, offset, regex = damaged
    # the whole copy in one Matroska block: a refusal names the frame and the file offset of that block
    m = mc.mkv_file('d_' + name, mc.Case(name, [data], [mc.FrameSpec(mode=0, rate=48000)]))
    path = m.write(tmp_path)
    with mk.MatroskaFile(path) as f:
        t = f.select('audio', None)
        block = int(f.frames([t.id])[t.id].block[0])
    with pytest.raises(SushiError, match=regex) as e:
        WavStream(path, 12000, 'uint8')
    assert 'MP2 frame %d at byte offset %d: ' % (frame, block) in str(e.value), str(e.value)


def test_command_line_on_a_capture_equals_wav(gpu_lib, tmp_path):
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
    ts = mc.TsFile('capture', data, np.random.default_rng([9]))
    src_ts = ts.write(tmp_path)
    src_wav = _ffmpeg_wav(tmp_path, src_ts)
    dst_wav = str(tmp_path / 'dst.wav')
    os.replace(src_wav, dst_wav)
    src_wav = _ffmpeg_wav(tmp_path, src_ts)
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    outs = []
    for a, name in ((src_ts, 'ts.ass'), (src_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', dst_wav, '-o', outs[-1]], cwd=ROOT, capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
