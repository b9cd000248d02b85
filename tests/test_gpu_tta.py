"""TTA inputs on the GPU: every .tta case and every A_TTA1 Matroska track loads bit for bit as the plain PCM WAV of the
samples FFmpeg's decoder returns (tests/test_tta_cases.py holds FFmpeg to the writer's PCM), through
sb_tta_decode_frames.  Also 90 minutes of 24-bit stereo, every damaged copy named by frame and offset, the Matroska
Duration cases, and the command line against the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, synth
from sushi_b200 import tta
from sushi_b200.common import py2_round
from sushi_b200.wavstream import WavStream
from tests import mkv_cases as mc
from tests import mkv_tta_cases as mtc
from tests import ts_cases as tsc
from tests import tta_cases as tc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', tc.all_cases(), ids=lambda c: c.name)
def test_tta_file_loads_as_the_wav_of_its_pcm(gpu_lib, tmp_path, case, stype):
    path = tmp_path / (case.name + '.tta')
    path.write_bytes(case.tta())
    got = WavStream(str(path), 12000, stype)
    want = WavStream(tsc.write_wav(tmp_path / 'w.wav', case.pcm16, case.rate), 12000, stype)
    assert_same_stream(got, want)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', mtc.cases(), ids=lambda p: p[0].name)
def test_matroska_tta_track_loads_as_its_pcm(gpu_lib, tmp_path, pair, stype):
    mkv, case, outcome = pair
    path = mkv.write(tmp_path)
    if outcome == 'refused':
        with pytest.raises(SushiError, match='TTA frame %d at byte offset %d: ' % (
                len(case.frames) - 1, mkv.expect[0][-1][2])):
            WavStream(path, 12000, stype)
        return
    got = WavStream(path, 12000, stype)
    assert_same_stream(got, WavStream.from_pcm(case.pcm16, case.rate, 12000, stype, channels=case.channels))


def test_host_loader_is_refused(gpu_lib, tmp_path):
    path = tmp_path / 'a.tta'
    path.write_bytes(tc.all_cases()[1].tta())
    with pytest.raises(SushiError, match="TTA input needs loader='gpu'"):
        WavStream(str(path), loader='host')


def test_ninety_minutes_of_24_bit_stereo_equals_from_pcm(gpu_lib, tmp_path):
    case, data, reps = tc.long_stream(bits=24, minutes=90)
    path = tmp_path / 'long.tta'
    path.write_bytes(data)
    del data
    got = WavStream(str(path), 12000, 'uint8')
    want = WavStream.from_pcm(tc.long_pcm16(case, reps), 48000, 12000, 'uint8', channels=2)
    assert got.sample_count == want.sample_count
    assert_same_stream(got, want)


@pytest.mark.parametrize('damaged', tc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_frame_and_offset(gpu_lib, tmp_path, damaged):
    name, data, frame, regex, kernel = damaged
    path = tmp_path / (name + '.tta')
    path.write_bytes(data)
    with pytest.raises(SushiError, match=regex) as e:
        WavStream(str(path), 12000, 'uint8')
    if kernel:
        where = int(tta.TTAFile(str(path)).where[frame])
        assert 'TTA frame %d at byte offset %d:' % (frame, where) in str(e.value), str(e.value)


def _stereo(x12):
    x = x12.astype(np.int64)
    return np.stack([x, x // 2], 1)


def test_command_line_on_tta_equals_wav(gpu_lib, tmp_path):
    from sushi_b200.common import format_time
    dur, seed = 40.0, 6
    src12, dst12 = synth.make_pair(dur, seed, -1.5)
    starts, ends = synth.make_events(24, dur - 8.0, seed, 0.8, 3.0, 1.5)
    head = mc.ass_script(seed)[0]
    lines = list(head) + ['Dialogue: 0,%s,%s,Default,,0,0,0,,line %d' % (
        format_time(py2_round(a * 100) / 100.0), format_time(py2_round(b * 100) / 100.0), i)
        for i, (a, b) in enumerate(zip(starts, ends))]
    (tmp_path / 'in.ass').write_text('\n'.join(lines) + '\n', encoding='utf-8')
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    src, dst = _stereo(src12), _stereo(dst12)
    src_tta = tmp_path / 'src.tta'
    src_tta.write_bytes(tc.make_case('src', 1, rate=12000, pcm=src).tta())
    dst_mkv = mtc.audio_only('dst', tc.make_case('dst', 2, rate=12000, pcm=dst)).write(tmp_path, '.mkv')
    src_wav = tsc.write_wav(tmp_path / 'src.wav', src.astype(np.int16), 12000)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', dst.astype(np.int16), 12000)
    outs = []
    for a, b, name in ((str(src_tta), dst_mkv, 'tta.ass'), (src_wav, dst_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', b, '-o', outs[-1]], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
    assert not list(tmp_path.glob('*.wav.*'))
