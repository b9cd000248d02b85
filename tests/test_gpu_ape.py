"""Monkey's Audio inputs on the GPU, through sb_ape_decode_frames: every case of tests/ape_cases.py loads bit for bit as
the plain PCM WAV of the samples FFmpeg's decoder returns (tests/test_ape_cases.py holds FFmpeg to the writer's PCM),
in both sample types, and its decoded handle holds those samples at the stream's own rate, every frame.  Also 90
minutes of insane-level stereo at 16 and 24 bits, every damaged copy named by frame and offset, --ffmpeg-audio on
16-bit mono and stereo against libswresample on FFmpeg's own decode (and the S32 refusal at 24 bits), and the command
line on .ape source and destination against the run on the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, ape, synth
from sushi_b200.common import py2_round
from sushi_b200.wavstream import WavStream
from tests import ape_cases as ac
from tests import mkv_cases as mc
from tests import ts_cases as tsc
from tests.test_gpu_decoded_pcm import Periodic, assert_decodes_to
from tests.test_gpu_ffmpeg_audio import assert_same, ffmpeg_decoded
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(name):
    return next(c for c in ac.all_cases() if c.name == name)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', ac.all_cases(), ids=lambda c: c.name)
def test_ape_file_loads_as_the_wav_of_its_pcm(gpu_lib, tmp_path, case, stype):
    path = tmp_path / (case.name + '.ape')
    path.write_bytes(case.ape())
    got = WavStream(str(path), 12000, stype)
    want = WavStream(tsc.write_wav(tmp_path / 'w.wav', case.pcm16, case.rate), 12000, stype)
    assert_same_stream(got, want)


@pytest.mark.parametrize('case', ac.all_cases(), ids=lambda c: c.name)
def test_decoded_handle_holds_every_frame(gpu_lib, tmp_path, case):
    path = tmp_path / (case.name + '.ape')
    path.write_bytes(case.ape())
    assert_decodes_to(str(path), case.pcm16, case.rate, case.bpf)


@pytest.mark.parametrize('bits', [16, 24])
def test_ninety_minutes_of_insane_stereo(gpu_lib, tmp_path, bits):
    case, data, reps = ac.long_stream(bits=bits, minutes=90)
    path = tmp_path / 'long.ape'
    path.write_bytes(data)
    del data
    assert_decodes_to(str(path), Periodic(case.pcm16, reps), 48000, case.bpf)
    got = WavStream(str(path), 12000, 'uint8')
    want = WavStream.from_pcm(ac.long_pcm16(case, reps), 48000, 12000, 'uint8', channels=2)
    assert got.sample_count == want.sample_count
    assert_same_stream(got, want)


def test_host_loader_is_refused(gpu_lib, tmp_path):
    path = tmp_path / 'a.ape'
    path.write_bytes(ac.all_cases()[0].ape())
    with pytest.raises(SushiError, match="APE input needs loader='gpu'"):
        WavStream(str(path), loader='host')


@pytest.mark.parametrize('damaged', ac.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_frame_and_offset(gpu_lib, tmp_path, damaged):
    name, data, frame, regex, kernel = damaged
    path = tmp_path / (name + '.ape')
    path.write_bytes(data)
    with pytest.raises(SushiError, match=regex) as e:
        WavStream(str(path), 12000, 'uint8')
    if kernel:
        where = int(ape.ApeFile(str(path)).offsets[frame])
        assert 'APE frame %d at byte offset %d:' % (frame, where) in str(e.value), str(e.value)


@pytest.mark.parametrize('name', ['l3_1ch_16', 'l5_2ch_16', 'specials_stereo', 'tags'])
def test_ffmpeg_audio_against_ffmpeg(gpu_lib, tmp_path, name):
    case = _case(name)
    path = tmp_path / (name + '.ape')
    path.write_bytes(case.ape())
    assert_same(WavStream(str(path), ffmpeg_audio=True), ffmpeg_decoded(tmp_path, str(path)))


def test_ffmpeg_audio_refuses_24_bits(gpu_lib, tmp_path):
    path = tmp_path / 'a.ape'
    path.write_bytes(_case('l5_2ch_24').ape())
    with pytest.raises(SushiError, match='this APE stream of 24 bits decodes to S32'):
        WavStream(str(path), ffmpeg_audio=True)


def _stereo(x12):
    x = x12.astype(np.int64)
    return np.stack([x, x // 2], 1)


def test_command_line_on_ape_equals_wav(gpu_lib, tmp_path):
    from sushi_b200.common import format_time
    dur, seed = 40.0, 7
    src12, dst12 = synth.make_pair(dur, seed, -1.5)
    starts, ends = synth.make_events(24, dur - 8.0, seed, 0.8, 3.0, 1.5)
    head = mc.ass_script(seed)[0]
    lines = list(head) + ['Dialogue: 0,%s,%s,Default,,0,0,0,,line %d' % (
        format_time(py2_round(a * 100) / 100.0), format_time(py2_round(b * 100) / 100.0), i)
        for i, (a, b) in enumerate(zip(starts, ends))]
    (tmp_path / 'in.ass').write_text('\n'.join(lines) + '\n', encoding='utf-8')
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    src, dst = _stereo(src12), _stereo(dst12)
    outs = []
    ape_pair = []
    for name, pcm, level in (('src', src, 5000), ('dst', dst, 2000)):
        case = ac.Case(name, pcm, 2, 16, 12000, level, ac.FULL[level])
        ape_pair.append(str(tmp_path / (name + '.ape')))
        with open(ape_pair[-1], 'wb') as f:
            f.write(case.ape())
    src_wav = tsc.write_wav(tmp_path / 'src.wav', src.astype(np.int16), 12000)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', dst.astype(np.int16), 12000)
    for a, b, name in ((ape_pair[0], ape_pair[1], 'ape.ass'), (src_wav, dst_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', b, '-o', outs[-1]], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
    assert not list(tmp_path.glob('*.wav.*'))
