"""TAK inputs on the GPU, through sb_tak_decode_file: every case of tests/tak_cases.py loads bit for bit as the plain
PCM WAV of the samples FFmpeg's decoder returns (tests/test_tak_cases.py holds FFmpeg to the writer's PCM), in both
sample types, and its decoded handle holds those samples at the stream's own rate, every frame.  Also 90 minutes of
stereo at 16 and 24 bits at the largest filter order, every damaged copy named by frame and offset, --ffmpeg-audio on
16-bit mono, stereo and multichannel against libswresample on FFmpeg's own decode (and the S32 refusal at 24 bits), a
.tak file named .wav, and the command line on .tak source and destination against the run on the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, synth
from sushi_b200.common import py2_round
from sushi_b200.wavstream import WavStream
from tests import mkv_cases as mc
from tests import tak_cases as tc
from tests import ts_cases as tsc
from tests.test_gpu_decoded_pcm import Periodic, assert_decodes_to
from tests.test_gpu_ffmpeg_audio import assert_same, ffmpeg_decoded
from tests.test_gpu_flac import assert_same_stream
from tests.test_kernel_emulation_tak import _frames_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(name):
    return next(c for c in tc.all_cases() if c.name == name)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', tc.all_cases(), ids=lambda c: c.name)
def test_tak_file_loads_as_the_wav_of_its_pcm(gpu_lib, tmp_path, case, stype):
    path = tmp_path / (case.name + '.tak')
    path.write_bytes(case.tak())
    got = WavStream(str(path), 12000, stype)
    want = WavStream(tsc.write_wav(tmp_path / 'w.wav', case.pcm16, case.rate), 12000, stype)
    assert_same_stream(got, want)


@pytest.mark.parametrize('case', tc.all_cases(), ids=lambda c: c.name)
def test_decoded_handle_holds_every_frame(gpu_lib, tmp_path, case):
    path = tmp_path / (case.name + '.tak')
    path.write_bytes(case.tak())
    assert_decodes_to(str(path), case.pcm16, case.rate, case.nb)


@pytest.mark.parametrize('bits', [16, 24])
def test_ninety_minutes_of_stereo_at_the_largest_order(gpu_lib, tmp_path, bits):
    case, data, reps = tc.long_stream(bits=bits, minutes=90)
    path = tmp_path / 'long.tak'
    path.write_bytes(data)
    del data
    assert_decodes_to(str(path), Periodic(case.pcm16, reps), 48000, case.nb)
    got = WavStream(str(path), 12000, 'uint8')
    want = WavStream.from_pcm(tc.long_pcm16(case, reps), 48000, 12000, 'uint8', channels=2)
    assert got.sample_count == want.sample_count
    assert_same_stream(got, want)


@pytest.mark.parametrize('damaged', tc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_frame_and_offset(gpu_lib, tmp_path, damaged):
    from sushi_b200 import tak
    name, data, frame, regex, _ = damaged
    path = tmp_path / (name + '.tak')
    path.write_bytes(data)
    with pytest.raises(SushiError, match=regex) as e:
        WavStream(str(path), 12000, 'uint8')
    if frame is not None:
        f = tak.TakFile(str(path))
        where = f.audio_start + sum(len(x) for x in _frames_of(f, frame))
        assert 'TAK frame %d at byte offset %d:' % (frame, where) in str(e.value), str(e.value)


@pytest.mark.parametrize('name', ['partitioned', 'dmode1', 'mc6_plain', 'mc3', 'tags'])
def test_ffmpeg_audio_against_ffmpeg(gpu_lib, tmp_path, name):
    case = _case(name)
    assert case.bits == 16
    path = tmp_path / (name + '.tak')
    path.write_bytes(case.tak())
    assert_same(WavStream(str(path), ffmpeg_audio=True), ffmpeg_decoded(tmp_path, str(path)))


def test_ffmpeg_audio_refuses_24_bits(gpu_lib, tmp_path):
    path = tmp_path / 'a.tak'
    path.write_bytes(_case('dmode0').tak())
    with pytest.raises(SushiError, match='this TAK stream of 24 bits decodes to S32'):
        WavStream(str(path), ffmpeg_audio=True)


def test_tak_named_wav_opens_as_tak(gpu_lib, tmp_path):
    case = _case('dmode3')
    path = tmp_path / 'renamed.wav'
    path.write_bytes(case.tak())
    want = WavStream(tsc.write_wav(tmp_path / 'w.wav', case.pcm16, case.rate), 12000, 'uint8')
    assert_same_stream(WavStream(str(path), 12000, 'uint8'), want)


def _stereo(x12):
    x = x12.astype(np.int64)
    return np.stack([x, x // 2], 1)


def test_command_line_on_tak_equals_wav(gpu_lib, tmp_path):
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
    tak_pair = []
    for name, pcm, ft in (('src', src, 7), ('dst', dst, 9)):
        case = tc.Case(name, pcm, 16, 12000, ft)
        tak_pair.append(str(tmp_path / (name + '.tak')))
        with open(tak_pair[-1], 'wb') as f:
            f.write(case.tak())
    src_wav = tsc.write_wav(tmp_path / 'src.wav', src.astype(np.int16), 12000)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', dst.astype(np.int16), 12000)
    for a, b, name in ((tak_pair[0], tak_pair[1], 'tak.ass'), (src_wav, dst_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', b, '-o', outs[-1]], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
    assert not list(tmp_path.glob('*.wav.*'))
