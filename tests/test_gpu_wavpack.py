"""WavPack inputs on the GPU: every .wv case and every A_WAVPACK4 Matroska track loads bit for bit as the plain PCM WAV
of the samples FFmpeg's decoder returns (tests/test_wavpack_cases.py holds FFmpeg to the writer's PCM), through
sb_wavpack_decode_blocks.  Also 90 minutes of 24-bit stereo, every damaged copy named by block and offset, and the
command line against the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, synth
from sushi_b200 import wavpack as wp
from sushi_b200.common import py2_round
from sushi_b200.wavstream import WavStream
from tests import flac_cases as fc
from tests import mkv_cases as mc
from tests import mkv_wavpack_cases as mwc
from tests import ts_cases as tsc
from tests import wavpack_cases as wc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _wav(tmp_path, pcm16, rate):
    return WavStream(tsc.write_wav(tmp_path / 'w.wav', pcm16, rate), 12000, 'uint8')


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', wc.all_cases(), ids=lambda c: c.name)
def test_wv_file_loads_as_the_wav_of_its_pcm(gpu_lib, tmp_path, case, stype):
    path = tmp_path / (case.name + '.wv')
    path.write_bytes(case.wv())
    got = WavStream(str(path), 12000, stype)
    want = WavStream(tsc.write_wav(tmp_path / 'w.wav', case.pcm16, case.rate), 12000, stype)
    assert_same_stream(got, want)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', mwc.cases(), ids=lambda p: p[0].name)
def test_matroska_wavpack_track_loads_as_its_pcm(gpu_lib, tmp_path, pair, stype):
    mkv, case = pair
    n = mwc.kept_samples(mkv, case)
    got = WavStream(mkv.write(tmp_path), 12000, stype)
    assert_same_stream(got, WavStream.from_pcm(case.pcm16[:n], case.rate, 12000, stype, channels=case.channels))


def test_host_loader_is_refused(gpu_lib, tmp_path):
    case = wc.all_cases()[1]
    path = tmp_path / 'a.wv'
    path.write_bytes(case.wv())
    with pytest.raises(SushiError, match="WavPack input needs loader='gpu'"):
        WavStream(str(path), loader='host')


def test_ninety_minutes_of_24_bit_stereo_equals_from_pcm(gpu_lib, tmp_path):
    case, data, reps = wc.long_stream(bits=24, minutes=90)
    path = tmp_path / 'long.wv'
    path.write_bytes(data)
    del data
    got = WavStream(str(path), 12000, 'uint8')
    want = WavStream.from_pcm(np.tile(case.pcm16, (reps, 1)), 48000, 12000, 'uint8', channels=2)
    assert got.sample_count == want.sample_count
    assert_same_stream(got, want)


@pytest.mark.parametrize('damaged', wc.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_copy_is_refused_naming_block_and_offset(gpu_lib, tmp_path, damaged):
    name, data, block, regex, kernel = damaged
    path = tmp_path / (name + '.wv')
    path.write_bytes(data)
    with pytest.raises(SushiError, match=regex) as e:
        WavStream(str(path), 12000, 'uint8')
    if kernel:
        where = int(wp.WavPackFile(str(path)).where[block])
        assert 'WavPack block %d at byte offset %d:' % (block, where) in str(e.value), str(e.value)


def _stereo(x12):
    up = np.repeat(x12, 4).astype(np.int64)
    return np.stack([up, up // 2], 1)


def test_command_line_on_wavpack_equals_wav(gpu_lib, tmp_path):
    from sushi_b200.common import format_time
    dur, seed = 40.0, 6
    src12, dst12 = synth.make_pair(dur, seed, -1.5)
    rng = np.random.default_rng(seed)
    starts, ends = synth.make_events(24, dur - 8.0, seed, 0.8, 3.0, 1.5)
    head = mc.ass_script(seed)[0]
    lines = list(head) + ['Dialogue: 0,%s,%s,Default,,0,0,0,,line %d' % (
        format_time(py2_round(a * 100) / 100.0), format_time(py2_round(b * 100) / 100.0), i)
        for i, (a, b) in enumerate(zip(starts, ends))]
    (tmp_path / 'in.ass').write_text('\n'.join(lines) + '\n', encoding='utf-8')
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    src, dst = _stereo(src12), _stereo(dst12)
    block = 24000
    src_case = wc.make_case('src', 1, counts=(block,) * (len(src) // block) + (len(src) % block,) * bool(len(src) % block),
                            nterms=[1], joint=True, x=src)
    src_wv = tmp_path / 'src.wv'
    src_wv.write_bytes(src_case.wv())
    src_mka = mwc.audio_only('src_mka', src_case).write(tmp_path, '.mka')
    src_wav = tsc.write_wav(tmp_path / 'src.wav', src.astype(np.int16), 48000)
    flac, _, _ = fc.encode(dst, 48000, 16, fc.fixed_blocks(len(dst), 4096),
                           fc.stereo_plan(['lpc'], assignments=(10, 0, 8, 9), order=10, porder=6), rng)
    dst_flac = tmp_path / 'dst.flac'
    dst_flac.write_bytes(flac)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', dst.astype(np.int16), 48000)
    outs = []
    for a, b, name in ((str(src_wv), str(dst_flac), 'wv.ass'), (src_mka, dst_wav, 'mka.ass'),
                       (src_wav, dst_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', b, '-o', outs[-1]], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    want = open(outs[2], 'rb').read()
    assert open(outs[0], 'rb').read() == want
    assert open(outs[1], 'rb').read() == want
