"""FLAC input on the GPU (sb_flac_decode_file / sb_pcm_load behind WavStream(path)): a FLAC file loads bit for bit as the
plain PCM WAV of the same samples loads -- .data, sample_count, padding_size, sample_rate and both clip values -- on
every case of tests/flac_cases.py in both sample types; damaged files raise SushiError naming the frame; the shift
solver and the command line give the same script on a FLAC pair as on the WAV pair; and a BASELINE-size file (90
minutes, 48 kHz stereo, about 1 GB) equals WavStream.from_pcm of its PCM."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, synth
from sushi_b200.wavstream import WavStream
from tests import flac_cases as fc
from tests.test_loader_cases import same_f32

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = fc.all_cases()
BASE, CORRUPT = fc.corrupt_cases()


def assert_same_stream(a, b):
    assert (int(a.sample_count), a.padding_size, a.sample_rate) == (int(b.sample_count), b.padding_size, b.sample_rate)
    assert a.data.dtype == b.data.dtype and a.data.shape == b.data.shape
    assert np.array_equal(a.data, b.data, equal_nan=a.data.dtype == np.float32), int(np.count_nonzero(a.data != b.data))
    assert same_f32(a.min_value, b.min_value) and same_f32(a.max_value, b.max_value), (a.min_value, b.min_value,
                                                                                          a.max_value, b.max_value)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_flac_loads_as_its_wav(gpu_lib, tmp_path, case, stype):
    f = WavStream(case.write(tmp_path), case.sample_rate, stype)
    w = WavStream(case.write_wav(tmp_path), case.sample_rate, stype)
    try:
        assert_same_stream(f, w)
    finally:
        f.close(); w.close()


@pytest.mark.parametrize('case', CORRUPT, ids=lambda c: c.name)
def test_corrupt_flac_raises_naming_the_frame(gpu_lib, tmp_path, case):
    with pytest.raises(SushiError, match=case.corrupt[3]):
        WavStream(case.write(tmp_path), 12000, 'uint8')


def test_undamaged_base_loads(gpu_lib, tmp_path):
    f = WavStream(BASE.write(tmp_path), 12000, 'uint8')
    w = WavStream(BASE.write_wav(tmp_path), 12000, 'uint8')
    assert_same_stream(f, w)


def test_unsupported_depth_and_host_loader(gpu_lib, tmp_path):
    path = fc.unsupported_bits_case().write(tmp_path)
    with pytest.raises(SushiError, match=re.escape('FLAC with 20 bits per sample is not supported (16 or 24)')):
        WavStream(path)
    with pytest.raises(SushiError, match='no host FLAC decoder'):
        WavStream(CASES[0].write(tmp_path), loader='host')


def _pair(tmp_path, dur=70.0, shift=2.25, seed=31):
    """A source / destination pair at 48 kHz stereo as FLAC (LPC, mid/side) and as WAV, and an ASS script."""
    from sushi_b200 import AssScript
    from sushi_b200.common import format_time
    src12, dst12 = synth.make_pair(dur, seed, shift)
    rng = np.random.default_rng(seed)
    paths = {}
    for name, pcm in (('src', src12), ('dst', dst12)):
        up = np.repeat(pcm, 4).astype(np.int64)
        st = np.stack([up, up // 2], 1)
        blocks = fc.fixed_blocks(len(st), 4096)
        flac, infos, offsets = fc.encode(st, 48000, 16, blocks, fc.stereo_plan(['lpc'], assignments=(10, 0, 8, 9),
                                                                               order=10, porder=6), rng)
        case = fc.FlacCase(name, flac, st, 48000, 16, infos, offsets, 12000, 'uint8')
        paths[name] = (case.write(tmp_path), case.write_wav(tmp_path))
    starts, ends = synth.make_events(24, dur - 8.0, seed, 0.8, 3.0, 1.5)
    lines = ['[Script Info]', 'Title: t', '', '[V4+ Styles]', AssScript.STYLES_FORMAT,
             'Style: Default,Arial,20,&H00FFFFFF,&H000000FF,&H00000000,&H00000000,0,0,0,0,100,100,0,0,1,2,2,2,10,10,10,1',
             '', '[Events]', AssScript.EVENTS_FORMAT]
    for i, (a, b) in enumerate(zip(starts, ends)):
        lines.append('Dialogue: 0,{0},{1},Default,,0,0,0,,line {2}'.format(format_time(a), format_time(b), i))
    (tmp_path / 'in.ass').write_text('\n'.join(lines), encoding='utf-8')
    return paths, str(tmp_path / 'in.ass')


def test_shift_script_on_flac_equals_wav(gpu_lib, tmp_path):
    from sushi_b200 import shift_script
    paths, script = _pair(tmp_path)
    shift_script(paths['src'][0], paths['dst'][0], script, str(tmp_path / 'flac.ass'))
    shift_script(paths['src'][1], paths['dst'][1], script, str(tmp_path / 'wav.ass'))
    assert (tmp_path / 'flac.ass').read_bytes() == (tmp_path / 'wav.ass').read_bytes()


def test_command_line_on_flac_equals_wav(gpu_lib, tmp_path):
    paths, script = _pair(tmp_path, dur=40.0, shift=-1.5, seed=5)
    out = {}
    for k, kind in enumerate(('flac', 'wav')):
        dst = str(tmp_path / ('out_%s.ass' % kind))
        p = subprocess.run([sys.executable, '-m', 'sushi_b200', '--src', paths['src'][k], '--dst', paths['dst'][k],
                            '--script', script, '-o', dst], cwd=ROOT, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        out[kind] = open(dst, 'rb').read()
    assert out['flac'] == out['wav']


def test_baseline_size_flac_equals_pcm(gpu_lib, tmp_path):
    """90 minutes of 48 kHz stereo in 225 001 frames (4-byte frame numbers, a 1 GB file: bit positions past 2^32)."""
    data, pcm = fc.baseline_file()
    assert len(data) * 8 > 2 ** 32
    path = str(tmp_path / 'baseline.flac')
    with open(path, 'wb') as f:
        f.write(data)
    del data
    got = WavStream(path, 12000, 'uint8')
    want = WavStream.from_pcm(pcm, fc.BASELINE_RATE, 12000, 'uint8', channels=2)
    assert_same_stream(got, want)
