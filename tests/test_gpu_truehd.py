"""TrueHD input on the GPU (sb_truehd_index / sb_truehd_decode behind WavStream): a raw .thd stream and a Matroska
A_TRUEHD track load bit for bit as the plain PCM WAV of the samples FFmpeg's decoder returns (tests/test_truehd_cases.py
holds FFmpeg to the writer's PCM) -- .data, sample_count, padding_size, sample_rate and both clip values -- in both
sample types; each damaged stream raises SushiError naming the access unit and its byte offset; the shift solver and
the command line give the same script on a TrueHD pair, raw or in Matroska, as on the WAV pair; and a 90-minute
24-bit 7.1 stream (about 1.2 GB, byte offsets past 2^32 bits) equals WavStream.from_pcm of its PCM."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, synth
from sushi_b200.wavstream import WavStream
from tests import mkv_truehd_cases as mtc
from tests import truehd_cases as tc
from tests.test_gpu_flac import assert_same_stream, _pair as flac_pair

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE, DAMAGED = tc.damaged_cases()


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case', tc.all_cases(), ids=lambda c: c.name)
def test_truehd_loads_as_its_wav(gpu_lib, tmp_path, case, stype):
    t = WavStream(case.write(tmp_path), 12000, stype)
    w = WavStream(case.write_wav(tmp_path), 12000, stype)
    try:
        assert_same_stream(t, w)
    finally:
        t.close(); w.close()


@pytest.mark.parametrize('case', DAMAGED, ids=lambda c: c.name)
def test_damaged_truehd_raises_naming_the_access_unit(gpu_lib, tmp_path, case):
    with pytest.raises(SushiError, match=case.damage[3]):
        WavStream(case.write(tmp_path), 12000, 'uint8')


def test_host_loader_and_mlp_are_refused(gpu_lib, tmp_path):
    with pytest.raises(SushiError, match='no host TrueHD decoder'):
        WavStream(tc.all_cases()[0].write(tmp_path), loader='host')
    with pytest.raises(SushiError, match=r'MLP \(DVD-Audio\) is not supported'):
        WavStream(tc.all_cases()[0].write(tmp_path, '.mlp'))


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', mtc.cases(), ids=lambda p: p[0].name)
def test_matroska_truehd_track_loads_as_its_wav(gpu_lib, tmp_path, pair, stype):
    mkv, case = pair
    t = WavStream(mkv.write(tmp_path), 12000, stype)
    w = WavStream(case.write_wav(tmp_path), 12000, stype)
    assert_same_stream(t, w)


def _thd_pair(tmp_path, dur=30.0, shift=-1.5, seed=5):
    """A 48 kHz stereo source / destination pair as (TrueHD, WAV, FLAC) of the same samples, the ASS script and the
    TrueHD cases."""
    paths, script = flac_pair(tmp_path, dur=dur, shift=shift, seed=seed)
    out, cases = {}, {}
    for name, (flac_path, wav_path) in paths.items():
        import wave
        with wave.open(wav_path, 'rb') as r:
            pcm = np.frombuffer(r.readframes(r.getnframes()), '<i2').reshape(-1, 2).astype(np.int64)
        n_au = len(pcm) // 40
        pcm = pcm[:n_au * 40] << 8
        w = tc.Writer(48000, pcm, 16, seed=seed, style={'permute': False, 'blocks': True},
                      restarts=(16,))
        case = tc.TrueHDCase(name, w.encode(), pcm, 48000, w.au_offsets, w.seg_starts)
        assert len(pcm) == n_au * 40                    # whole AUs: the FLAC holds the same samples
        out[name] = (case.write(tmp_path), case.write_wav(tmp_path), flac_path)
        cases[name] = case
    return out, script, cases


def test_command_line_on_truehd_equals_wav(gpu_lib, tmp_path):
    paths, script, _ = _thd_pair(tmp_path)
    out = {}
    for k, kind in enumerate(('thd', 'wav')):
        dst = str(tmp_path / ('out_%s.ass' % kind))
        p = subprocess.run([sys.executable, '-m', 'sushi_b200', '--src', paths['src'][k], '--dst', paths['dst'][k],
                            '--script', script, '-o', dst], cwd=ROOT, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        out[kind] = open(dst, 'rb').read()
    assert out['thd'] == out['wav']


def test_command_line_on_matroska_truehd_and_flac_equals_wav(gpu_lib, tmp_path):
    """--src a.mkv (TrueHD track) --dst b.flac against the same audio as WAV files; no WAV is written for the MKV."""
    from tests import mkv_truehd_cases as mtc
    paths, script, cases = _thd_pair(tmp_path)
    mkv = mtc.audio_only('src_mkv', cases['src']).write(tmp_path)
    dst_flac = paths['dst'][2]
    out = {}
    for kind, src, dst in (('mkv', mkv, dst_flac), ('wav', paths['src'][1], paths['dst'][1])):
        o = str(tmp_path / ('out_%s.ass' % kind))
        p = subprocess.run([sys.executable, '-m', 'sushi_b200', '--src', src, '--dst', dst, '--script', script, '-o', o],
                           cwd=ROOT, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        out[kind] = open(o, 'rb').read()
    assert out['mkv'] == out['wav']
    assert not [n for n in os.listdir(str(tmp_path)) if n.startswith('src_mkv') and n.endswith('.wav')]


def test_ninety_minute_71_stream_equals_pcm(gpu_lib, tmp_path):
    seg, pcm, reps = tc.long_stream()
    path = str(tmp_path / 'long.thd')
    with open(path, 'wb') as f:
        for _ in range(reps):
            f.write(seg)
    assert os.path.getsize(path) * 8 > 2 ** 32
    got = WavStream(path, 12000, 'uint8')
    want = WavStream.from_pcm(np.tile(pcm, (reps, 1)), 48000, 12000, 'uint8', channels=8)
    assert_same_stream(got, want)
