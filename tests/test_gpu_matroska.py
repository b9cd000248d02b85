"""Matroska input on the GPU (WavStream(path, track=...) over sb_flac_index_frames / sb_flac_decode and sb_load_pcm):
every audio track of tests/mkv_cases.py loads bit for bit as the plain PCM WAV of its samples loads -- .data,
sample_count, padding_size, sample_rate and both clip values -- in both sample types, the cut FLAC track and each
track of the multi-track file included; damaged FLAC frames raise SushiError naming their block's file offset; the
command line on two MKVs writes the same script as on their WAVs with the side products passed explicitly; and a
BASELINE-size file (90 minutes of 48 kHz stereo FLAC beside 129 600 video frames) equals WavStream.from_pcm."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, synth
from sushi_b200 import matroska as mk
from sushi_b200.common import py2_round
from sushi_b200.script import format_srt_time
from sushi_b200.wavstream import WavStream
from tests import flac_cases as fc
from tests import mkv_cases as mc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = mc.all_cases()
TRACKS = [(c, sid) for c in CASES if c.damage is None and c.refused is None for sid in c.audio_ids()]


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('case,sid', TRACKS, ids=lambda x: x.name if hasattr(x, 'name') else str(x))
def test_matroska_track_loads_as_its_wav(gpu_lib, tmp_path, case, sid, stype):
    rate = (12000, 8000, 24000)[sid % 3]
    m = WavStream(case.write(tmp_path), rate, stype, track=sid)
    w = WavStream(case.write_wav(tmp_path, sid), rate, stype)
    try:
        assert_same_stream(m, w)
    finally:
        m.close(); w.close()


def test_default_track_is_loaded_without_an_id(gpu_lib, tmp_path):
    case = [c for c in CASES if c.name == 'multi'][0]
    m = WavStream(case.write(tmp_path), 12000, 'uint8')
    w = WavStream(case.write_wav(tmp_path, 0), 12000, 'uint8')
    assert_same_stream(m, w)
    with pytest.raises(SushiError, match='More than one audio stream'):
        WavStream([c for c in CASES if c.name == 'two_no_default'][0].write(tmp_path))


def test_host_loader_on_pcm_and_refused_on_flac(gpu_lib, tmp_path):
    case = [c for c in CASES if c.name == 'multi'][0]
    path = case.write(tmp_path)
    for sid in (1, 2):
        m = WavStream(path, 12000, 'float32', loader='host', track=sid)
        w = WavStream(case.write_wav(tmp_path, sid), 12000, 'float32', loader='host')
        assert_same_stream(m, w)
    with pytest.raises(SushiError, match='no host FLAC decoder'):
        WavStream(path, loader='host', track=0)


@pytest.mark.parametrize('case', [c for c in CASES if c.damage and c.damage[0] in ('crc8', 'crc16', 'empty')],
                         ids=lambda c: c.name)
def test_damaged_flac_frame_names_its_block(gpu_lib, tmp_path, case):
    with pytest.raises(SushiError, match=case.damage[2]):
        WavStream(case.write(tmp_path), 12000, 'uint8')


@pytest.mark.parametrize('name', ['refused_aac', 'refused_pcm_big', 'refused_encrypted'])
def test_refused_tracks_never_reach_the_gpu(gpu_lib, tmp_path, name):
    case = [c for c in CASES if c.name == name][0]
    with pytest.raises(SushiError, match=case.refused):
        WavStream(case.write(tmp_path))


def _pair(tmp_path, dur=40.0, shift=-1.5, seed=5):
    """Source and destination as MKVs (48 kHz stereo FLAC, an ASS track, chapters, video) and as WAVs, and the files
    the WAV command is given: the script, OGM chapters, timecodes and keyframes."""
    from sushi_b200.common import format_time
    src12, dst12 = synth.make_pair(dur, seed, shift)
    rng = np.random.default_rng(seed)
    starts, ends = synth.make_events(24, dur - 8.0, seed, 0.8, 3.0, 1.5)
    head, events = mc.ass_script(seed)[0], []
    for i, (a, b) in enumerate(zip(starts, ends)):
        sa, sb = int(py2_round(a * 100)), int(py2_round(b * 100))
        events.append((i, sa, sb, '%d,0,Default,,0,0,0,,line %d' % (i, i)))
    chapters = [0, 12345 * 1000000, 27 * 10 ** 9]
    kf = '# XviD 2pass stat file\n\n\n' + ''.join('i\n' if n % 97 == 0 else 'p\n' for n in range(int(dur * 24)))
    out = {}
    for name, pcm in (('src', src12), ('dst', dst12)):
        up = np.repeat(pcm, 4).astype(np.int64)
        st = np.stack([up, up // 2], 1)
        flac, infos, offsets = fc.encode(st, 48000, 16, fc.fixed_blocks(len(st), 4096),
                                         fc.stereo_plan(['lpc'], assignments=(10, 0, 8, 9), order=10, porder=6), rng)
        case = fc.FlacCase(name, flac, st, 48000, 16, infos, offsets, 12000, 'uint8')
        mkv = str(tmp_path / (name + '.mkv'))
        mc.pair_mkv(mkv, case, head, events, chapters, int(dur * 24), seed)
        (tmp_path / 'cache').mkdir(exist_ok=True)
        (tmp_path / 'cache' / (name + '.mkv.sushi.keyframes.txt')).write_text(kf)
        with mk.MatroskaFile(mkv) as f:
            tc = tmp_path / (name + '.tc.txt')
            tc.write_text(f.timecodes_text())
        out[name] = (mkv, case.write_wav(tmp_path), str(tc))
    (tmp_path / 'kf.txt').write_text(kf)
    lines = list(head) + ['Dialogue: %s,%s,%s,%s' % (e[3].split(',')[1], format_time(e[1] / 100.0),
                                                     format_time(e[2] / 100.0), ','.join(e[3].split(',')[2:]))
                          for e in events]
    (tmp_path / 'in.ass').write_text('\n'.join(lines) + '\n', encoding='utf-8')
    (tmp_path / 'ch.txt').write_text(''.join('CHAPTER%02d=%s\nCHAPTER%02dNAME=\n' % (
        k + 1, format_srt_time(c / 1e9).replace(',', '.'), k + 1) for k, c in enumerate(chapters)))
    return out


def test_command_line_on_mkv_equals_wav(gpu_lib, tmp_path):
    p = _pair(tmp_path)
    cmd = [sys.executable, '-m', 'sushi_b200']
    mkv_out, wav_out = str(tmp_path / 'mkv.ass'), str(tmp_path / 'wav.ass')
    r = subprocess.run(cmd + ['--src', p['src'][0], '--dst', p['dst'][0], '-o', mkv_out, '--src-keyframes', 'auto',
                              '--dst-keyframes', 'auto', '--temp-dir', str(tmp_path / 'cache')],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run(cmd + ['--src', p['src'][1], '--dst', p['dst'][1], '-o', wav_out, '--script',
                              str(tmp_path / 'in.ass'), '--chapters', str(tmp_path / 'ch.txt'),
                              '--src-timecodes', p['src'][2], '--dst-timecodes', p['dst'][2],
                              '--src-keyframes', str(tmp_path / 'kf.txt'), '--dst-keyframes', str(tmp_path / 'kf.txt')],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert open(mkv_out, 'rb').read() == open(wav_out, 'rb').read()
    assert sorted(os.listdir(tmp_path / 'cache')) == ['dst.mkv.sushi.keyframes.txt', 'src.mkv.sushi.keyframes.txt']


def test_baseline_size_mkv_equals_pcm(gpu_lib, tmp_path):
    """90 minutes of 48 kHz stereo FLAC (63 282 frames, about 1 GB) beside 129 600 video frames."""
    path = str(tmp_path / 'baseline.mkv')
    pcm = mc.baseline_mkv(path)
    assert os.path.getsize(path) > 10 ** 9
    got = WavStream(path, 12000, 'uint8')
    want = WavStream.from_pcm(pcm, 48000, 12000, 'uint8', channels=2)
    assert_same_stream(got, want)
