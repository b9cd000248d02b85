"""MP4 / QuickTime and A_ALAC Matroska inputs on the GPU: every audio track loads bit for bit as the plain PCM WAV of
the samples FFmpeg's decoder returns (tests/test_mp4_cases.py and tests/test_alac_cases.py hold FFmpeg to the
writers' PCM): ALAC through sb_alac_decode_frames, FLAC through sb_flac_decode_frames, PCM through sb_load_pcm or sb_pcm_from_be.
Also 90 minutes of 24-bit stereo ALAC, the sparse file past 4 GiB, damaged frames named by frame and offset, and the
command line against the WAV pair."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, mp4, synth
from sushi_b200.common import py2_round
from sushi_b200.wavstream import WavStream
from tests import alac_cases as ac
from tests import flac_cases as fc
from tests import mkv_alac_cases as mac
from tests import mkv_cases as mc
from tests import mp4_cases as m
from tests import ts_cases as tsc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRACKS = [(c, sid) for c in m.good_cases() for sid in c.audio_ids()]


def _want(tmp_path, t, stype):
    """WavStream of the plain 16-bit WAV of the track's samples (their top 16 bits: what a 20-, 24- or 32-bit WAV
    loads as)."""
    return WavStream(tsc.write_wav(tmp_path / 'w.wav', ac.to16(t.pcm, t.bits), t.rate), 12000, stype)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', TRACKS, ids=lambda p: '%s-%d' % (p[0].name, p[1]))
def test_track_loads_as_the_wav_of_its_pcm(gpu_lib, tmp_path, pair, stype):
    case, sid = pair
    t = case.traks[sid]
    got = WavStream(case.write(tmp_path), 12000, stype, track=sid)
    if t.codec == 'flac':
        flac = tmp_path / 'a.flac'
        spec = mc.flac_track(9000, 2, 16, 44100, 1152, 10)
        flac.write_bytes(spec.private + b''.join(f for f, _, _ in spec.frames))
        assert_same_stream(got, WavStream(str(flac), 12000, stype))
    assert_same_stream(got, _want(tmp_path, t, stype))


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', mac.cases(), ids=lambda p: p[0].name)
def test_matroska_alac_track_loads_as_its_pcm(gpu_lib, tmp_path, pair, stype):
    mkv, case = pair
    got = WavStream(mkv.write(tmp_path), 12000, stype)
    assert_same_stream(got, WavStream.from_pcm(case.pcm16, case.rate, 12000, stype, channels=case.channels))


def test_opened_file_and_host_loader_for_pcm(gpu_lib, tmp_path):
    case = [c for c in m.good_cases() if c.name == 'mov_master'][0]
    path = case.write(tmp_path)
    with mp4.Mp4File(path) as f:
        for sid in (1, 3):                           # big-endian 16 and 24 bits
            gpu = WavStream(f, 8000, 'float32', track=sid)
            host = WavStream(f, 8000, 'float32', track=sid, loader='host')
            assert_same_stream(gpu, host)
    alac = [c for c in m.good_cases() if c.name == 'm4a_alac'][0].write(tmp_path)
    with pytest.raises(SushiError, match="needs loader='gpu'"):
        WavStream(alac, loader='host')


def test_ninety_minutes_of_24_bit_stereo_alac_equals_from_pcm(gpu_lib, tmp_path):
    cfg, frames, pcm, reps = ac.long_stream()
    case = ac.AlacCase('long', cfg, frames * reps, pcm, set())          # pcm, pcm16: one period
    path = str(tmp_path / 'long.m4a')
    with open(path, 'wb') as f:
        f.write(m.build('long', [m.alac_trak(case, per_chunk=(64,), edits=None)], ftyp=b'M4A '))
    del case.data
    assert os.path.getsize(path) * 8 > 2 ** 32
    got = WavStream(path, 12000, 'uint8')
    want = WavStream.from_pcm(np.tile(case.pcm16, (reps, 1)), 48000, 12000, 'uint8', channels=2)
    assert got.sample_count == want.sample_count
    assert_same_stream(got, want)


def test_sparse_file_loads(gpu_lib, tmp_path):
    path = str(tmp_path / 'sparse.m4a')
    case = m.sparse_file(path)
    assert_same_stream(WavStream(path, 12000, 'float32'),
                       WavStream.from_pcm(case.pcm16, case.rate, 12000, 'float32', channels=case.channels))


@pytest.mark.parametrize('damaged', ac.damaged_cases()[1], ids=lambda d: d[0])
def test_damaged_frame_is_refused_naming_frame_and_offset(gpu_lib, tmp_path, damaged):
    name, cfg, frames, f, regex = damaged
    case = ac.AlacCase(name, cfg, frames, np.zeros((0, cfg.channels), np.int64), set())
    t = m.alac_trak(case, per_chunk=(2,), edits=None)
    t.durations = [cfg.frame_length] * len(frames)
    path = str(tmp_path / (name + '.m4a'))
    with open(path, 'wb') as fh:
        fh.write(m.build(name, [t]))
    with mp4.Mp4File(path) as mf:
        where = int(mf.frames(mf.select('audio', None)).block[f])
    with pytest.raises(SushiError, match=regex) as e:
        WavStream(path, 12000, 'uint8')
    assert 'ALAC frame %d at byte offset %d:' % (f, where) in str(e.value), str(e.value)


def test_command_line_on_m4a_equals_wav(gpu_lib, tmp_path):
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
    up = np.repeat(src12, 4).astype(np.int64)
    st = np.stack([up, up // 2], 1)
    case = ac.escape_stream(st, ac.Config(frame_length=4096, bit_depth=16, channels=2))
    src_m4a = str(tmp_path / 'src.m4a')
    with open(src_m4a, 'wb') as f:
        f.write(m.build('src', [m.alac_trak(case, per_chunk=(8,), edits=None)], ftyp=b'M4A '))
    src_wav = tsc.write_wav(tmp_path / 'src.wav', st.astype(np.int16), 48000)
    up = np.repeat(dst12, 4).astype(np.int64)
    st = np.stack([up, up // 2], 1)
    flac, _, _ = fc.encode(st, 48000, 16, fc.fixed_blocks(len(st), 4096),
                           fc.stereo_plan(['lpc'], assignments=(10, 0, 8, 9), order=10, porder=6), rng)
    dst_flac = tmp_path / 'dst.flac'
    dst_flac.write_bytes(flac)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', st.astype(np.int16), 48000)
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    outs = []
    for a, b, name in ((src_m4a, str(dst_flac), 'm4a.ass'), (src_wav, dst_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', b, '-o', outs[-1]], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
    assert not os.path.exists(src_m4a + '.sushi.chapters.txt')
