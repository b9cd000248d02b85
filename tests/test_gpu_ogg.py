"""Ogg FLAC on the GPU: every stream of every good case of tests/ogg_cases.py loads bit for bit as the WAV of FFmpeg's
decode, in both sample types, and again with chunks small enough to split capture patterns, page headers and packets;
--ffmpeg-audio equals libswresample on FFmpeg's decode and layout; damaged copies are refused with the CPU build's
message and cut copies load as FFmpeg decodes them, at the default chunk size and at small ones; the command line on
an .oga source writes what it writes for the WAV of the same audio."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sushi_b200 import SushiError, ogg
from sushi_b200.wavstream import WavStream
from tests import flac_cases as fc
from tests import ogg_cases as oc
from tests import ref_mp4
from tests import ref_swr
from tests import ts_cases as tsc
from tests.test_gpu_flac import assert_same_stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOOD = oc.good_cases()


def _pairs():
    return [(c, k) for c in GOOD for k in range(len(c.streams))]


def _ffmpeg_wav(tmp_path, path, k, stream):
    """the WAV of FFmpeg's decode of stream k, at the stream's bit depth"""
    pcm, refused = ref_mp4.decode_pcm(path, k, stream.case.channels, stream.case.bits)
    assert refused == 0 and np.array_equal(pcm, stream.case.pcm)
    return stream.case.write_wav(tmp_path)


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('pair', _pairs(), ids=lambda p: '%s_%d' % (p[0].name, p[1]))
def test_ogg_flac_loads_as_ffmpegs_decode(gpu_lib, tmp_path, pair, stype):
    case, k = pair
    path = case.write(tmp_path)
    want = WavStream(_ffmpeg_wav(tmp_path, path, k, case.streams[k]), 12000, stype)
    assert_same_stream(WavStream(ogg.OggFile(path), 12000, stype, track=k), want)


@pytest.mark.parametrize('pair', _pairs(), ids=lambda p: '%s_%d' % (p[0].name, p[1]))
def test_small_chunks_split_pages(gpu_lib, tmp_path, monkeypatch, pair):
    """every stream at chunks that split capture patterns, page headers, lacing values and packets"""
    case, k = pair
    path = case.write(tmp_path)
    want = WavStream(_ffmpeg_wav(tmp_path, path, k, case.streams[k]), 12000, 'uint8')
    for chunk in (5, 28, 777, 4096):
        monkeypatch.setattr(ogg, 'CHUNK_BYTES', chunk)
        assert_same_stream(WavStream(path, 12000, 'uint8', track=k), want)


@pytest.mark.parametrize('name', ['ch2_16', 'ch6_16'])
def test_ffmpeg_audio_equals_libswresample_on_ffmpegs_decode(gpu_lib, tmp_path, name):
    path = next(c for c in GOOD if c.name == name).write(tmp_path)
    pcm, mask, rate = ref_mp4.decode_s16(path, 0)
    mono = ref_swr.convert(pcm, mask, rate, 12000)
    want = WavStream(tsc.write_wav(tmp_path / 'swr.wav', mono.reshape(-1, 1), 12000), 12000, 'float32')
    assert_same_stream(WavStream(path, 12000, 'float32', ffmpeg_audio=True), want)


def test_ffmpeg_audio_refuses_24_bit(gpu_lib, tmp_path):
    path = next(c for c in GOOD if c.name == 'count0').write(tmp_path)
    with pytest.raises(SushiError, match='S32'):
        WavStream(path, 12000, 'float32', ffmpeg_audio=True)


@pytest.mark.parametrize('case', oc.damaged_cases(), ids=lambda c: c.name)
def test_damaged_copy_is_refused_with_the_cpu_builds_message(gpu_lib, tmp_path, monkeypatch, case):
    path = case.write(tmp_path)
    for chunk in (ogg.CHUNK_BYTES, 4096, 777, 28):
        monkeypatch.setattr(ogg, 'CHUNK_BYTES', chunk)
        with pytest.raises(SushiError, match='Ogg page at byte offset %d: .*%s' % (case.offset, case.regex)):
            WavStream(ogg.OggFile(path), 12000, 'uint8', track=0)


@pytest.mark.parametrize('name,data,serial', oc.cut_cases(), ids=lambda v: v if isinstance(v, str) else '')
def test_cut_copy_loads_as_ffmpeg_decodes_it(gpu_lib, tmp_path, monkeypatch, name, data, serial):
    path = str(tmp_path / (name + '.oga'))
    with open(path, 'wb') as f:
        f.write(data)
    pcm, _, rate = ref_mp4.decode_s16(path, 0)
    want = WavStream(tsc.write_wav(tmp_path / 'ffmpeg.wav', pcm, rate), 12000, 'uint8')
    for chunk in (ogg.CHUNK_BYTES, 777, 28):
        monkeypatch.setattr(ogg, 'CHUNK_BYTES', chunk)
        assert_same_stream(WavStream(ogg.OggFile(path), 12000, 'uint8', track=0), want)


def test_command_line_on_an_ogg_source_equals_wav(gpu_lib, tmp_path):
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
    rng = np.random.default_rng([oc.SEED, seed])
    frames = int(dur * 48000)
    pcm = fc.make_pcm('programme', frames, 2, 16, 48000, rng)
    blocks = fc.fixed_blocks(frames, 4096)
    flac, infos, offsets = fc.encode(pcm, 48000, 16, blocks, fc.uniform_plan(2, kind='fixed', order=2), rng)
    flac_case = fc.FlacCase('capture', flac, pcm, 48000, 16, infos, offsets, 12000, 'uint8')
    case = oc.make('capture', [(0x5EED, flac_case, [], None, 'mixed')], seed)
    src = case.write(tmp_path)
    src_wav = flac_case.write_wav(tmp_path)
    pcm16, _, _ = ref_mp4.decode_s16(src, 0)
    assert np.array_equal(pcm16, pcm)
    dst_wav = tsc.write_wav(tmp_path / 'dst.wav', pcm16, 48000)
    cmd = [sys.executable, '-m', 'sushi_b200', '--script', str(tmp_path / 'in.ass')]
    outs = []
    for a, name in ((src, 'ogg.ass'), (src_wav, 'wav.ass')):
        outs.append(str(tmp_path / name))
        r = subprocess.run(cmd + ['--src', a, '--dst', dst_wav, '-o', outs[-1]], cwd=ROOT, capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr
    assert open(outs[0], 'rb').read() == open(outs[1], 'rb').read()
