"""Keyframe snapping end to end on the GPU: the command line on WAV inputs against the reference's
own run() sequence (tests/golden/keyframes.npz, part b, from oracle/gen_golden_keyframes.py).
The scenarios were generated so that moving any search group's shift by one sample or its diff by
1e-5 moves no final time by more than one sample: within the matcher's tolerance no grouping or
snapping decision flips, so every final time must be within 1/12000 s of the reference's."""
import ast
import os
import wave
import zlib

import numpy as np
import pytest

from sushi_b200 import cli, load_keyframe_times, load_script, shift_script, shift_scripts, synth
from sushi_b200.common import format_time
from sushi_b200.script import format_srt_time, parse_ass_time

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'keyframes.npz'))
TOL = 1.0 / 12000 + 1e-9
NAMES = bytes(GOLDEN['b_names']).decode().split(',')


def text(key):
    return bytes(GOLDEN[key]).decode('utf-8')


def write_inputs(name, tmp_path):
    """WAVs regenerated from the seed (CRC-checked) and the stored script / side files; returns (spec, paths)."""
    p = 'b_{0}_'.format(name)
    spec = ast.literal_eval(text(p + 'spec'))
    shift = spec['shift'] if len(spec['shift']) > 1 else spec['shift'][0][1]
    src_pcm, dst_pcm = synth.make_pair(spec['dur'], spec['seed'], shift)
    assert [zlib.crc32(src_pcm.tobytes()), zlib.crc32(dst_pcm.tobytes())] == list(GOLDEN[p + 'pcm_crc'])
    paths = {}
    for key, pcm in (('src', src_pcm), ('dst', dst_pcm)):
        paths[key] = str(tmp_path / (name + '_' + key + '.wav'))
        with wave.open(paths[key], 'wb') as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(12000); w.writeframes(pcm.tobytes())
    for key, ext in (('script', spec['script']), ('src_kf', '.txt'), ('dst_kf', '.txt'), ('src_tc', '.txt'),
                     ('dst_tc', '.txt'), ('chapters', '.xml')):
        if p + key in GOLDEN:
            paths[key] = str(tmp_path / (name + '_' + key + ext))
            with open(paths[key], 'w') as f:
                f.write(text(p + key))
    paths['out'] = str(tmp_path / (name + '_out' + spec['script']))
    return spec, paths


def cli_args(spec, paths, stype, keyframes=True):
    args = ['--src', paths['src'], '--dst', paths['dst'], '--script', paths['script'], '-o', paths['out'],
            '--sample-type', stype, '--kf-mode', spec['kf_mode']]
    if 'chapters' in paths:
        args += ['--chapters', paths['chapters']]
    if not spec['grouping']:
        args += ['--no-grouping']
    if keyframes:
        args += ['--src-keyframes', paths['src_kf'], '--dst-keyframes', paths['dst_kf']]
        for side in ('src', 'dst'):
            if spec[side][0] == 'fps':
                args += ['--{0}-fps'.format(side), repr(spec[side][1])]
            else:
                args += ['--{0}-timecodes'.format(side), paths[side + '_tc']]
    return args


def run_cli(monkeypatch, args):
    """cli.main in-process; returns the script object its shift_script call produced."""
    seen = []

    def recording(*a, **k):
        seen.append(shift_script(*a, **k))
        return seen[-1]
    monkeypatch.setattr(cli, 'shift_script', recording)
    assert cli.main(args) == 0
    (script, _), = seen
    return script


def times(script):
    return {e.source_index: (e.start, e.end) for e in script.events}


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
@pytest.mark.parametrize('name', NAMES)
def test_cli_with_keyframes_matches_reference(gpu_lib, monkeypatch, tmp_path, name, stype):
    spec, paths = write_inputs(name, tmp_path)
    script = run_cli(monkeypatch, cli_args(spec, paths, stype))
    got = times(script)
    p = 'b_{0}_{1}_'.format(name, stype)
    want = GOLDEN[p + 'times']
    assert sorted(got) == sorted(GOLDEN[p + 'index'].tolist())
    err = max(max(abs(got[i][0] - a), abs(got[i][1] - b)) for i, (a, b) in zip(GOLDEN[p + 'index'], want))
    assert err <= TOL, err
    # the written file holds those times as the writer rounds them
    fmt = format_time if spec['script'] == '.ass' else format_srt_time
    parse = parse_ass_time if spec['script'] == '.ass' else (lambda s: parse_ass_time(s.replace(',', '.')))
    written = times(load_script(paths['out']))
    assert written == {i: (parse(fmt(a)), parse(fmt(b))) for i, (a, b) in got.items()}


@pytest.mark.parametrize('stype', ['uint8', 'float32'])
def test_cli_without_keyframes_equals_shift_script(gpu_lib, monkeypatch, tmp_path, stype):
    spec, paths = write_inputs('chapter_jump', tmp_path)
    via_cli = times(run_cli(monkeypatch, cli_args(spec, paths, stype, keyframes=False)))
    from sushi_b200.timing import get_xml_start_times
    script, _ = shift_script(paths['src'], paths['dst'], paths['script'], str(tmp_path / 'direct.ass'),
                             sample_type=stype, chapter_times=get_xml_start_times(paths['chapters']),
                             kf_mode=spec['kf_mode'])
    assert via_cli == times(script)


def test_shift_scripts_with_per_job_keyframes_equals_per_job_runs(gpu_lib, tmp_path):
    jobs = []
    for name in NAMES:
        spec, paths = write_inputs(name, tmp_path)
        side = {}
        for s in ('src', 'dst'):
            side[s + ('_fps' if spec[s][0] == 'fps' else '_timecodes')] = spec[s][1] if spec[s][0] == 'fps' else paths[s + '_tc']
        kt = load_keyframe_times(paths['src_kf'], paths['dst_kf'], **side)
        chapters = [0.0, 40.0] if 'chapters' in paths else []
        jobs.append((paths['src'], paths['dst'], paths['script'], paths['out'], chapters, kt))
    together = shift_scripts(jobs)
    for job, (script, groups) in zip(jobs, together):
        alone, alone_groups = shift_script(*job[:3], job[3] + '.alone' + os.path.splitext(job[3])[1],
                                           chapter_times=job[4], keyframes=job[5])
        assert [(e.source_index, e.start, e.end) for e in script.events] == \
            [(e.source_index, e.start, e.end) for e in alone.events]
        assert len(groups) == len(alone_groups)
    # and the keyframes did something: the same jobs without them end elsewhere
    plain = shift_scripts([j[:5] for j in jobs])
    assert any(times(a) != times(b) for (a, _), (b, _) in zip(together, plain))
