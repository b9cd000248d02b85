"""The WAV-input command line (sushi_b200.cli): flags and the validation of the reference's run()
(sushi.py:528-651), port of its MainScriptTestCase (tests/main.py:184-218) plus the WAV-specific errors.
Every case here fails before the GPU is touched, so they all pass on a machine without one."""
import os
import subprocess
import sys

import pytest

from sushi_b200 import cli
from sushi_b200.common import SushiError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def checked(monkeypatch):
    """The reference's tests patch check_file_exists: record the calls, let every file 'exist'."""
    calls = []
    monkeypatch.setattr(cli, 'check_file_exists', lambda path, title: calls.append((path, title)))
    return calls


@pytest.fixture
def no_gpu_run(monkeypatch):
    """Anything that gets past validation ends in shift_script: record its arguments instead."""
    runs = []
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **k: runs.append((a, k)))
    return runs


def run(keys):
    return cli.run(cli.create_arg_parser().parse_args(keys))


# tests/main.py: MainScriptTestCase
def test_checks_that_files_exist(checked):
    keys = ['--dst', 'dst', '--src', 'src', '--script', 'script', '--chapters', 'chapters',
            '--dst-keyframes', 'dst-keyframes', '--src-keyframes', 'src-keyframes',
            '--src-timecodes', 'src-tcs', '--dst-timecodes', 'dst-tcs']
    with pytest.raises(SushiError):
        run(keys)
    paths = [p for p, _ in checked]
    for p in ('src', 'dst', 'script', 'chapters', 'dst-keyframes', 'src-keyframes', 'dst-tcs', 'src-tcs'):
        assert p in paths


def test_raises_on_unknown_script_type(checked):
    with pytest.raises(SushiError, match='(?i)script.*type'):
        run(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.mp4'])


def test_raises_on_script_type_not_matching(checked):
    with pytest.raises(SushiError, match='(?i)script.*type.*match'):
        run(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.ass', '-o', 'd.srt'])


def test_raises_on_timecodes_and_fps_being_defined_together(checked):
    with pytest.raises(SushiError, match='(?i)timecodes'):
        run(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.ass', '--src-timecodes', 'tc.txt', '--src-fps', '25'])


# real files: the existence checks themselves
def test_missing_file_is_reported():
    with pytest.raises(SushiError, match="Source file doesn't exist"):
        run(['--src', '/nonexistent/s.wav', '--dst', 'd.wav', '--script', 's.ass'])


def test_missing_destination_timecodes_keeps_the_reference_title(tmp_path):
    for n in ('s.wav', 'd.wav', 's.ass'):
        (tmp_path / n).write_bytes(b'')
    with pytest.raises(SushiError, match="Source timecodes file doesn't exist"):
        run(['--src', str(tmp_path / 's.wav'), '--dst', str(tmp_path / 'd.wav'), '--script', str(tmp_path / 's.ass'),
             '--dst-timecodes', str(tmp_path / 'none.txt')])


# WAV-specific errors
@pytest.mark.parametrize('src,dst', [('s.mkv', 'd.wav'), ('s.wav', 'd.mp4')])
def test_non_wav_input_needs_converting(checked, src, dst):
    with pytest.raises(SushiError, match='demuxing is not supported.*WAV'):
        run(['--src', src, '--dst', dst, '--script', 's.ass'])


def test_script_is_required_for_wav_input(checked):
    with pytest.raises(SushiError, match="Script file isn't specified"):
        run(['--src', 's.wav', '--dst', 'd.wav'])


@pytest.mark.parametrize('side', ['--src-keyframes', '--dst-keyframes'])
def test_keyframes_on_one_side_only(checked, side):
    with pytest.raises(SushiError, match='Either none or both of src and dst keyframes'):
        run(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.ass', side, 'kf.txt'])


def test_keyframes_without_fps_or_timecodes(checked):
    with pytest.raises(SushiError, match='Fps, timecodes or video files must be provided if keyframes are used'):
        run(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.ass', '--src-keyframes', 'a.txt',
             '--dst-keyframes', 'b.txt', '--src-fps', '23.976'])


@pytest.mark.parametrize('mode', ['auto', 'make'])
def test_keyframes_cannot_be_made_from_wav(checked, tmp_path, mode):
    src = str(tmp_path / 's.wav')
    with pytest.raises(SushiError, match=r"Cannot make keyframes for .*s\.wav because it doesn't have any video!"):
        run(['--src', src, '--dst', 'd.wav', '--script', 's.ass', '--src-keyframes', mode, '--dst-keyframes', mode,
             '--src-fps', '25', '--dst-fps', '25'])


def test_auto_keyframes_reuse_a_cached_file(checked, no_gpu_run, tmp_path):
    kf = ('# XviD 2pass stat file\n\n\n' + 'p\n' * 25 + 'i\n' + 'p\n' * 10)
    (tmp_path / 'cache').mkdir()
    (tmp_path / 'cache' / 's.wav.sushi.keyframes.txt').write_text(kf)
    (tmp_path / 'cache' / 'd.wav.sushi.keyframes.txt').write_text(kf)
    run(['--src', str(tmp_path / 'in' / 's.wav'), '--dst', str(tmp_path / 'd.wav'), '--script', 's.ass',
         '--src-keyframes', 'auto', '--dst-keyframes', 'auto', '--src-fps', '25', '--dst-fps', '25',
         '--temp-dir', str(tmp_path / 'cache')])
    (args, kwargs), = no_gpu_run
    assert kwargs['keyframes'].src_keytimes == [0, 1.0] and kwargs['keyframes'].dst_keytimes == [0, 1.0]
    # the temp dir is where the default output goes
    assert args[3] == str(tmp_path / 'cache' / 'd.wav.sushi.ass')


def test_defaults_reach_shift_script(checked, no_gpu_run):
    run(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.srt'])
    (args, kwargs), = no_gpu_run
    assert args == ('s.wav', 'd.wav', 's.srt', 'd.wav.sushi.srt')
    assert kwargs == dict(sample_rate=12000, sample_type='uint8', chapter_times=[], window=10, max_window=30,
                          rewind_thresh=5, grouping=True, smooth_radius=3, max_ts_duration=1001.0 / 24000.0 * 10,
                          max_ts_distance=1001.0 / 24000.0 * 10, keyframes=None, max_kf_distance=2, kf_mode='all')


OGM = 'CHAPTER01=00:00:00.000\nCHAPTER02=00:00:17.017\n'


def test_chapters_files(checked, no_gpu_run, tmp_path):
    (tmp_path / 'c.txt').write_text(OGM)
    (tmp_path / 'c.xml').write_text('<ChapterTimeStart>00:00:05.500000000</ChapterTimeStart>')
    base = ['--src', 's.wav', '--dst', 'd.wav', '--script', 's.ass', '-o', 'o.ass']
    run(base + ['--chapters', str(tmp_path / 'c.txt')])
    run(base + ['--chapters', str(tmp_path / 'c.xml')])
    run(base + ['--chapters', 'none'])
    run(base + ['--chapters', 'NONE', '--no-grouping'])
    run(base + ['--chapters', str(tmp_path / 'c.txt'), '--no-grouping'])
    assert [k['chapter_times'] for _, k in no_gpu_run] == [[0, 17.017], [0, 5.5], [], [], []]
    assert [p for p, _ in checked].count('none') == 0               # 'none' is not a file to check


def test_main_logs_the_error_and_returns_2(checked, caplog):
    assert cli.main(['--src', 's.wav', '--dst', 'd.wav', '--script', 's.ass', '--src-keyframes', 'kf.txt']) == 2
    assert any(r.levelname == 'CRITICAL' and 'keyframes' in r.getMessage() for r in caplog.records)


def test_module_entry_point_exits_2():
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, '-m', 'sushi_b200', '--src', 'missing.wav', '--dst', 'd.wav', '--script', 's.ass'],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=120)
    assert p.returncode == 2, p.stderr
    assert "Source file doesn't exist" in p.stderr


def test_test_shift_plot_is_not_offered():
    with pytest.raises(SystemExit):
        cli.create_arg_parser().parse_args(['--src', 's.wav', '--dst', 'd.wav', '--test-shift-plot', 'p.png'])
