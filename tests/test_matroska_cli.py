"""The command line on Matroska inputs, up to the shift_script call (no GPU): audio track selection (the default
rule, the ambiguous list, an unknown id), the refusal of codecs the GPU loader does not decode, the script, chapters
and timecodes taken out of the inputs and handed to shift_script, the files written for them and their cleanup, and
the refusal to make keyframes.  Uses the `checked` fixture of tests/test_cli.py; `seen` stands in for its
`no_gpu_run` and also records the text of the extracted script at the time of the call."""
import os

import pytest

from sushi_b200 import cli
from sushi_b200 import matroska as mk
from sushi_b200.common import SushiError
from tests import mkv_cases as mc
from tests.test_cli import checked, run  # noqa: F401  (a fixture)

CASES = {c.name: c for c in mc.all_cases()}
KF = '# XviD 2pass stat file\n\n\n' + 'p\n' * 5 + 'i\n' + 'p\n' * 40 + 'i\n' + 'p\n' * 10


@pytest.fixture
def files(tmp_path):
    return {name: c.write(tmp_path) for name, c in CASES.items()}


@pytest.fixture
def seen(monkeypatch):
    """shift_script's arguments (an opened Matroska input as its path) and, at the time of the call, the text of
    the script it is handed.  The audio tables WavStream would take are fetched too, counting the walks over the
    clusters."""
    calls = []
    walks = []
    real = mk.MatroskaFile.prefetch
    monkeypatch.setattr(mk.MatroskaFile, 'prefetch', lambda self, *a: (walks.append(self.path), real(self, *a))[1])

    def fake(*a, **k):
        texts = {p: open(p, encoding='utf-8').read() for p in a[2:3] if os.path.exists(p)}
        kf = k.get('keyframes')
        for m, key in ((a[0], 'src_track'), (a[1], 'dst_track')):
            if isinstance(m, mk.MatroskaFile):
                assert len(m.frames([k[key]])[k[key]]) > 0
        calls.append(((getattr(a[0], 'path', a[0]), getattr(a[1], 'path', a[1])) + a[2:], k, texts, kf, list(walks)))
    monkeypatch.setattr(cli, 'shift_script', fake)
    return calls


def test_default_audio_track_and_embedded_srt(checked, files, seen, tmp_path):
    run(['--src', files['multi'], '--dst', files['multi'], '-o', str(tmp_path / 'out.srt')])
    (args, kwargs, texts, _, _), = seen
    assert kwargs['src_track'] == 0 and kwargs['dst_track'] == 0        # FlagDefault absent counts as set
    assert args[2] == files['multi'] + '.sushi.srt'
    assert texts[args[2]].startswith('1\n00:00:')
    assert not os.path.exists(args[2])                                   # cleaned up
    assert kwargs['chapter_times'] == []


def test_audio_track_by_id(checked, files, seen, tmp_path):
    run(['--src', files['multi'], '--dst', files['multi'], '--src-audio', '2', '--dst-audio', '1',
         '-o', str(tmp_path / 'out.srt')])
    (_, kwargs, _, _, _), = seen
    assert (kwargs['src_track'], kwargs['dst_track']) == (2, 1)


def test_ambiguous_and_unknown_tracks(checked, files, seen):
    with pytest.raises(SushiError, match=r'More than one audio stream found in .*two_no_default\.mkv\.You need to '
                                         r'specify the exact one to demux\. Here are all candidates:\n0: A_PCM/INT/LIT'):
        run(['--src', files['multi'], '--dst', files['two_no_default'], '--script', 's.srt'])
    with pytest.raises(SushiError, match=r"Stream with index 7 doesn't exist in .*multi\.mkv\.\nHere are all that do:"):
        run(['--src', files['multi'], '--dst', files['multi'], '--dst-audio', '7', '--script', 's.srt'])
    assert seen == []


@pytest.mark.parametrize('name', ['refused_aac', 'refused_pcm_big', 'refused_encrypted', 'refused_bzlib'])
def test_lossy_or_unsupported_audio_is_refused(checked, files, seen, name):
    with pytest.raises(SushiError, match=CASES[name].refused):
        run(['--src', files[name], '--dst', files['multi'], '--script', 's.srt'])
    assert seen == []


def test_not_a_matroska_file_needs_converting(checked, tmp_path, seen):
    p = tmp_path / 'x.mkv'
    p.write_bytes(b'not EBML at all')
    with pytest.raises(SushiError, match=r'demuxing is not supported.*WAV.*not an EBML file'):
        run(['--src', str(p), '--dst', 'd.wav', '--script', 's.ass'])


def _main_run(files, tmp_path, extra):
    cache = tmp_path / 'cache'
    cache.mkdir()
    for side in ('src', 'dst'):
        (cache / ('%s.mkv.sushi.keyframes.txt' % side)).write_text(KF)
    src, dst = str(tmp_path / 'src.mkv'), str(tmp_path / 'dst.mkv')
    os.rename(files['main'], src)
    with open(dst, 'wb') as f:
        f.write(CASES['main'].data)
    run(['--src', src, '--dst', dst, '--src-keyframes', 'auto', '--dst-keyframes', 'auto', '--temp-dir', str(cache),
         '-o', str(tmp_path / 'out.ass')] + extra)
    return cache, src, dst


@pytest.mark.parametrize('cleanup', [True, False])
def test_script_chapters_and_timecodes_come_from_the_inputs(checked, files, seen, tmp_path, cleanup):
    cache, src, dst = _main_run(files, tmp_path, [] if cleanup else ['--no-cleanup'])
    (args, kwargs, texts, kf, walks), = seen
    assert walks == [src, dst]                      # one walk per input: audio, script and video times together
    case = CASES['main']
    script = str(cache / 'src.mkv.sushi.ass')
    assert args == (src, dst, script, str(tmp_path / 'out.ass'))
    assert texts[script].startswith('[Script Info]') and texts[script].count('Dialogue:') == len(case.script[1])
    assert kwargs['chapter_times'] == [float('%f' % (s / 1e9)) for s in case.chapters]
    video = sorted(t for _, t, _ in case.expect[0])
    assert kf.src_timecodes.times == [t / 1e9 for t in video] == kf.dst_timecodes.times
    assert kf.src_keytimes == [video[0] / 1e9, video[5] / 1e9, video[46] / 1e9]     # frame 0, then the i lines
    written = [script, str(cache / 'src.mkv.sushi.chapters.txt'), str(cache / 'src.mkv.sushi.timecodes.txt'),
               str(cache / 'dst.mkv.sushi.timecodes.txt')]
    assert [os.path.exists(p) for p in written] == [not cleanup] * 4
    assert os.path.exists(cache / 'src.mkv.sushi.keyframes.txt')         # inputs are never removed
    if not cleanup:
        assert open(written[1]).read().startswith('CHAPTER01=00:00:00.000\nCHAPTER01NAME=\nCHAPTER02=00:00:05.000\n')
        assert open(written[2]).read().startswith('# timestamp format v2\n0\n')


def test_explicit_files_win_over_the_inputs(checked, files, seen, tmp_path):
    (tmp_path / 'c.txt').write_text('CHAPTER01=00:00:00.000\nCHAPTER02=00:00:17.017\n')
    cache, src, dst = _main_run(files, tmp_path, ['--script', 's.ass', '--chapters', str(tmp_path / 'c.txt'),
                                                  '--src-fps', '25', '--dst-fps', '25'])
    (args, kwargs, _, kf, _), = seen
    assert args[2] == 's.ass' and kwargs['chapter_times'] == [0.0, 17.017]
    assert sorted(os.listdir(cache)) == ['dst.mkv.sushi.keyframes.txt', 'src.mkv.sushi.keyframes.txt']


@pytest.mark.parametrize('mode', ['make', 'auto'])
def test_making_keyframes_is_refused(checked, files, seen, tmp_path, mode):
    with pytest.raises(SushiError, match=r'Cannot make keyframes for .*main\.mkv: making keyframes \(SCXvid\) is not '
                                         r'supported'):
        run(['--src', files['main'], '--dst', files['main'], '--src-keyframes', mode, '--dst-keyframes', mode,
             '--temp-dir', str(tmp_path / 'empty')])
    # an input without video keeps the reference's message
    with pytest.raises(SushiError, match=r"Cannot make keyframes for .*multi\.mkv because it doesn't have any video!"):
        run(['--src', files['multi'], '--dst', files['multi'], '--src-keyframes', mode, '--dst-keyframes', mode,
             '--script', 's.srt'])
    assert seen == []
