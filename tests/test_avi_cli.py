"""The command line's refusals on AVI inputs, all before the GPU is touched: lossy and other refused audio named by
FFmpeg's codec name, several audio streams without --src-audio, a GAB2 subtitle stream as the script, keyframes
without fps or timecodes, `make` keyframes, a name that does not open as an AVI file.  Also the streams it selects."""
import pytest

from sushi_b200 import cli
from sushi_b200.common import SushiError
from tests import avi_cases as ac


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def files(tmp_path):
    good = {c.name: c for c in ac.good_cases()}
    out = {name: good[name].write(tmp_path) for name in ('pcm16_every_frame', 'two_audio_preload', 'mp2_cbr_subs')}
    for case, _, _ in ac.refused_cases():
        out[case.name] = case.write(tmp_path)
    (tmp_path / 'in.ass').write_text('[Script Info]\n')
    (tmp_path / 'kf.txt').write_text('# XviD 2pass stat file\n\n\ni\n')
    out['script'] = str(tmp_path / 'in.ass')
    out['kf'] = str(tmp_path / 'kf.txt')
    return out


def test_refusals(files, tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    s, dst = files['script'], files['pcm16_every_frame']
    for case, sid, regex in ac.refused_cases():
        with pytest.raises(SushiError, match=r'Audio track {0} {1}, which cannot be decoded here'.format(sid, regex)):
            run(['--src', files[case.name], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='More than one audio stream found'):
        run(['--src', files['two_audio_preload'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='^Unknown script type$'):
        run(['--src', files['mp2_cbr_subs'], '--dst', dst])
    with pytest.raises(SushiError, match='No subtitles streams found in'):
        run(['--src', dst, '--dst', files['mp2_cbr_subs']])
    with pytest.raises(SushiError, match='pcm16_every_frame.avi: video timestamps cannot be read from an AVI file'):
        run(['--src', dst, '--dst', files['mp2_cbr_subs'], '--script', s, '--src-keyframes', files['kf'],
             '--dst-keyframes', files['kf']])
    with pytest.raises(SushiError, match='making keyframes \\(SCXvid\\) is not supported'):
        run(['--src', dst, '--dst', files['mp2_cbr_subs'], '--script', s, '--src-keyframes', 'make',
             '--dst-keyframes', 'make', '--src-fps', '25', '--dst-fps', '25'])
    bad = tmp_path / 'x.avi'
    bad.write_bytes(b'RIFF\x04\x00\x00\x00WAVE' + bytes(100))
    with pytest.raises(SushiError, match='demuxing is not supported.*does not open as an AVI file.*not an AVI file'):
        run(['--src', str(bad), '--dst', dst, '--script', s])


def test_selected_streams_reach_shift_script(files, monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, 'shift_script', lambda src, dst, *a, **kw: seen.update(kw, src=src, dst=dst))
    run(['--src', files['two_audio_preload'], '--dst', files['mp2_cbr_subs'], '--script', files['script'],
         '--src-audio', '2', '--src-fps', '25', '--dst-fps', '25'])
    assert seen['src_track'] == 2 and seen['dst_track'] == 1 and seen['chapter_times'] == []
