"""The command line's refusals on MP4 / QuickTime inputs, all before the GPU is touched: AAC named with its track,
a fragmented file, an edit list, a mov_text script ("Unknown script type"), no subtitle stream, keyframes without fps
or timecodes, and a name that does not open as MP4.  Also the OGM chapters file an MP4 source gives, written at the
reference's path and kept with --no-cleanup."""
import os

import pytest

from sushi_b200 import cli
from sushi_b200.common import SushiError
from tests import mp4_cases as m


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def files(tmp_path):
    good = {c.name: c.write(tmp_path) for c in m.good_cases()}
    refused = {c.name: c.write(tmp_path) for c, _ in m.refused_cases()}
    (tmp_path / 'in.ass').write_text('[Script Info]\n')
    (tmp_path / 'kf.txt').write_text('# XviD 2pass stat file\n\n\ni\n')
    out = dict(good, **refused)
    out['script'] = str(tmp_path / 'in.ass')
    out['kf'] = str(tmp_path / 'kf.txt')
    return out


def test_refusals(files, tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    s = files['script']
    dst = files['m4a_alac']
    with pytest.raises(SushiError, match=r'Audio track 0 is aac, which cannot be decoded here'):
        run(['--src', files['mp4_aac'], '--dst', dst, '--script', s, '--src-audio', '0'])
    mov = tmp_path / 'aac.mov'
    mov.write_bytes(open(files['aac_only'], 'rb').read())
    with pytest.raises(SushiError, match=r'Audio track 0 is aac'):
        run(['--src', str(mov), '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='fragmented MP4 files are not supported'):
        run(['--src', files['fragmented'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='track 0 has an edit list'):
        run(['--src', files['edit_shift'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='^Unknown script type$'):
        run(['--src', files['mov_master'], '--dst', dst, '--src-audio', '2'])
    with pytest.raises(SushiError, match='No subtitles streams found in'):
        run(['--src', files['m4a_alac'], '--dst', dst])
    with pytest.raises(SushiError, match='m4a_alac.m4a: video timestamps cannot be read from an MP4 file'):
        run(['--src', files['m4a_alac'], '--dst', files['mov_alac24'], '--script', s, '--dst-audio', '0',
             '--src-keyframes', files['kf'], '--dst-keyframes', files['kf']])
    with pytest.raises(SushiError, match='making keyframes .SCXvid. is not supported'):
        run(['--src', files['mov_master'], '--dst', dst, '--script', s, '--src-audio', '2',
             '--src-keyframes', 'make', '--dst-keyframes', 'make'])
    bad = tmp_path / 'x.mp4'
    bad.write_bytes(b'\1' * 1000)
    with pytest.raises(SushiError, match='demuxing is not supported, convert the input to WAV or FLAC first '
                                         r'\(it does not open as an MP4 file: .*not an MP4'):
        run(['--src', str(bad), '--dst', dst, '--script', s])


def test_chapters_file_and_selected_tracks(files, monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, 'shift_script', lambda src, dst, *a, **kw: seen.update(kw, src=src, dst=dst))
    run(['--src', files['mov_master'], '--dst', files['m4a_alac'], '--script', files['script'], '--src-audio', '3',
         '--no-cleanup'])
    assert seen['src_track'] == 3 and seen['dst_track'] == 0
    assert seen['chapter_times'] == [0.0, 1.5, 4.0, 9.0]
    path = files['mov_master'] + '.sushi.chapters.txt'
    assert open(path).read() == ('CHAPTER01=00:00:00.000\nCHAPTER01NAME=\nCHAPTER02=00:00:01.500\nCHAPTER02NAME=\n'
                                 'CHAPTER03=00:00:04.000\nCHAPTER03NAME=\nCHAPTER04=00:00:09.000\nCHAPTER04NAME=\n')
    os.remove(path)
    run(['--src', files['mov_master'], '--dst', files['m4a_alac'], '--script', files['script'], '--src-audio', '3'])
    assert not os.path.exists(path)
