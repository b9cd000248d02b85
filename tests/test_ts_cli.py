"""The command line's refusals on transport stream inputs, all before the GPU is touched: a lossy stream named by its
codec, several audio streams without --src-audio, a PGS-only script, keyframes without fps or timecodes, several
programs, a name that does not open as a transport stream.  Also the empty chapter file a transport stream source
gives, written at the reference's path and kept with --no-cleanup."""
import os

import pytest

from sushi_b200 import cli
from sushi_b200.common import SushiError
from tests import ts_cases as tsc


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def files(tmp_path):
    out = {name: tsc.case(name).write(tmp_path) for name in ('bd_lossy', 'bd_two_lpcm', 'bd_8ch24_48k', 'bd_two_programs',
                                                             'bd_stereo16_48k')}
    (tmp_path / 'in.ass').write_text('[Script Info]\n')
    (tmp_path / 'kf.txt').write_text('# XviD 2pass stat file\n\n\ni\n')
    out['script'] = str(tmp_path / 'in.ass')
    out['kf'] = str(tmp_path / 'kf.txt')
    return out


def test_refusals(files, tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    s = files['script']
    with pytest.raises(SushiError, match=r'Audio track 0 is ac3, which cannot be decoded here'):
        run(['--src', files['bd_lossy'], '--dst', files['bd_8ch24_48k'], '--script', s, '--src-audio', '0'])
    with pytest.raises(SushiError, match='More than one audio stream found'):
        run(['--src', files['bd_two_lpcm'], '--dst', files['bd_8ch24_48k'], '--script', s])
    with pytest.raises(SushiError, match='^Unknown script type$'):
        run(['--src', files['bd_stereo16_48k'], '--dst', files['bd_8ch24_48k']])
    with pytest.raises(SushiError, match='No subtitles streams found in'):
        run(['--src', files['bd_8ch24_48k'], '--dst', files['bd_stereo16_48k']])
    with pytest.raises(SushiError, match='bd_stereo16_48k.m2ts: video timestamps cannot be read from a transport stream'):
        run(['--src', files['bd_stereo16_48k'], '--dst', files['bd_8ch24_48k'], '--script', s,
             '--src-keyframes', files['kf'], '--dst-keyframes', files['kf']])
    with pytest.raises(SushiError, match='making keyframes .SCXvid. is not supported'):
        run(['--src', files['bd_stereo16_48k'], '--dst', files['bd_8ch24_48k'], '--script', s,
             '--src-keyframes', 'make', '--dst-keyframes', 'make'])
    with pytest.raises(SushiError, match='demuxing is not supported.*does not open as a transport stream.*2 programs'):
        run(['--src', files['bd_two_programs'], '--dst', files['bd_8ch24_48k'], '--script', s])
    bad = tmp_path / 'x.ts'
    bad.write_bytes(b'\1' * 1000)
    with pytest.raises(SushiError, match='demuxing is not supported.*not a transport stream'):
        run(['--src', str(bad), '--dst', files['bd_8ch24_48k'], '--script', s])


def test_selected_streams_reach_shift_script(files, tmp_path, monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, 'shift_script', lambda src, dst, *a, **kw: seen.update(kw, src=src, dst=dst))
    run(['--src', files['bd_two_lpcm'], '--dst', files['bd_8ch24_48k'], '--script', files['script'], '--src-audio', '2',
         '--no-cleanup', '--src-fps', '23.976', '--dst-fps', '23.976'])
    assert seen['src_track'] == 2 and seen['dst_track'] == 0 and seen['chapter_times'] == []
    chapters = files['bd_two_lpcm'] + '.sushi.chapters.txt'
    assert os.path.exists(chapters) and open(chapters).read() == ''
