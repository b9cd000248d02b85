"""The command line's refusals on Ogg inputs, all before the GPU is touched: Opus, Vorbis and Speex named with their
stream, the FLAC mapping before 1.0, several audio streams without --src-audio, no script stream, keyframes without fps
or timecodes, a name that does not open as an Ogg file.  Also the streams and chapters it selects."""
import pytest

from sushi_b200 import cli
from sushi_b200.common import SushiError
from tests import ogg_cases as oc


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def files(tmp_path):
    good = {c.name: c for c in oc.good_cases()}
    out = {name: good[name].write(tmp_path) for name in ('ch2_16', 'two_streams', 'headers')}
    for name, data, _, _ in oc.refused_cases():
        p = tmp_path / (name + ('.opus' if name == 'opus' else '.ogg'))
        p.write_bytes(data)
        out[name] = str(p)
    (tmp_path / 'in.ass').write_text('[Script Info]\n')
    (tmp_path / 'kf.txt').write_text('# XviD 2pass stat file\n\n\ni\n')
    out['script'] = str(tmp_path / 'in.ass')
    out['kf'] = str(tmp_path / 'kf.txt')
    return out


def test_refusals(files, tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    s, dst = files['script'], files['ch2_16']
    for name in ('opus', 'vorbis', 'speex'):
        with pytest.raises(SushiError, match=r'Audio track 0 is {0}, which cannot be decoded here'.format(name)):
            run(['--src', files[name], '--dst', dst, '--script', s, '--src-audio', '0'])
    with pytest.raises(SushiError, match='More than one audio stream found'):
        run(['--src', files['opus'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='stream 0 uses the FLAC-in-Ogg mapping from before FLAC 1.1.1'):
        run(['--src', files['old_mapping'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='More than one audio stream found'):
        run(['--src', files['two_streams'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='No subtitles streams found in'):
        run(['--src', files['ch2_16'], '--dst', dst])
    with pytest.raises(SushiError, match='ch2_16.oga: video timestamps cannot be read from an Ogg file'):
        run(['--src', dst, '--dst', files['headers'], '--script', s, '--src-keyframes', files['kf'],
             '--dst-keyframes', files['kf']])
    bad = tmp_path / 'x.oga'
    bad.write_bytes(b'\1' * 1000)
    with pytest.raises(SushiError, match='demuxing is not supported.*does not open as an Ogg file.*not an Ogg file'):
        run(['--src', str(bad), '--dst', dst, '--script', s])


def test_selected_streams_and_chapters_reach_shift_script(files, monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, 'shift_script', lambda src, dst, *a, **kw: seen.update(kw, src=src, dst=dst))
    run(['--src', files['two_streams'], '--dst', files['headers'], '--script', files['script'], '--src-audio', '1',
         '--src-fps', '25', '--dst-fps', '25'])
    assert seen['src_track'] == 1 and seen['dst_track'] == 0
    run(['--src', files['headers'], '--dst', files['ch2_16'], '--script', files['script']])
    assert seen['chapter_times'] == [1.5, 3.25, 3723.004]
