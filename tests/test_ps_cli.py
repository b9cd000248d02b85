"""The command line's refusals on program stream and raw MPEG audio inputs, all before the GPU is touched: AC-3, DTS,
DVD-LPCM and layer III named, several audio streams without --src-audio, a DVD subtitle script, keyframes without fps
or timecodes, a name that does not open as a program stream.  Also the streams it selects."""
import pytest

from sushi_b200 import cli
from sushi_b200.common import SushiError
from tests import mpa_cases
from tests import ps_cases as pc


def run(argv):
    return cli.run(cli.create_arg_parser().parse_args(argv))


@pytest.fixture
def files(tmp_path):
    good = {c.name: c for c in pc.good_cases()}
    out = {name: good[name].write(tmp_path) for name in ('dvd_joint', 'two_audio', 'vcd_stereo', 'dvb_lsf')}
    l3, lossy = pc.refused_cases()
    out['layer3'], out['dvd_lossy'] = l3.write(tmp_path), lossy.write(tmp_path)
    (tmp_path / 'l3.mp2').write_bytes(mpa_cases.layer3())
    out['l3_mp2'] = str(tmp_path / 'l3.mp2')
    (tmp_path / 'in.ass').write_text('[Script Info]\n')
    (tmp_path / 'kf.txt').write_text('# XviD 2pass stat file\n\n\ni\n')
    out['script'] = str(tmp_path / 'in.ass')
    out['kf'] = str(tmp_path / 'kf.txt')
    return out


def test_refusals(files, tmp_path, monkeypatch):
    monkeypatch.setattr(cli, 'shift_script', lambda *a, **kw: pytest.fail('the GPU path was reached'))
    s, dst = files['script'], files['vcd_stereo']
    for path, idx, what in ((files['dvd_lossy'], '0', 'pcm_dvd'), (files['dvd_lossy'], '1', 'ac3'),
                            (files['dvd_lossy'], '2', 'dts'), (files['layer3'], '0', r'MPEG audio layer III \(MP3\)')):
        with pytest.raises(SushiError, match=r'Audio track {0} is {1}, which cannot be decoded here'.format(idx, what)):
            run(['--src', path, '--dst', dst, '--script', s, '--src-audio', idx])
    with pytest.raises(SushiError, match=r'l3.mp2 is MPEG audio layer III \(MP3\), which cannot be decoded here'):
        run(['--src', files['l3_mp2'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='More than one audio stream found'):
        run(['--src', files['two_audio'], '--dst', dst, '--script', s])
    with pytest.raises(SushiError, match='^Unknown script type$'):
        run(['--src', files['dvd_joint'], '--dst', dst, '--src-audio', '5'])
    with pytest.raises(SushiError, match='No subtitles streams found in'):
        run(['--src', files['vcd_stereo'], '--dst', dst])
    with pytest.raises(SushiError, match='vcd_stereo.mpg: video timestamps cannot be read from a program stream'):
        run(['--src', dst, '--dst', files['dvb_lsf'], '--script', s, '--src-keyframes', files['kf'],
             '--dst-keyframes', files['kf']])
    bad = tmp_path / 'x.vob'
    bad.write_bytes(b'\1' * 1000)
    with pytest.raises(SushiError, match='demuxing is not supported.*does not open as a program stream.*not a program '
                                         'stream'):
        run(['--src', str(bad), '--dst', dst, '--script', s])


def test_selected_streams_reach_shift_script(files, monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, 'shift_script', lambda src, dst, *a, **kw: seen.update(kw, src=src, dst=dst))
    run(['--src', files['two_audio'], '--dst', files['dvb_lsf'], '--script', files['script'], '--src-audio', '2',
         '--src-fps', '25', '--dst-fps', '25'])
    assert seen['src_track'] == 2 and seen['dst_track'] == 0 and seen['chapter_times'] == []
