"""sushi_b200/matroska.py on the A_TRUEHD files of tests/mkv_truehd_cases.py, held to FFmpeg's Matroska demuxer
(tests/ref_mkv.py): the same streams, the same video frames and times, and the same TrueHD bytes (FFmpeg's TrueHD
parser may split a frame of several access units into one packet per unit, so the track's bytes are compared end to
end) -- on the whole file and on a copy cut inside a late cluster, of which both keep what precedes the cut."""
import logging

import pytest

from sushi_b200 import matroska as mk
from tests import mkv_truehd_cases as mtc
from tests import ref_mkv

PAIRS = mtc.cases()


def _check(path, scale):
    ref = ref_mkv.demux(path, scale)
    with mk.MatroskaFile(path) as f:
        assert [t.kind for t in f.tracks] == [s[0] for s in ref.streams if s[0] != 'attachment']
        assert mk.audio_codec(f.select('audio', None)) == 'truehd'
        tables = f.frames([t.id for t in f.tracks])
        for t in f.tracks:
            tb = tables[t.id]
            if t.kind == 'audio':
                assert tb.data == b''.join(p for p, _ in ref.track(t.id))
            else:
                assert [(tb.frame(i), int(tb.time[i])) for i in range(len(tb))] == ref.track(t.id)
        return tables


@pytest.mark.parametrize('pair', PAIRS, ids=lambda p: p[0].name)
def test_reader_equals_ffmpeg_on_truehd_tracks(tmp_path, pair):
    mkv, _ = pair
    _check(mkv.write(tmp_path), mkv.scale)


@pytest.mark.parametrize('pair', PAIRS, ids=lambda p: p[0].name)
def test_cut_file_keeps_what_precedes_the_cut(tmp_path, caplog, pair):
    mkv, _ = pair
    path = str(tmp_path / (mkv.name + '_cut.mkv'))
    with open(path, 'wb') as f:
        f.write(mkv.data[:len(mkv.data) * 3 // 4])
    with caplog.at_level(logging.WARNING):
        tables = _check(path, mkv.scale)
    assert 'file ends inside the element' in caplog.text
    assert 0 < len(tables[1]) < len(mtc.cases()[PAIRS.index(pair)][1].au_offsets)
