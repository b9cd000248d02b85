"""The Matroska reader (sushi_b200/matroska.py) on every case of tests/mkv_cases.py, against FFmpeg's libavformat
demuxer (tests/ref_mkv.py): streams, stream ids, default flags, each track's frame bytes and timestamps, chapter times
as the reference parses them, and which packets survive a truncated file.  Also: FFmpeg's FLAC decoder gives the
encoder's PCM from each FLAC track, the extracted scripts and timecodes are what the case was built from, an audio
load reads almost none of the video, and damaged or refused files raise SushiError naming the byte offset or track."""
import logging
import re

import numpy as np
import pytest

from oracle import ref_flac
from sushi_b200 import matroska as mk
from sushi_b200.common import SushiError
from sushi_b200.script import AssScript, SrtScript
from tests import mkv_cases as mc
from tests import ref_mkv

CASES = mc.all_cases()
TRUNCATED = [c for c in CASES if c.damage and c.damage[0].startswith('truncated')]
READABLE = [c for c in CASES if c.refused is None and (c.damage is None or c in TRUNCATED)]
CODECS = {'A_FLAC': 'flac', 'A_PCM/INT/LIT': {16: 'pcm_s16le', 24: 'pcm_s24le'}, 'A_PCM/INT/BIG': {16: 'pcm_s16be'},
          'A_AAC': 'aac', 'V_VP9': 'vp9', 'S_TEXT/ASS': 'ass', 'S_TEXT/SSA': 'ass', 'S_TEXT/UTF8': 'subrip'}


def codec_name(t):
    c = CODECS[t.codec_id]
    return c[t.bit_depth] if isinstance(c, dict) else c


@pytest.fixture(scope='module')
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp('mkv')
    return {c.name: c.write(d) for c in CASES}


@pytest.mark.parametrize('case', READABLE, ids=lambda c: c.name)
def test_reader_equals_ffmpeg(files, case):
    path = files[case.name]
    ref = ref_mkv.demux(path, case.scale)
    with mk.MatroskaFile(path) as f:
        tracks = [(t.kind, codec_name(t), t.default) for t in f.tracks]
        assert tracks == [s for s in ref.streams if s[0] != 'attachment']
        assert [t.id for t in f.tracks] == list(range(len(f.tracks)))
        tables = f.frames([t.id for t in f.tracks])
        for t in f.tracks:
            tb = tables[t.id]
            got = [(tb.frame(i), int(tb.time[i])) for i in range(len(tb))]
            assert got == ref.track(t.id), (t.id, len(got), len(ref.track(t.id)))
            # and what the case put there
            assert [(e[0], e[1], e[2]) for e in case.expect[t.id]] == [g + (int(tb.block[i]),) for i, g in enumerate(got)]
        # the reference's parse of ffmpeg's "Chapter #0.N: start %f" lines
        text = ''.join('    Chapter #0.%d: start %f, end 0.000000\n' % (i, s / 1e9) for i, s in enumerate(ref.chapters))
        assert f.chapters == [float(x) for x in re.findall(r'Chapter #0.\d+: start (\d+\.\d+)', text)]
        assert f.chapter_starts == case.chapters


@pytest.mark.parametrize('case', TRUNCATED, ids=lambda c: c.name)
def test_truncated_file_keeps_what_precedes_the_cut(files, caplog, case):
    with caplog.at_level(logging.WARNING), mk.MatroskaFile(files[case.name]) as f:
        tb = f.frames([0])[0]
    assert len(tb) == len(case.expect[0]) > 0
    assert 'file ends inside the element at byte %d' % case.damage[1] in caplog.text


@pytest.mark.parametrize('case', [c for c in READABLE if sum(s.kind == 'audio' for s in c.specs) == 1
                                  and any(s.codec == 'A_FLAC' for s in c.specs) and c.damage is None],
                         ids=lambda c: c.name)
def test_ffmpeg_decodes_each_flac_track_to_the_pcm(files, case):
    spec = [s for s in case.specs if s.codec == 'A_FLAC'][0]
    got = ref_flac.decode_pcm(files[case.name], spec.channels, spec.bits, len(spec.pcm))
    assert np.array_equal(got, spec.pcm)


def _ass_source(case):
    head, events = case.script
    lines = list(head)
    for k, start, end, payload in events:
        f = payload.split(',', 8)
        lines.append('Dialogue: %s,%s,%s,%s' % (f[1], mk._ass_time(start * 10 ** 7), mk._ass_time(end * 10 ** 7),
                                                ','.join(f[2:])))
    return '\n'.join(lines) + '\n'


@pytest.mark.parametrize('name', ['main', 'unknown_sizes'])
def test_extracted_ass_is_the_script_it_was_built_from(files, tmp_path, name):
    case = [c for c in CASES if c.name == name][0]
    sid = [i for i, s in enumerate(case.specs) if s.kind == 'subtitles'][0]
    with mk.MatroskaFile(files[name]) as f:
        text = f.script_text(f.select('subtitles', None))
        assert f.select('subtitles', None).id == sid
    (tmp_path / 'got.ass').write_text(text, encoding='utf-8')
    (tmp_path / 'want.ass').write_text(_ass_source(case), encoding='utf-8')
    got, want = AssScript.from_file(str(tmp_path / 'got.ass')), AssScript.from_file(str(tmp_path / 'want.ass'))
    fields = lambda e: (e.layer, e.start, e.end, e.style, e.name, e.margin_left, e.margin_right, e.margin_vertical,
                        e.effect, e.text)
    assert [fields(e) for e in got.events] == [fields(e) for e in want.events]
    # ReadOrder is not time order
    starts = [e.start for e in got.events]
    assert starts != sorted(starts)


def test_extracted_srt_is_the_script_it_was_built_from(files, tmp_path):
    case = [c for c in CASES if c.name == 'multi'][0]
    spec = case.specs[3]
    with mk.MatroskaFile(files['multi']) as f:
        text = f.script_text(f.select('subtitles', 3))
    (tmp_path / 'got.srt').write_text(text, encoding='utf-8')
    got = SrtScript.from_file(str(tmp_path / 'got.srt'))
    want = [(k + 1, t / 1000.0, (t + d) / 1000.0, b.decode()) for k, (b, t, d) in enumerate(spec.frames)]
    assert [(e.source_index, e.start, e.end, e.text) for e in got.events] == want


def test_unknown_script_codec_is_refused(files):
    with mk.MatroskaFile(files['main']) as f:
        with pytest.raises(SushiError, match='Unknown script type'):
            f.script_text(f.tracks[1])


def test_timecodes_are_the_sorted_video_pts(files):
    case = [c for c in CASES if c.name == 'main'][0]
    ref = ref_mkv.demux(files['main'], case.scale)
    with mk.MatroskaFile(files['main']) as f:
        text = f.timecodes_text()
    lines = text.splitlines()
    assert lines[0] == '# timestamp format v2'
    pts = sorted(t for _, t in ref.track(0))
    assert [float(x) for x in lines[1:]] == [t / 1e6 for t in pts]
    assert pts != [t for _, t in ref.track(0)]                      # B-frames: decode order is not time order
    from sushi_b200.timing import Timecodes
    assert Timecodes.parse(text).times == [t / 1e9 for t in pts]


class CountingFile(object):
    """A file object that records every read as (offset, bytes)."""

    def __init__(self, path):
        self.f = open(path, 'rb', buffering=0)
        self.reads = []

    def seek(self, pos, whence=0):
        return self.f.seek(pos, whence)

    def tell(self):
        return self.f.tell()

    def read(self, n):
        at = self.f.tell()
        b = self.f.read(n)
        self.reads.append((at, len(b)))
        return b

    def close(self):
        self.f.close()


def _overlap(reads, spans):
    total = 0
    for a, n in reads:
        for s, e in spans:
            total += max(0, min(a + n, e) - max(a, s))
    return total


@pytest.mark.parametrize('what', ['audio', 'timecodes'])
def test_loading_reads_under_one_percent_of_the_video(files, what):
    case = [c for c in CASES if c.name == 'main'][0]
    data = case.data
    spans = []
    for _, _, pos in case.expect[0]:
        hl = 1 + (9 - data[pos + 1].bit_length())
        spans.append((pos + hl, pos + hl + (int.from_bytes(data[pos + 1:pos + hl], 'big') & ((1 << (7 * (hl - 1))) - 1))))
    video = sum(e - s for s, e in spans)
    assert video > 1000000
    cf = CountingFile(files['main'])
    with mk.MatroskaFile(files['main'], fileobj=cf) as f:
        if what == 'audio':
            assert len(f.frames([f.select('audio', None).id])[1]) == len(case.expect[1])
        else:
            f.timecodes_text()
    cf.close()
    assert _overlap(cf.reads, spans) < 0.01 * video, (_overlap(cf.reads, spans), video)


@pytest.mark.parametrize('case', [c for c in CASES if c.damage and c.damage[0] in ('lace', 'parent')],
                         ids=lambda c: c.name)
def test_damaged_container_names_the_byte_offset(files, case):
    with mk.MatroskaFile(files[case.name]) as f:
        with pytest.raises(SushiError, match=case.damage[2]):
            f.frames([0])


def test_empty_flac_frame_names_its_block(files):
    case = [c for c in CASES if c.damage and c.damage[0] == 'empty'][0]
    with mk.MatroskaFile(files[case.name]) as f:
        table = f.frames([0])[0]
    with pytest.raises(SushiError, match=case.damage[2]):
        table.refuse_empty(files[case.name], 'FLAC')


@pytest.mark.parametrize('case', [c for c in CASES if c.refused], ids=lambda c: c.name)
def test_refused_audio_names_the_track_and_codec(files, case):
    with mk.MatroskaFile(files[case.name]) as f:
        with pytest.raises(SushiError, match=case.refused):
            mk.audio_codec(f.select('audio', None))


def test_select_follows_the_reference(files, caplog):
    with mk.MatroskaFile(files['multi']) as f:
        with caplog.at_level(logging.WARNING):
            assert f.select('audio', None).id == 0                      # FlagDefault absent counts as set
        assert 'Using default track 0 (flac): A_FLAC, jpn, 2 channels, 48000 Hz (default)' in caplog.text
        assert f.select('audio', 2).id == 2
        with pytest.raises(SushiError, match=r"Stream with index 3 doesn't exist in .*multi.mkv\.\nHere are all that do:\n"
                                             r"0 \(flac\): A_FLAC.*\n1 \(pcm16\): A_PCM/INT/LIT, eng, 2 channels, 48000 Hz\n"
                                             r"2 \(pcm24\): A_PCM/INT/LIT, eng, 1 channels, 44100 Hz \(default\)$"):
            f.select('audio', 3)
        assert f.select('subtitles', None).id == 3
        with pytest.raises(SushiError, match='No video streams found in'):
            f.select('video', None)
    with mk.MatroskaFile(files['two_no_default']) as f:
        with pytest.raises(SushiError, match=r'More than one audio stream found in .*two_no_default.mkv\.You need to '
                                             r'specify the exact one to demux\. Here are all candidates:\n0: A_PCM'):
            f.select('audio', None)


def test_not_ebml_and_bad_doctype(tmp_path):
    p = tmp_path / 'x.mkv'
    p.write_bytes(b'RIFF' + b'\0' * 40)
    with pytest.raises(SushiError, match='not an EBML file'):
        mk.MatroskaFile(str(p))
    data = bytearray(CASES[0].data)
    at = data.index(b'matroska')
    data[at:at + 8] = b'matrosky'
    p.write_bytes(bytes(data))
    with pytest.raises(SushiError, match='unsupported EBML document type matrosky'):
        mk.MatroskaFile(str(p))
    assert not mk.is_matroska(str(tmp_path / 'missing.mkv'))
