"""FFmpeg's `wav` demuxer, Matroska demuxer and `wavpack` decoder, driven through ctypes, against tests/wavpack_cases.py
and sushi_b200/wavpack.py: every .wv case and every A_WAVPACK4 track decodes to the PCM the writer meant; the host's
block tables hold FFmpeg's packets (bytes, file positions, sample counts); and what FFmpeg does with each damaged copy
is recorded beside the refusal this project gives instead (DESIGN.md section 2)."""
import numpy as np
import pytest

from sushi_b200 import SushiError
from sushi_b200 import matroska as mk
from sushi_b200 import wavpack as wp
from tests import mkv_wavpack_cases as mwc
from tests import ref_wavpack as ref
from tests import wavpack_cases as wc

CASES = wc.all_cases()
MKV = mwc.cases()
BASE, DAMAGED = wc.damaged_cases()
# (samples FFmpeg decodes, packets its decoder refuses) for each damaged copy; the base holds 3 blocks of 400 samples
FFMPEG = {
    'bad_version': (400, 0), 'size_past_file': (800, 0), 'subblock_overrun': (1200, 0), 'no_bitstream': (800, 1),
    'bad_term': (800, 1), 'too_many_terms': (800, 1), 'bitstream_overrun': (1200, 0), 'crc': (1200, 0),
    'index_gap': (1200, 0), 'cut_last_block': (800, 0), 'total_mismatch': (1200, 0), 'trailing_junk': (1200, 0),
    'not_initial': (800, 1), 'hybrid': (0, 3), 'float': (0, 3), 'dsd': (0, 3), '1-byte': (1200, 0),
    '4-byte': (1200, 0), 'int32_sent_bits': (300, 0), 'wvx': (1200, 0), 'mono_no_terms': (600, 0),
}


def _write(tmp_path, name, data):
    path = str(tmp_path / (name + '.wv'))
    with open(path, 'wb') as f:
        f.write(data)
    return path


def test_cases_cover_the_decoder():
    wc.assert_coverage(CASES)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_ffmpeg_decodes_the_wv_file_to_its_pcm(tmp_path, case):
    out, refused = ref.decode(_write(tmp_path, case.name, case.wv()), case.channels, case.bits)
    assert refused == 0
    assert np.array_equal(out, case.pcm)


@pytest.mark.parametrize('pair', MKV, ids=lambda p: p[0].name)
def test_ffmpeg_decodes_the_matroska_track_to_its_pcm(tmp_path, pair):
    mkv, case = pair
    out, refused = ref.decode(mkv.write(tmp_path), case.channels, case.bits)
    assert refused == 0
    assert np.array_equal(out, case.pcm[:mwc.kept_samples(mkv, case)])


def _same_blocks(table, data, packets):
    """each packet's blocks are the table's rows of one frame, in order: bytes, flags, CRC and sample count"""
    rows = [r for r in table]
    k = 0
    for pos, blocks in packets:
        for count, flags, crc, body in blocks:
            r = rows[k]
            assert (int(r[2]), int(r[3]), int(r[4])) == (count, flags, crc)
            assert data[int(r[0]):int(r[0] + r[1])] == body
            k += 1
    assert k == len(rows)


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_block_table_holds_ffmpegs_packets(tmp_path, case):
    path = _write(tmp_path, case.name, case.wv())
    f = wp.WavPackFile(path)
    packets = ref.packets(path)
    _same_blocks(f.table, f.data, packets)
    starts = f.table[f.table[:, 6] == 0]
    assert [p for p, _ in packets] == [int(w) for w in starts[:, 7]]
    assert list(starts[:, 5]) == list(np.concatenate([[0], np.cumsum(case.counts)[:-1]]))
    assert (f.stream.channels, f.stream.rate, f.stream.bits_per_sample) == (case.channels, case.rate, case.bits)


@pytest.mark.parametrize('pair', MKV, ids=lambda p: p[0].name)
def test_matroska_block_table_holds_ffmpegs_packets(tmp_path, pair):
    mkv, case = pair
    path = mkv.write(tmp_path)
    with mk.MatroskaFile(path) as f:
        t = f.select('audio', None)
        assert mk.audio_codec(t) == 'wavpack'
        frames = f.frames([t.id])[t.id]
    table, stream = wp.matroska_table(frames, t.codec_private, t.id, t.channels)
    packets = ref.packets(path)
    _same_blocks(table, frames.data, packets)
    assert len(packets) == int((table[:, 6] == 0).sum())          # one packet per frame
    assert stream.channels == case.channels


@pytest.mark.parametrize('damaged', DAMAGED, ids=lambda d: d[0])
def test_what_ffmpeg_does_with_each_damaged_copy(tmp_path, damaged):
    name, data, block, regex, kernel = damaged
    path = _write(tmp_path, name, data)
    out, refused = ref.decode(path, 1 if name == 'mono_no_terms' else 2, 16)
    assert (len(out), refused) == FFMPEG[name]
    if not kernel:
        with pytest.raises(SushiError, match=regex):
            wp.WavPackFile(path)
    else:
        wp.WavPackFile(path)                     # the header chain is sound: the GPU decoder refuses the block


def test_tags_end_the_block_chain_as_for_ffmpeg(tmp_path):
    """An APEv2 or ID3v1 tag after the last block ends the chain; the same bytes without the tag end it too."""
    for case in CASES:
        if case.tail:
            with_tag = wp.WavPackFile(_write(tmp_path, 'a', case.wv()))
            case.tail, tail = b'', case.tail
            without = wp.WavPackFile(_write(tmp_path, 'b', case.wv()))
            case.tail = tail
            assert np.array_equal(with_tag.table, without.table)
            assert len(ref.packets(_write(tmp_path, 'c', case.wv()))) == len(case.counts)
