"""Ogg files on the CPU: the writer of tests/ogg_cases.py, sushi_b200.ogg and the CPU build of sushi_b200/csrc/sb_ogg.cuh
(tests/emu/emu_ogg_driver.cpp, compiled with g++) against FFmpeg's `ogg` demuxer (tests/ref_ogg.py):
  - the stream list ogg.py reads (order, kinds, codec names) and its chapters equal FFmpeg's;
  - the emulation driver gives the packets FFmpeg's demuxer returns, at chunk sizes down to a few bytes, and names
    the page where each packet starts;
  - the CRC-32 of 32 combined slices equals a plain bitwise CRC-32 of every page;
  - every damaged copy is refused naming the expected offset, and what FFmpeg makes of it is recorded;
  - cut copies keep the packets that end before the cut, as FFmpeg does;
  - the refusals by codec name and mapping, and stream selection."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from sushi_b200 import ogg
from sushi_b200.common import SushiError
from tests import ogg_cases as oc
from tests import ref_ogg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, 'tests', 'emu')
DRIVER = os.path.join(EMU, 'emu_ogg_driver.cpp')
SOURCES = [DRIVER, os.path.join(ROOT, 'sushi_b200', 'csrc', 'sb_ogg.cuh')]
LIB = os.path.join(EMU, '_build', 'libsb_emu_ogg.so')
GOOD = oc.good_cases()
CHUNKS = (1 << 20, 4096, 2051, 777, 37, 28, 5)


@pytest.fixture(scope='module')
def emu():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(['g++', '-std=c++17', '-O2', '-Wall', '-Wno-unused-function', '-I',
                               os.path.join(ROOT, 'sushi_b200', 'csrc'), '-shared', '-fPIC', DRIVER, '-o', LIB])
    lib = ctypes.CDLL(LIB)
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.emu_ogg_demux.argtypes = [vp, i64, ctypes.c_uint32, i64, vp, i64, vp, vp, i64, vp, ctypes.c_char_p, ctypes.c_int]
    lib.emu_ogg_demux.restype = i64
    lib.emu_ogg_crc.argtypes = [vp, i64]
    lib.emu_ogg_crc.restype = ctypes.c_uint32
    return lib


def demux(emu, data, serial, chunk):
    """-> (complete packets, file offset of each one's page, cut) or (None, message)"""
    buf = np.frombuffer(data, np.uint8)
    es = np.zeros(len(data) + 1, np.uint8)
    starts = np.zeros(len(data) + 1, np.int64)
    files = np.zeros(len(data) + 1, np.int64)
    info = np.zeros(3, np.int64)
    msg = ctypes.create_string_buffer(256)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    n = emu.emu_ogg_demux(p(buf), len(data), serial, chunk, p(es), len(es), p(starts), p(files), len(starts), p(info),
                          msg, 256)
    if n < 0:
        return None, msg.value.decode()
    count, closed = int(info[0]), int(info[1])
    bounds = [int(x) for x in starts[:count]] + [closed]
    packets = [es[bounds[i]:bounds[i + 1]].tobytes() for i in range(count) if bounds[i] < closed]
    return packets, [int(x) for x in files[:len(packets)]], int(info[2])


def start_pages(data, serial):
    """the file offset of the page where each packet of stream `serial` starts, walked here page by page"""
    out, open_packet = [], False
    for at in oc.page_offsets(data):
        if int.from_bytes(data[at + 14:at + 18], 'little') != serial:
            continue
        lacing = data[at + 27:at + 27 + data[at + 26]]
        for i, v in enumerate(lacing):
            if (i == 0 and not open_packet) or (i > 0 and lacing[i - 1] < 255):
                out.append(at)
        if lacing:                         # a page without segments leaves the open packet open
            open_packet = lacing[-1] == 255
    return out


@pytest.mark.parametrize('case', GOOD, ids=lambda c: c.name)
def test_stream_list_and_chapters_equal_ffmpegs(tmp_path, case):
    path = case.write(tmp_path)
    f = ogg.OggFile(path)
    mine = [dict(kind=s.kind, codec=s.codec) for s in f.streams_all]
    assert [s.id for s in f.streams_all] == list(range(len(mine)))
    assert mine == ref_ogg.streams(path)
    assert f.chapters == ref_ogg.chapters(path)
    assert len(f.chapters) == len(case.chapters)


@pytest.mark.parametrize('case', GOOD, ids=lambda c: c.name)
def test_emulation_gives_ffmpegs_packets(emu, tmp_path, case):
    path = case.write(tmp_path)
    f = ogg.OggFile(path)
    for k, s in enumerate(case.streams):
        mine = f.streams_all[k]
        assert mine.serial == s.serial and len(mine.packets) - 1 == len(s.headers)
        want = ref_ogg.packets(path, k)
        assert want == s.frames
        pages = start_pages(case.data, s.serial)
        for chunk in CHUNKS:
            packets, files, cut = demux(emu, case.data, s.serial, chunk)
            assert packets == s.packets, chunk
            assert files == pages and cut == 0


@pytest.mark.parametrize('case', GOOD, ids=lambda c: c.name)
def test_sliced_crc_equals_bitwise_crc(emu, case):
    d = case.data
    offs = oc.page_offsets(d) + [len(d)]
    for a, b in zip(offs, offs[1:]):
        pg = bytearray(d[a:b])
        stored = int.from_bytes(pg[22:26], 'little')
        pg[22:26] = b'\0\0\0\0'
        want = oc.crc32_bitwise(bytes(pg)) if b - a < 4096 else oc.crc32_ogg(bytes(pg))
        assert want == stored
        buf = np.frombuffer(d[a:b], np.uint8)
        assert emu.emu_ogg_crc(buf.ctypes.data_as(ctypes.c_void_p), b - a) == want


def test_table_crc_equals_bitwise_crc():
    rng = np.random.default_rng(5)
    for n in (0, 1, 27, 300, 2000):
        data = rng.integers(0, 256, n).astype(np.uint8).tobytes()
        assert oc.crc32_ogg(data) == oc.crc32_bitwise(data)


# FFmpeg drops a page that fails its CRC, resyncs past a broken capture pattern and reads on; what it returns for each
# damaged copy, as frames of the chosen stream (None: the file does not open)
def _ffmpeg_frames(path):
    try:
        return len(ref_ogg.packets(path, 0))
    except RuntimeError:
        return None


@pytest.mark.parametrize('case', oc.damaged_cases(), ids=lambda c: c.name)
def test_damaged_copies_are_refused_at_their_offset(emu, tmp_path, case):
    for chunk in (1 << 20, 777, 28):
        out = demux(emu, case.data, case.serial, chunk)
        assert out[0] is None, (chunk, case.name)
        assert out[1].startswith('Ogg page at byte offset %d: ' % case.offset), out[1]
        assert case.regex in out[1]
    good = next(c for c in GOOD if c.name == 'headers')
    frames = _ffmpeg_frames(case.write(tmp_path))
    whole = len(good.streams[0].frames)
    # FFmpeg: a damaged page is dropped (or resynced past) and the rest is read; a chained stream reads on
    if case.name in ('no_capture', 'version', 'crc'):
        assert frames is not None and frames < whole
    else:
        assert frames is not None and frames >= whole - 1


@pytest.mark.parametrize('name,data,serial', oc.cut_cases(), ids=lambda v: v if isinstance(v, str) else '')
def test_cut_copies_keep_the_packets_ffmpeg_keeps(emu, tmp_path, name, data, serial):
    path = os.path.join(str(tmp_path), name + '.oga')
    with open(path, 'wb') as f:
        f.write(data)
    want = ref_ogg.packets(path, 0)
    good = next(c for c in GOOD if c.name == 'headers').streams[0]
    for chunk in (1 << 20, 777, 5):
        packets, files, cut = demux(emu, data, serial, chunk)
        assert packets[1 + len(good.headers):] == want, chunk
        assert cut == 1
    if name == 'cut_capture':
        assert want == good.frames
    else:
        assert len(want) < len(good.frames)


@pytest.mark.parametrize('name,data,index,regex', oc.refused_cases(), ids=lambda v: v if isinstance(v, str) else '')
def test_refusals_name_the_stream_and_codec(tmp_path, name, data, index, regex):
    path = os.path.join(str(tmp_path), name + '.ogg')
    with open(path, 'wb') as f:
        f.write(data)
    f = ogg.OggFile(path)
    assert [dict(kind=s.kind, codec=s.codec) for s in f.streams_all] == ref_ogg.streams(path)
    with pytest.raises(SushiError, match=regex) as e:
        f.select_audio(index)
    assert 'stream 0' in str(e.value) or 'track 0' in str(e.value)


def test_selection_and_default_rule(tmp_path):
    case = next(c for c in GOOD if c.name == 'two_streams')
    path = case.write(tmp_path)
    f = ogg.OggFile(path)
    with pytest.raises(SushiError, match='More than one audio stream'):
        f.select_audio(None)
    a = f.select_audio(1)
    assert a.id == 1 and a.label == 'FLAC' and a.bits == 24 and a.fmt == 'S32'
    with pytest.raises(SushiError, match="doesn't exist"):
        f.select_audio(5)


def test_header_count_zero_is_resolved_by_content(tmp_path):
    case = next(c for c in GOOD if c.name == 'count0')
    s = case.streams[0]
    assert s.mapping[7:9] == b'\0\0'
    f = ogg.OggFile(case.write(tmp_path))
    assert len(f.streams_all[0].packets) - 1 == len(s.headers)
    assert ref_ogg.packets(case.write(tmp_path), 0) == s.frames


def test_skeleton_and_theora_are_listed_as_ffmpeg_lists_them(tmp_path):
    base = next(c for c in GOOD if c.name == 'ch3_16')
    import struct
    theora = b'\x80theora' + bytes([3, 2, 1]) + struct.pack('>HH', 20, 15) + bytes([0, 0x01, 0x40, 0, 0xF0, 0, 0]) + \
        struct.pack('>II', 25, 1) + bytes([0, 0, 1, 0, 0, 1]) + bytes([0, 0, 0, 0x80, 0x68, 0x50])
    skel = b'fishead\0' + struct.pack('<HHqqqq', 3, 0, 0, 1000, 0, 1000) + bytes(20)
    for name, pk in (('theora', theora), ('skeleton', skel)):
        path = os.path.join(str(tmp_path), name + '.ogg')
        with open(path, 'wb') as f:
            f.write(oc.other_stream_page(0x99, pk, name) + base.data)
        r = ogg.OggFile(path)
        assert [dict(kind=s.kind, codec=s.codec) for s in r.streams_all] == ref_ogg.streams(path)
        assert r.select_audio(None).id == 1


def test_is_ogg_sniffs_the_capture_pattern(tmp_path):
    case = GOOD[0]
    assert ogg.is_ogg(case.write(tmp_path))
    p = tmp_path / 'x.ogg'
    p.write_bytes(b'RIFF0000WAVE')
    assert not ogg.is_ogg(str(p))
    assert not ogg.is_ogg(str(tmp_path / 'missing.ogg'))


ODD_CHAPTERS = [('CHAPTER001', '00:00:01.500'), ('CHAPTER02', '100:00:00.000'), ('CHAPTER003', '01.02.03.004'),
                ('chapter004', ' 1:2:3.4'), ('CHAPTER005', '1:02:03.0045'), ('CHAPTER001NAME', 'x'),
                ('CHAPTERx1', '00:00:01.000'), ('CHAPTER006', '+1:-2:03.004'), ('CHAPTER007', '00:01:02'),
                ('CHAPTER008', '00:00:09.5'), ('CHAPTER008', '00:00:07.25'), ('CHAPTER0009', '00:00:02.000')]


@pytest.mark.parametrize('codec', ['flac', 'opus', 'speex', 'vorbis'])
def test_chapters_are_read_as_ffmpeg_reads_them(tmp_path, codec):
    """field widths, separators, signs, white space, short and long keys, a number given twice, in every codec's
    comment header FFmpeg reads"""
    path = str(tmp_path / ('chapters_%s.ogg' % codec))
    with open(path, 'wb') as f:
        f.write(oc.comment_file(codec, ODD_CHAPTERS))
    want = ref_ogg.chapters(path)
    assert ogg.OggFile(path).chapters == want
    assert 1.5 in want and 100 * 3600.0 not in want


def test_pages_without_segments(emu, tmp_path):
    """a page without segments keeps an open packet open; a chunk made mostly of such pages holds more pages than it
    has 28-byte slots, and every one of them is kept in the page table"""
    case = next(c for c in GOOD if c.name == 'empty_pages')
    s = case.streams[0]
    assert len(case.pages) > len(case.data) // 28 + 1
    assert sum(1 for i in case.pages if i['segs'] == 0) >= oc.EMPTY_RUN
    path = case.write(tmp_path)
    assert ref_ogg.packets(path, 0) == s.frames
    assert len(ogg.OggFile(path).streams_all[0].packets) == 1 + len(s.headers)
    for chunk in (1 << 20, 4096, 27, 5):
        packets, files, cut = demux(emu, case.data, s.serial, chunk)
        assert packets == s.packets and cut == 0
