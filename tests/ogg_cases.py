"""Seeded writer of Ogg FLAC files for the tests, with FLAC frames from tests/flac_cases.py's encoder.

A case is one or two logical streams.  Each FLAC stream is the mapping header (0x7F "FLAC" 1.0, a header count, "fLaC"
and STREAMINFO), its metadata blocks as header packets (VORBIS_COMMENT with CHAPTERxxx comments, PADDING, SEEKTABLE),
then one frame per packet.  Packets are laid into pages by a seeded plan: pages of one segment up to 255, packets that
span two or more pages, packets that end exactly at a page's end, packets whose length is a multiple of 255 (ended by
a lacing value of 0), granule position -1 on pages where no packet ends, EOS on the last page.  A second stream is
interleaved page by page.

`good_cases()` the cases that load, `refused_cases()` files whose streams are refused by codec or mapping,
`damaged_cases()` copies with one fault each and the byte offset the refusal names, `cut_cases()` copies cut inside a
page, a page header or a capture pattern.  `assert_coverage` checks the cases reach all of the above."""
import functools
import struct

import numpy as np

from tests import flac_cases as fc

SEED = 0x0665
EMPTY_RUN = 20000                 # pages without segments in a row in the case 'empty_pages'


def _crc_table():
    t = np.zeros(256, np.uint32)
    for i in range(256):
        c = i << 24
        for _ in range(8):
            c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
        t[i] = c
    return t


CRC_TABLE = _crc_table()


def crc32_ogg(data):
    """Ogg's CRC-32: polynomial 0x04C11DB7, MSB first, initial value 0, no final XOR (table driven)"""
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFFFFFF) ^ int(CRC_TABLE[(c >> 24) ^ b])
    return c


def crc32_bitwise(data):
    """the same CRC one bit at a time, as RFC 3533 defines it"""
    c = 0
    for b in data:
        c ^= b << 24
        for _ in range(8):
            c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
    return c


def page(serial, seq, flags, granule, lacing, body):
    h = b'OggS' + bytes([0, flags]) + struct.pack('<qII', granule, serial, seq) + b'\0\0\0\0' + bytes([len(lacing)]) + \
        bytes(lacing)
    p = h + body
    return p[:22] + struct.pack('<I', crc32_ogg(p)) + p[26:]


def recrc(data, at):
    """data with the CRC of the page at `at` recomputed"""
    n = data[at + 26]
    end = at + 27 + n + sum(data[at + 27:at + 27 + n])
    p = bytearray(data[at:end])
    p[22:26] = b'\0\0\0\0'
    p[22:26] = struct.pack('<I', crc32_ogg(bytes(p)))
    return data[:at] + bytes(p) + data[end:]


def page_offsets(data):
    out, at = [], 0
    while at + 27 <= len(data) and data[at:at + 4] == b'OggS':
        n = data[at + 26]
        out.append(at)
        at += 27 + n + sum(data[at + 27:at + 27 + n])
    return out


def paginate(serial, packets, granules, rng, plan, empty=None):
    """Pages of one stream.  plan: 'mixed' (page sizes drawn per page), or a fixed segment limit; empty(i, rng): how
    many pages without segments follow page i (they carry the continuation flag when a packet is open).  Returns
    [(page bytes, info)]: info has the segment count, whether a packet ends at the page's end, and the flags."""
    segs = []                                  # (lacing value, packet index, last segment of its packet)
    for i, pk in enumerate(packets):
        n = len(pk)
        vals = [255] * (n // 255) + [n % 255]
        for j, v in enumerate(vals):
            segs.append((v, i, j == len(vals) - 1))
    data = b''.join(packets)
    pages, at, byte, seq, open_packet = [], 0, 0, 0, False
    while at < len(segs):
        if plan == 'mixed':
            limit = int(rng.choice([1, 2, 3, 17, 64, 255, 255, int(rng.integers(1, 256))]))
        else:
            limit = plan
        take = segs[at:at + limit]
        if at == 0:
            take = segs[:1]                    # the mapping header alone on the first page (the mapping asks so)
        elif plan == 'mixed' and rng.random() < 0.3:
            # flush at a packet end: a packet ends exactly at the page's end
            ends = [k for k, s in enumerate(take) if s[2]]
            if ends:
                take = take[:ends[-1] + 1]
        lacing = [s[0] for s in take]
        body_len = sum(lacing)
        ended = [s[1] for s in take if s[2]]
        flags = (1 if open_packet else 0) | (2 if at == 0 else 0) | (4 if at + len(take) == len(segs) else 0)
        granule = granules[ended[-1]] if ended else -1
        pages.append((page(serial, seq, flags, granule, lacing, data[byte:byte + body_len]),
                      dict(segs=len(take), flush=take[-1][2], flags=flags, granule=granule,
                           spans=not take[-1][2])))
        open_packet = not take[-1][2]
        byte += body_len
        at += len(take)
        seq += 1
        for _ in range(empty(seq - 1 - sum(1 for _, i in pages if not i['segs']), rng) if empty and at < len(segs) else 0):
            flags = 1 if open_packet else 0
            pages.append((page(serial, seq, flags, -1, [], b''), dict(segs=0, flush=False, flags=flags, granule=-1,
                                                                     spans=open_packet)))
            seq += 1
    return pages


def split_blocks(flac, first_frame):
    """the metadata blocks of a FLAC file (marker stripped), STREAMINFO first"""
    out, at = [], 4
    while at < first_frame:
        size = int.from_bytes(flac[at + 1:at + 4], 'big')
        out.append(bytearray(flac[at:at + 4 + size]))
        at += 4 + size
    return out


def vorbis_comment_block(comments):
    vendor = b'sushi-b200 tests'
    body = struct.pack('<I', len(vendor)) + vendor + struct.pack('<I', len(comments)) + b''.join(
        struct.pack('<I', len(c)) + c for c in comments)
    return bytearray([4]) + len(body).to_bytes(3, 'big') + body


def seektable_block(n):
    body = b''.join(struct.pack('>QQH', 4096 * i, 1000 * i, 4096) for i in range(n))
    return bytearray([3]) + len(body).to_bytes(3, 'big') + body


def padding_block(n):
    return bytearray([1]) + n.to_bytes(3, 'big') + bytes(n)


class Stream(object):
    """One FLAC stream of a case: its packets (mapping header, header packets, frames), the FlacCase it came from"""

    def __init__(self, serial, flac_case, extra, count=None, chapters=(), comments=()):
        self.serial, self.case = serial, flac_case
        flac = flac_case.flac
        blocks = split_blocks(flac, int(flac_case.offsets[0]))
        info = blocks[0]
        comments = [b'ENCODER=tests'] + [('CHAPTER%03d=%s' % (i + 1, t)).encode() for i, t in enumerate(chapters)] + \
            [('CHAPTER%03dNAME=part %d' % (i + 1, i + 1)).encode() for i in range(len(chapters))] + \
            [('%s=%s' % kv).encode() for kv in comments]
        headers = [vorbis_comment_block(comments)] + [b for b in extra]
        for k, b in enumerate(headers):
            b[0] = (b[0] & 0x7F) | (0x80 if k == len(headers) - 1 else 0)
        info[0] &= 0x7F
        n_hdr = len(headers) if count is None else count
        self.mapping = b'\x7fFLAC\x01\x00' + struct.pack('>H', n_hdr) + b'fLaC' + bytes(info)
        self.headers = [bytes(b) for b in headers]
        self.frames = [flac[int(flac_case.offsets[i]):int(flac_case.offsets[i + 1])]
                       for i in range(len(flac_case.offsets) - 1)]
        self.packets = [self.mapping] + self.headers + self.frames
        samples = np.cumsum([0] * (1 + len(self.headers)) + [f['block_size'] for f in flac_case.frames])
        self.granules = [int(s) for s in samples]


class OggCase(object):
    def __init__(self, name, data, streams, pages, chapters=()):
        self.name, self.data, self.streams, self.pages = name, data, streams, pages
        self.chapters = list(chapters)

    def write(self, directory, suffix='.oga'):
        import os
        path = os.path.join(str(directory), self.name + suffix)
        with open(path, 'wb') as f:
            f.write(self.data)
        return path

    def __repr__(self):
        return 'OggCase(%s)' % self.name


def interleave(page_lists, rng):
    """pages of several streams in one file: every stream's BOS first, then the rest interleaved at random"""
    out = [pl[0] for pl in page_lists]
    rest = [list(pl[1:]) for pl in page_lists]
    while any(rest):
        k = int(rng.choice([i for i, r in enumerate(rest) if r]))
        out.append(rest[k].pop(0))
    return out


def _flac(pred):
    return next(c for c in fc.all_cases() if pred(c) and c.corrupt is None)


def make(name, specs, seed, chapters=(), comments=()):
    """specs: [(serial, FlacCase, extra header blocks, header count or None, page plan[, empty pages])]; `chapters`
    (hh:mm:ss.mmm starts) and `comments` ((key, value) pairs) go into the first stream's VORBIS_COMMENT"""
    rng = np.random.default_rng([SEED, seed])
    streams, lists = [], []
    for k, (serial, case, extra, count, plan, *empty) in enumerate(specs):
        s = Stream(serial, case, extra, count, chapters if k == 0 else (), comments if k == 0 else ())
        streams.append(s)
        lists.append(paginate(serial, s.packets, s.granules, rng, plan, empty[0] if empty else None))
    pages = interleave(lists, rng) if len(lists) > 1 else lists[0]
    return OggCase(name, b''.join(p for p, _ in pages), streams, [i for _, i in pages], chapters)


@functools.lru_cache(maxsize=None)
def good_cases():
    cases = []
    by_ch = {}
    for c in fc.all_cases():
        if c.corrupt is None and c.bits in (16, 24) and c.channels not in by_ch and len(c.frames) > 1:
            by_ch[c.channels] = c
    for k, ch in enumerate(sorted(by_ch)):
        c = by_ch[ch]
        cases.append(make('ch%d_%d' % (ch, c.bits), [(0x1000 + ch, c, [padding_block(251)], None, 'mixed')], 10 + k))
    st16 = _flac(lambda c: c.channels == 2 and c.bits == 16 and len(c.frames) > 4)
    st24 = _flac(lambda c: c.channels == 2 and c.bits == 24 and len(c.frames) > 4)
    var = _flac(lambda c: c.flac[int(c.offsets[0]) + 1] & 1 and c.bits in (16, 24) and len(c.frames) > 2)
    cases.append(make('headers', [(0x51, st16, [seektable_block(5), padding_block(251), padding_block(300)], None,
                                   'mixed')], 30, chapters=('00:00:01.500', '00:00:03.250', '01:02:03.004')))
    cases.append(make('count0', [(0x52, st24, [padding_block(40)], 0, 'mixed')], 31))
    cases.append(make('one_segment', [(0x53, st16, [], None, 1)], 32))
    cases.append(make('full_pages', [(0x54, st24, [], None, 255)], 33))
    cases.append(make('two_streams', [(0x55, st16, [], None, 'mixed'), (0x56, st24, [padding_block(10)], None,
                                                                         'mixed')], 34))
    cases.append(make('variable', [(0x57, var, [], None, 'mixed')], 35))
    # pages without segments: some inside open packets, and after the headers a run of them that makes most of the
    # file (more pages than a chunk has 28-byte slots)
    ch3 = next(c for c in cases if c.name == 'ch3_16').streams[0].case
    cases.append(make('empty_pages', [(0x58, ch3, [], None, 17, lambda i, rng: {0: 1, 1: EMPTY_RUN}.get(
                                       i, int(rng.integers(0, 3))))], 36))
    assert_coverage(cases)
    return cases


def assert_coverage(cases):
    infos = [i for c in cases for i in c.pages]
    assert any(i['spans'] for i in infos), 'a packet spanning pages'
    assert any(i['flags'] & 1 and i['spans'] for i in infos), 'a packet spanning three pages or more'
    assert any(i['flush'] for i in infos), 'a packet ending at a page end'
    assert any(i['segs'] == 255 for i in infos) and any(i['segs'] == 1 for i in infos)
    assert any(i['granule'] == -1 for i in infos)
    assert all(c.pages[-1]['flags'] & 4 or len(c.streams) > 1 for c in cases)
    packets = [p for c in cases for s in c.streams for p in s.packets]
    assert any(len(p) % 255 == 0 for p in packets), 'a packet ended by a lacing value of 0'
    flac = [s.case for c in cases for s in c.streams]
    assert {f.bits for f in flac} == {16, 24}
    assert {f.channels for f in flac} == set(range(1, 9))
    assert any(s.mapping[7:9] == b'\0\0' for c in cases for s in c.streams), 'a header count of 0'
    assert any(len(c.streams) > 1 for c in cases)
    assert {bool(s.frames[0][1] & 1) for c in cases for s in c.streams} == {False, True}, 'fixed and variable blocks'
    assert any(c.chapters for c in cases)
    assert any(i['segs'] == 0 and i['flags'] & 1 for i in infos) and any(i['segs'] == 0 and not i['flags'] & 1
                                                                         for i in infos), 'pages without segments'
    assert any(len(c.pages) > len(c.data) // 28 + 1 for c in cases), 'a file that is mostly pages without segments'


# ---- damaged, cut and refused copies -----------------------------------------------------------------------------
class Damaged(object):
    def __init__(self, name, data, serial, offset, regex):
        self.name, self.data, self.serial, self.offset, self.regex = name, data, serial, offset, regex

    def write(self, directory):
        import os
        path = os.path.join(str(directory), self.name + '.oga')
        with open(path, 'wb') as f:
            f.write(self.data)
        return path


def damaged_cases():
    base = next(c for c in good_cases() if c.name == 'headers')
    d, serial = base.data, base.streams[0].serial
    offs = page_offsets(d)
    k = len(offs) // 2
    at = offs[k]
    out = []
    b = bytearray(d); b[at + 2] = ord('x')
    out.append(Damaged('no_capture', bytes(b), serial, at, 'no capture pattern'))
    b = bytearray(d); b[at + 4] = 1
    out.append(Damaged('version', bytes(b), serial, at, 'structure version'))
    b = bytearray(d); b[offs[k + 1] - 1] ^= 0x20
    out.append(Damaged('crc', bytes(b), serial, at, 'CRC-32 mismatch'))
    b = bytearray(d); b[at + 18:at + 22] = struct.pack('<I', struct.unpack_from('<I', d, at + 18)[0] + 1)
    out.append(Damaged('sequence', recrc(bytes(b), at), serial, at, 'sequence number'))
    b = bytearray(d); b[at + 5] ^= 1
    out.append(Damaged('continuation', recrc(bytes(b), at), serial, at, 'continuation flag'))
    other = next(c for c in good_cases() if c.name == 'ch3_16')
    out.append(Damaged('chained', d + other.data, serial, len(d), 'chained Ogg'))
    return out


def cut_cases():
    """(name, data, serial): a copy cut inside its last page's body, one cut inside a page header, one that ends
    with the first two bytes of a capture pattern"""
    base = next(c for c in good_cases() if c.name == 'headers')
    d, serial = base.data, base.streams[0].serial
    offs = page_offsets(d)
    return [('cut_body', d[:len(d) - 7], serial), ('cut_header', d[:offs[-1] + 12], serial),
            ('cut_capture', d + b'Og', serial)]


def other_stream_page(serial, packet, kind):
    return page(serial, 0, 2, 0, [255] * (len(packet) // 255) + [len(packet) % 255], packet)


CODEC_HEADERS = {
    'opus': (b'OpusHead' + bytes([1, 2]) + struct.pack('<HIhB', 312, 48000, 0, 0), b'OpusTags', b''),
    'vorbis': (b'\x01vorbis' + struct.pack('<IBIiii', 0, 2, 44100, 0, 128000, 0) + bytes([0xB8, 1]), b'\x03vorbis',
               b'\x01'),
    'speex': (b'Speex   ' + b'1.2'.ljust(20, b'\0') + struct.pack('<12i', 1, 80, 16000, 1, 4, 1, -1, 320, 0, 0, 0, 0),
              b'', b''),
}


def comment_file(codec, comments):
    """An Ogg file whose stream 0 is `codec` ('flac', or a lossy one of CODEC_HEADERS ahead of a FLAC stream) with
    the Vorbis comments `comments` ((key, value) pairs) in its comment header"""
    flac = next(c for c in good_cases() if c.name == 'ch3_16').streams[0].case
    if codec == 'flac':
        return make('comments', [(0x61, flac, [], None, 'mixed')], 40, comments=comments).data
    data = make('comments', [(0x61, flac, [], None, 'mixed')], 40).data
    second = page_offsets(data)[1]
    head, magic, tail = CODEC_HEADERS[codec]
    vendor = b'tests'
    block = struct.pack('<I', len(vendor)) + vendor + struct.pack('<I', len(comments)) + b''.join(
        struct.pack('<I', len(c)) + c for c in (('%s=%s' % kv).encode() for kv in comments))
    packet = magic + block + tail
    return (other_stream_page(0x62, head, codec) + data[:second] +
            page(0x62, 1, 0, 0, [255] * (len(packet) // 255) + [len(packet) % 255], packet) + data[second:])


def refused_cases():
    """(name, data, stream index, regex): files whose first stream is refused by name"""
    base = next(c for c in good_cases() if c.name == 'ch2_16' or c.name.startswith('ch2_'))
    opus = b'OpusHead' + bytes([1, 2]) + struct.pack('<HIhB', 312, 48000, 0, 0)
    vorbis = b'\x01vorbis' + struct.pack('<IBIiii', 0, 2, 44100, 0, 128000, 0) + bytes([0xB8, 1])
    speex = b'Speex   ' + b'1.2'.ljust(20, b'\0') + struct.pack('<12i', 1, 80, 16000, 1, 4, 1, -1, 320, 0, 0, 0, 0)
    out = []
    for name, pk in (('opus', opus), ('vorbis', vorbis), ('speex', speex)):
        out.append((name, other_stream_page(0x77, pk, name) + base.data, 0, name))
    s = base.streams[0]
    old = b'fLaC' + s.mapping[13:]
    old_data = page(0x78, 0, 2, 0, [len(old)], old) + b''.join(
        page(0x78, i + 1, 4 if i == len(s.frames) - 1 else 0, 0, [255] * (len(f) // 255) + [len(f) % 255], f)
        for i, f in enumerate(s.frames[:3]))
    out.append(('old_mapping', old_data, 0, 'before FLAC 1.1.1'))
    return out
