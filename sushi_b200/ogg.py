"""Ogg files on the host: `.ogg`, `.oga` and `.opus`.

The host reads only the head of the file: the pages that begin the streams, then each stream's header packets.  It
lists the streams as FFmpeg's `ogg` demuxer lists them: in the order their first pages appear, with FFmpeg's kind and
codec name (`flac`, `vorbis`, `opus`, `speex`, `theora`; Skeleton is a data
stream without a codec).  Chapters are the CHAPTERxxx Vorbis comments FFmpeg reads from the streams' comment headers.

Ogg FLAC (the FLAC-to-Ogg mapping 1.0: a packet 0x7F "FLAC", major 1, minor 0, a header count, "fLaC" and STREAMINFO,
then one metadata block per header packet, then one frame per packet) is demuxed and decoded on the GPU (sb_ogg_*):
the host reads the file in large chunks and hands them over, and does no per-page work.  The header packets are the
ones before the first packet that starts with a frame's sync byte, as FFmpeg counts them; the header count field is
not used.  Lossy streams, the mapping before 1.0 and chained files are refused by name.
"""
import logging
import os
import re
import struct

from . import _native, swr
from .common import Audio, Container, SushiError
from .flac import FlacFile

OGG_EXTENSIONS = ('.ogg', '.oga', '.opus')
HEAD_BYTES = 16 << 20            # how far the header packets are looked for
# bytes of file each sb_ogg_feed call takes, through one page-locked buffer
CHUNK_BYTES = 64 << 20

# the first bytes of a stream's first packet: (kind, FFmpeg's codec name)
MAPPINGS = ((b'\x7fFLAC', ('audio', 'flac')), (b'fLaC', ('audio', 'flac')), (b'\x01vorbis', ('audio', 'vorbis')),
            (b'OpusHead', ('audio', 'opus')), (b'Speex   ', ('audio', 'speex')), (b'\x80theora', ('video', 'theora')),
            (b'fishead\x00', ('data', 'none')))
# the header packet that holds a codec's Vorbis comments: (index among its packets, bytes before the comments)
COMMENTS = {'vorbis': (1, 7), 'opus': (1, 8), 'speex': (1, 0), 'theora': (1, 7)}
_SPACE = re.compile(r'[ \t\n\v\f\r]*')


def is_ogg(path):
    """True when the file starts with an Ogg capture pattern (False when it cannot be read)."""
    try:
        with open(path, 'rb') as f:
            return f.read(4) == b'OggS'
    except OSError:
        return False


def read_pages(f, limit):
    """(file offset, flags, serial, sequence, lacing values, body) of each page from the file's start, following the
    chain by length, until `limit` bytes or a page that does not parse"""
    at = 0
    while at < limit:
        f.seek(at)
        h = f.read(27)
        if len(h) < 27 or h[:4] != b'OggS' or h[4] != 0:
            return
        lacing = f.read(h[26])
        body = f.read(sum(lacing))
        if len(lacing) < h[26] or len(body) < sum(lacing):
            return
        serial, seq = struct.unpack_from('<II', h, 14)
        yield at, h[5], serial, seq, lacing, body
        at += 27 + len(lacing) + len(body)


def vorbis_comments(data):
    """[(key, value)] of a Vorbis comment block (vendor string, count, then length-prefixed KEY=value strings); the
    comments that fit when the block is short"""
    out = []
    try:
        n = struct.unpack_from('<I', data, 0)[0]
        at = 4 + n
        count = struct.unpack_from('<I', data, at)[0]
        at += 4
        for _ in range(count):
            n = struct.unpack_from('<I', data, at)[0]
            s = data[at + 4:at + 4 + n]
            at += 4 + n
            if len(s) < n:
                break
            key, eq, value = s.partition(b'=')
            if eq:
                out.append((key.decode('ascii', 'replace'), value.decode('utf-8', 'replace')))
    except struct.error:
        pass
    return out


def _scan_int(text, at, width):
    """C's sscanf %<width>d at text[at]: white space skipped, then a sign and digits, `width` characters at most;
    (value, position after it), or None when no digit is read"""
    m = _SPACE.match(text, at)
    at = m.end()
    m = re.compile(r'[+-]?[0-9]{1,%d}' % width).match(text, at, at + width)
    if not m or not m.group().lstrip('+-'):
        return None
    return int(m.group()), m.end()


def chapter_starts(comments, chapters):
    """FFmpeg's reading of CHAPTERxxx comments (ogm_chapter) into `chapters` ({number: start in seconds}): the key is
    9 or 10 characters and its number is read as %03d; the value as "%02d:%02d:%02d.%03d", all four fields or no
    chapter.  A later start with the same number replaces the earlier one; CHAPTERxxxNAME names one and is not a
    start."""
    for key, value in comments:
        if len(key) < 9 or len(key) > 10 or key[:7].upper() != 'CHAPTER':
            continue
        num = _scan_int(key, 7, 3)
        if num is None:
            continue
        fields, at = [], 0
        for width, sep in ((2, ':'), (2, ':'), (2, '.'), (3, '')):
            got = _scan_int(value, at, width)
            if got is None:
                break
            fields.append(got[0])
            at = got[1]
            if sep:
                if value[at:at + 1] != sep:
                    break
                at += 1
        if len(fields) < 4:
            continue
        h, m, sec, ms = fields
        chapters[num[0]] = (ms + 1000 * (sec + 60 * (m + 60 * h))) / 1000.0


class Stream(object):
    """One stream as FFmpeg lists it: `id` its index (FFmpeg's stream id), `serial` its serial number, `kind`,
    `codec` FFmpeg's codec name ('none' when there is none), `packets` its header packets read from the head."""

    def __init__(self, sid, serial, kind, codec):
        self.id, self.serial, self.kind, self.codec = sid, serial, kind, codec
        self.default = False
        self.title = ''
        self.packets = []
        self.frames_seen = False          # FLAC: a packet starting with a frame's sync byte was read

    @property
    def info(self):
        return '{0}, serial 0x{1:x}'.format(self.codec, self.serial)

    @property
    def script_type(self):
        return self.codec


class OggFile(Container):
    """The head of an Ogg file, its stream list and chapters."""
    no_timecodes = 'an Ogg file'        # what the command line says video timestamps cannot be read from

    def __init__(self, path):
        self.path = path
        self.size = os.path.getsize(path)
        self.tracks = []
        by_serial = {}
        open_packets = {}
        data_seen = False
        with open(path, 'rb') as f:
            if f.read(4) != b'OggS':
                raise SushiError('{0}: not an Ogg file (no capture pattern at its start)'.format(path))
            for at, flags, serial, seq, lacing, body in read_pages(f, min(self.size, HEAD_BYTES)):
                if flags & 2:
                    if data_seen:
                        raise SushiError('{0}: a new stream begins at byte offset {1} after the first data page '
                                         '(chained Ogg is not supported)'.format(path, at))
                    kind, codec = next((v for magic, v in MAPPINGS if body.startswith(magic)), ('data', 'none'))
                    s = Stream(len(self.tracks), serial, kind, codec)
                    self.tracks.append(s)
                    by_serial[serial] = s
                else:
                    data_seen = True
                s = by_serial.get(serial)
                if s is None:
                    continue
                # the page's packets, the first continuing the one the stream's last page left open
                pos = 0
                cur = open_packets.pop(serial, b'') if flags & 1 else b''
                for v in lacing:
                    cur += body[pos:pos + v]
                    pos += v
                    if v < 255:
                        self._packet(s, cur)
                        cur = b''
                if cur:                       # still open (a page without segments passes it on)
                    open_packets[serial] = cur
                if data_seen and all(t.frames_seen if t.codec == 'flac' else len(t.packets) >= 2 for t in self.tracks):
                    break
        if not self.tracks:
            raise SushiError('{0}: not an Ogg file (no stream begins at its start)'.format(path))
        chapters = {}
        for s in self.tracks:
            for comments in self._comments(s):
                chapter_starts(comments, chapters)
        self.chapters = [chapters[k] for k in chapters]

    @staticmethod
    def _packet(s, packet):
        if s.codec == 'flac':
            if s.frames_seen or (s.packets and packet[:1] == b'\xff'):
                s.frames_seen = True
            else:
                s.packets.append(packet)
        elif len(s.packets) < 3:
            s.packets.append(packet)

    @staticmethod
    def _comments(s):
        if s.codec == 'flac':
            for p in s.packets[1:]:
                if p[:1] and p[0] & 0x7F == 4:
                    yield vorbis_comments(p[4:])
        elif s.codec in COMMENTS:
            k, skip = COMMENTS[s.codec]
            if len(s.packets) > k:
                yield vorbis_comments(s.packets[k][skip:])

    def flac_info(self, s):
        """The STREAMINFO of a FLAC stream's mapping header, with the refusals flac.py makes; the old mapping refused"""
        first = s.packets[0] if s.packets else b''
        where = '{0}: stream {1}'.format(self.path, s.id)
        if first.startswith(b'fLaC'):
            raise SushiError('{0} uses the FLAC-in-Ogg mapping from before FLAC 1.1.1, which is not supported: remux '
                             'it with a current flac or ffmpeg first'.format(where))
        if len(first) < 13 or first[5:7] != b'\x01\x00' or first[9:13] != b'fLaC':
            raise SushiError('{0}: unsupported FLAC-in-Ogg mapping header (version {1}.{2})'.format(
                where, first[5] if len(first) > 5 else '?', first[6] if len(first) > 6 else '?'))
        if not s.frames_seen:
            raise SushiError('{0}: no FLAC frame in the first {1} bytes'.format(where, HEAD_BYTES))
        # STREAMINFO is read alone: the metadata blocks after it are the header packets
        info = FlacFile.from_bytes(first[9:13] + bytes([first[13] | 0x80]) + first[14:], where)
        info.check_depth()
        return info

    def select_audio(self, track=None):
        s = self.select('audio', track)
        if s.codec != 'flac':
            raise SushiError('Audio track {0} is {1}, which cannot be decoded here (FLAC can): convert it to FLAC or '
                             'WAV first'.format(s.id, s.codec))
        info = self.flac_info(s)
        return Audio('FLAC', s.id, self.path, decode=lambda device: self._decode(device, s, info),
                     **swr.audio_format(info.bits_per_sample, swr.FLAC))

    def _decode(self, device, s, info):
        """The FLAC stream `s`, demuxed and decoded on the GPU (sb_ogg_*) from chunks of CHUNK_BYTES."""
        args = (s.serial, info.channels_count, info.bits_per_sample, info.framerate, len(s.packets) - 1)
        h, cut, _ = _native.demux_file(device, 'sb_ogg', args, self.path, CHUNK_BYTES)
        if cut:
            logging.warning('{0}: stream {1} is cut short at the end of the file; the frames whose packets end before '
                            'the cut are kept'.format(self.path, s.id))
        return h
