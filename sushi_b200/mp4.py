"""ISO base media / QuickTime files on the host: `.mp4`, `.m4a`, `.m4v` and `.mov`.

The host reads the box structure (positioned reads; `moov` is read whole, `mdat` only where an audio track's chunks
lie), the stream list (ids, kinds, default flags and codec names as FFmpeg's mov demuxer gives them), the chapters and
the sample tables.  A track's sample table is expanded with NumPy into each sample's file offset and size, and its
bytes are read with one positioned read per run of file-contiguous chunks.  The audio is decoded on the GPU (ALAC,
FLAC) or goes to the PCM loader as it stands.

What is kept of FFmpeg's rules:
  - one stream per `trak` in `moov` order; the kind from the handler (`soun`, `vide`, `subp` / `clcp`) or, failing
    that, from the sample description's fourcc; a chapter track (named by the last `tref/chap`) that is not video is a
    data stream (`bin_data`); the default flag is the track header's `enabled` bit;
  - codec names from the sample description: `mp4a` by the object type indication of its `esds`, `lpcm` by its
    format flags, `sowt` / `twos` by bits per sample, `in24` with `enda` as little-endian, `ipcm` by its `pcmC`; anything unknown by its fourcc;
  - chapters: Nero `chpl` (time base 1/10^7), then the samples of the QuickTime chapter tracks named by `tref/chap`,
    which replace the `chpl` entries of the same index, as avpriv_new_chapter does.
Refused, naming the file, track, box or byte offset: a compressed `cmov`, a fragmented file (`mvex` / `moof`), a data
reference that is not self-contained, several sample descriptions, edit lists other than the identity, and damage
(a box running past its parent, a table count past its box, `stsc` naming chunks past `stco`, a sample count that
disagrees between `stsz` and `stsc`, a sample past the end of a file that is not cut).  A file cut inside `mdat`
after a whole `moov` keeps its whole samples (PCM: whole sample frames of a partial chunk), with a warning.
"""
import logging
import os
import struct

import numpy as np

from . import alac, flac, swr
from .common import Container, SushiError
from .matroska import FrameTable, track_audio, track_pcm

MP4_EXTENSIONS = ('.mp4', '.m4a', '.m4v', '.mov')
TOP_LEVEL = (b'ftyp', b'moov', b'mdat', b'free', b'skip', b'wide', b'uuid', b'pnot', b'meta', b'moof', b'mfra',
             b'styp', b'sidx', b'pdin')
# mp4a object type indication -> FFmpeg codec name
OBJECT_TYPES = {0x40: 'aac', 0x66: 'aac', 0x67: 'aac', 0x68: 'aac', 0x69: 'mp3', 0x6B: 'mp3', 0xA5: 'ac3',
                0xA6: 'eac3', 0xA9: 'dts', 0xAD: 'opus', 0xDD: 'vorbis', 0xE1: 'qcelp', 0x6D: 'alac', 0xF1: 'flac'}
AUDIO_FOURCC = {b'alac': 'alac', b'fLaC': 'flac', b'sowt': 'pcm_s16le', b'twos': 'pcm_s16be', b'in24': 'pcm_s24be',
                b'in32': 'pcm_s32be', b'fl32': 'pcm_f32be', b'fl64': 'pcm_f64be', b'raw ': 'pcm_u8', b'NONE': 'pcm_u8',
                b'ulaw': 'pcm_mulaw', b'alaw': 'pcm_alaw', b'ac-3': 'ac3', b'ec-3': 'eac3', b'Opus': 'opus',
                b'mlpa': 'truehd', b'.mp3': 'mp3', b'samr': 'amr_nb', b'dtsc': 'dts', b'ima4': 'adpcm_ima_qt'}
VIDEO_FOURCC = {b'avc1': 'h264', b'avc3': 'h264', b'hvc1': 'hevc', b'hev1': 'hevc', b'mp4v': 'mpeg4',
                b'av01': 'av1', b'vp09': 'vp9', b'apch': 'prores', b'apcn': 'prores', b'apcs': 'prores',
                b'apco': 'prores', b'ap4h': 'prores', b'jpeg': 'mjpeg', b'AVdh': 'dnxhd', b'AVdn': 'dnxhd'}
SUB_FOURCC = {b'tx3g': 'mov_text', b'text': 'mov_text', b'c608': 'eia_608', b'wvtt': 'webvtt', b'stpp': 'ttml'}
HANDLER_KINDS = {b'vide': 'video', b'soun': 'audio', b'subp': 'subtitles', b'clcp': 'subtitles'}
PCM_DECODED = {'pcm_s16le': (2, False), 'pcm_s16be': (2, True), 'pcm_s24le': (3, False), 'pcm_s24be': (3, True)}


def is_mp4(path):
    """True when the file starts with a box FFmpeg's mov demuxer opens (`ftyp`, or for old QuickTime files `moov`,
    `mdat`, `free`, `skip`, `wide`, `pnot`) of a plausible size (False when it cannot be read)."""
    try:
        with open(path, 'rb') as f:
            head = f.read(8)
    except OSError:
        return False
    # a RIFF WAV's size field can spell a box name (files of about 1.7 to 2 GB): those stay WAV files
    if len(head) < 8 or head[:4] == b'RIFF' or head[4:8] not in (b'ftyp', b'moov', b'mdat', b'free', b'skip', b'wide',
                                                                  b'pnot'):
        return False
    size = struct.unpack('>I', head[:4])[0]
    return size in (0, 1) or size >= 8


class Box(object):
    __slots__ = ('type', 'start', 'body', 'end')

    def __init__(self, btype, start, body, end):
        self.type, self.start, self.body, self.end = btype, start, body, end


def _boxes(data, at, end, base, where):
    """The boxes of data[at:end) (base: the file offset of data[0]); a box running past its parent is damage."""
    while at + 8 <= end:
        size, btype = struct.unpack('>I4s', data[at:at + 8])
        head = 8
        if size == 1:
            if at + 16 > end:
                raise SushiError('{0}: box {1} at byte offset {2} runs past its parent'.format(where, _t(btype), base + at))
            size = struct.unpack('>Q', data[at + 8:at + 16])[0]
            head = 16
        elif size == 0:
            size = end - at
        if size < head or at + size > end:
            raise SushiError('{0}: box {1} at byte offset {2} runs past its parent'.format(where, _t(btype), base + at))
        yield Box(btype, base + at, at + head, at + size)
        at += size
    if at != end and end - at < 8 and any(data[at:end]):
        raise SushiError('{0}: box at byte offset {1} runs past its parent'.format(where, base + at))


def _t(btype):
    return "'" + btype.decode('latin-1') + "'"


class Track(object):
    """One `trak`: `id` is the stream id (trak order)."""

    def __init__(self, sid):
        self.id = sid
        self.track_id = 0
        self.kind, self.codec, self.fourcc = 'other', 'none', b''
        self.default = False
        self.title = ''
        self.handler = b''
        self.timescale = 1
        self.channels = self.bits = self.rate = 0
        self.config = None          # ALAC: the 24-byte ALACSpecificConfig; FLAC: the STREAMINFO block
        self.frame_bytes = 0        # PCM: bytes per sample frame
        self.refusal = None
        self.edits = None
        self.media_duration = 0
        self.chap = []
        self.table = None           # (chunk offsets, samples per chunk, sample sizes or None, constant size)
        self.stts = None

    @property
    def info(self):
        parts = [self.codec]
        if self.kind == 'audio':
            parts += ['{0} channels'.format(self.channels), '{0} Hz'.format(self.rate)]
        return ', '.join(parts) + (' (default)' if self.default else '')

    @property
    def script_type(self):
        return '.' + self.codec


class Mp4File(Container):
    """The box structure of an MP4 / QuickTime file."""
    no_timecodes = 'an MP4 file'                # what the command line says video timestamps cannot be read from

    def __init__(self, path):
        self.path = path
        self._f = open(path, 'rb', buffering=0)
        self.bytes_read = 0
        try:
            self.size = os.fstat(self._f.fileno()).st_size
            self._read_top()
        except Exception:
            self.close()
            raise

    def close(self):
        if self._f is not None:
            self._f.close()
        self._f = None

    def _read(self, pos, n):
        b = os.pread(self._f.fileno(), max(0, min(n, self.size - pos)), pos)
        self.bytes_read += len(b)
        return b

    # -- top level --------------------------------------------------------------------------------------------------
    def _read_top(self):
        pos, moov = 0, None
        self.cut = False
        self.movie_timescale = 1
        while pos + 8 <= self.size:
            head = self._read(pos, 16)
            size, btype = struct.unpack('>I4s', head[:8])
            hl = 8
            if size == 1:
                size = struct.unpack('>Q', head[8:16])[0]
                hl = 16
            elif size == 0:
                size = self.size - pos
            if btype not in TOP_LEVEL and pos == 0:
                raise SushiError('{0}: not an MP4 / QuickTime file'.format(self.path))
            if size < hl:
                raise SushiError('{0}: box {1} at byte offset {2} has a size of {3}'.format(self.path, _t(btype), pos,
                                                                                           size))
            if btype in (b'moof', b'mfra'):
                raise SushiError('{0}: fragmented MP4 files are not supported'.format(self.path))
            if pos + size > self.size:
                if btype == b'moov' or moov is None and btype != b'mdat':
                    raise SushiError('{0}: box {1} at byte offset {2} runs past the end of the file'.format(
                        self.path, _t(btype), pos))
                self.cut = True
                logging.warning('{0}: the file ends inside box {1} at byte offset {2}; its whole samples are '
                                'kept'.format(self.path, _t(btype), pos))
            if btype == b'moov':
                if moov is not None:
                    raise SushiError('{0}: a second moov box at byte offset {1}'.format(self.path, pos))
                moov = (pos, self._read(pos, size), hl)
            pos += size
        if pos < self.size and pos + 8 > self.size:
            self.cut = True
        if moov is None:
            raise SushiError('{0}: no moov box'.format(self.path))
        try:
            self._read_moov(*moov)
        except (struct.error, IndexError, ValueError) as e:
            # a field no check above names; still damage, not a crash
            raise SushiError('{0}: moov box at byte offset {1} is damaged ({2})'.format(self.path, moov[0], e))

    def _field(self, data, b, off, fmt):
        """struct.unpack(fmt) of the bytes at `off` of box b's body; SushiError naming the box when they run past it."""
        at = b.body + off
        if at < b.body or at + struct.calcsize(fmt) > b.end:
            raise SushiError('{0}: box {1} at byte offset {2} is too short for its fields'.format(self.path, _t(b.type),
                                                                                                 b.start))
        return struct.unpack(fmt, data[at:at + struct.calcsize(fmt)])

    def _read_moov(self, base, data, hl):
        self.tracks, self.chpl = [], []
        where = self.path
        for b in _boxes(data, hl, len(data), base, where):
            if b.type == b'cmov':
                raise SushiError('{0}: compressed movie header (cmov) is not supported'.format(self.path))
            if b.type == b'mvex':
                raise SushiError('{0}: fragmented MP4 files are not supported'.format(self.path))
            if b.type == b'mvhd':
                v = self._field(data, b, 0, 'B')[0]
                self.movie_timescale = self._field(data, b, 20 if v == 1 else 12, '>I')[0] or 1
            elif b.type == b'trak':
                t = Track(len(self.tracks))
                self.tracks.append(t)
                self._read_trak(t, data, b, base)
            elif b.type == b'udta':
                for u in _boxes(data, b.body, b.end, base, where):
                    if u.type == b'chpl':
                        self._read_chpl(data, u)
        # the chapter tracks: those the last `tref/chap` names (each one replaces the list before it, as in FFmpeg).
        # FFmpeg turns every one that is not video into a data stream and takes the chapters from its samples
        self.chapter_tracks = []
        for t in self.tracks:
            if t.chap:
                self.chapter_tracks = list(t.chap)
        for tid in self.chapter_tracks:
            for t in self.tracks:
                if t.track_id == tid and t.kind != 'video':
                    t.kind, t.codec = 'data', 'bin_data'

    def _read_chpl(self, data, b):
        body = data[b.body:b.end]
        at = 4 + (4 if self._field(data, b, 0, 'B')[0] else 0)
        n = self._field(data, b, at, 'B')[0]
        at += 1
        self.chpl = []
        for _ in range(n):
            if at + 9 > len(body) or at + 9 + body[at + 8] > len(body):
                raise SushiError('{0}: chpl box at byte offset {1}: a chapter runs past the box'.format(self.path,
                                                                                                       b.start))
            start = struct.unpack('>Q', body[at:at + 8])[0]
            at += 9 + body[at + 8]
            self.chpl.append(start)

    def _read_trak(self, t, data, trak, base):
        where = self.path
        for b in _boxes(data, trak.body, trak.end, base, where):
            if b.type == b'tkhd':
                v, f0, flags = self._field(data, b, 0, '>BBH')
                t.default = bool(flags & 1)
                t.track_id = self._field(data, b, 20 if v == 1 else 12, '>I')[0]
            elif b.type == b'tref':
                for r in _boxes(data, b.body, b.end, base, where):
                    if r.type == b'chap':
                        t.chap = list(struct.unpack('>%dI' % ((r.end - r.body) // 4), data[r.body:r.end]))
            elif b.type == b'edts':
                for e in _boxes(data, b.body, b.end, base, where):
                    if e.type == b'elst':
                        t.edits = self._read_elst(data, e, t)
            elif b.type == b'mdia':
                self._read_mdia(t, data, b, base)

    def _read_elst(self, data, b, t):
        v, n = self._field(data, b, 0, '>B3xI')
        row = 20 if v == 1 else 12
        if b.body + 8 + n * row > b.end:
            raise SushiError('{0}: elst box at byte offset {1}: {2} entries run past the box'.format(self.path, b.start,
                                                                                                    n))
        out = []
        for k in range(n):
            at = b.body + 8 + k * row
            if v == 1:
                dur, mt = struct.unpack('>Qq', data[at:at + 16])
                rate = struct.unpack('>i', data[at + 16:at + 20])[0]
            else:
                dur, mt, rate = struct.unpack('>Iii', data[at:at + 12])
            out.append((dur, mt, rate))
        return out

    def _read_mdia(self, t, data, mdia, base):
        where = self.path
        for b in _boxes(data, mdia.body, mdia.end, base, where):
            if b.type == b'mdhd':
                v = self._field(data, b, 0, 'B')[0]
                if v == 1:
                    t.timescale, t.media_duration = self._field(data, b, 20, '>IQ')
                else:
                    t.timescale, t.media_duration = self._field(data, b, 12, '>II')
                t.timescale = t.timescale or 1
            elif b.type == b'hdlr':
                t.handler = self._field(data, b, 8, '4s')[0]
                t.kind = HANDLER_KINDS.get(t.handler, 'other')
            elif b.type == b'minf':
                for m in _boxes(data, b.body, b.end, base, where):
                    if m.type == b'dinf':
                        self._read_dinf(t, data, m, base)
                    elif m.type == b'stbl':
                        self._read_stbl(t, data, m, base)

    def _read_dinf(self, t, data, dinf, base):
        for d in _boxes(data, dinf.body, dinf.end, base, self.path):
            if d.type != b'dref':
                continue
            self._field(data, d, 0, '>II')
            for r in _boxes(data, d.body + 8, d.end, base, self.path):
                flags = self._field(data, r, 0, '>I')[0] & 0xFFFFFF
                if not flags & 1 and t.refusal is None:
                    t.refusal = 'track {0} refers to its media in another file, which is not supported'.format(t.id)

    def _count(self, data, b, row, extra=0):
        n = self._field(data, b, 4 + extra, '>I')[0]
        if b.body + 8 + extra + n * row > b.end:
            raise SushiError('{0}: {1} box at byte offset {2}: {3} entries run past the box'.format(
                self.path, b.type.decode('latin-1'), b.start, n))
        return n

    def _read_stbl(self, t, data, stbl, base):
        chunks = spc = sizes = None
        const = 0
        for b in _boxes(data, stbl.body, stbl.end, base, self.path):
            if b.type == b'stsd':
                self._read_stsd(t, data, b, base)
            elif b.type == b'stts':
                n = self._count(data, b, 8)
                t.stts = np.frombuffer(data, '>u4', 2 * n, b.body + 8).reshape(n, 2).astype(np.int64)
            elif b.type == b'stsc':
                n = self._count(data, b, 12)
                stsc = np.frombuffer(data, '>u4', 3 * n, b.body + 8).reshape(n, 3).astype(np.int64)
                spc = (stsc, b.start)
            elif b.type == b'stsz':
                const, n = self._field(data, b, 4, '>II')
                if const == 0:
                    if b.body + 12 + 4 * n > b.end:
                        raise SushiError('{0}: stsz box at byte offset {1}: {2} entries run past the box'.format(
                            self.path, b.start, n))
                    sizes = np.frombuffer(data, '>u4', n, b.body + 12).astype(np.int64)
                else:
                    sizes = np.full(n, const, np.int64)
                sizes = (sizes, b.start)
            elif b.type == b'stz2':
                field, n = self._field(data, b, 7, '>BI')
                if field not in (4, 8, 16) or b.body + 12 + (n * field + 7) // 8 > b.end:
                    raise SushiError('{0}: stz2 box at byte offset {1}: {2} entries of {3} bits run past the box'.format(
                        self.path, b.start, n, field))
                raw = np.frombuffer(data, np.uint8, (n * field + 7) // 8, b.body + 12)
                if field == 16:
                    s = raw.view('>u2').astype(np.int64)
                elif field == 8:
                    s = raw.astype(np.int64)
                else:
                    s = np.stack([raw >> 4, raw & 15], 1).reshape(-1)[:n].astype(np.int64)
                sizes = (s, b.start)
            elif b.type in (b'stco', b'co64'):
                n = self._count(data, b, 4 if b.type == b'stco' else 8)
                chunks = np.frombuffer(data, '>u4' if b.type == b'stco' else '>u8', n, b.body + 8).astype(np.int64)
                chunks = (chunks, b.start)
        t.table = (chunks, spc, sizes)

    def _read_stsd(self, t, data, b, base):
        n = self._field(data, b, 4, '>I')[0]
        entries = list(_boxes(data, b.body + 8, b.end, base, self.path))
        if n != 1 or len(entries) != 1:
            t.refusal = 'track {0} has {1} sample descriptions; only one is supported'.format(t.id, n)
            if not entries:
                return
        e = entries[0]
        t.fourcc = e.type
        if t.kind == 'audio' or (t.kind == 'other' and e.type in AUDIO_FOURCC):
            t.kind = 'audio'
            self._read_sound(t, data, e, base)
        elif e.type in VIDEO_FOURCC:
            t.codec = VIDEO_FOURCC[e.type]
            t.kind = 'video' if t.kind == 'other' else t.kind
        elif e.type in SUB_FOURCC:
            t.codec = SUB_FOURCC[e.type]
            t.kind = 'subtitles' if t.kind == 'other' else t.kind
        else:
            t.codec = e.type.decode('latin-1').strip()

    def _read_sound(self, t, data, e, base):
        """The ISO form, QuickTime v0 / v1 (four extra fields) / v2 (`lpcm`), with the `wave` wrapper."""
        # offsets into the entry's body: reserved, data reference index, then the version
        version = self._field(data, e, 8, '>H')[0]
        if version == 2:
            # always 3, 16, -2, 0, 65536, then sizeOfStructOnly, rate (f64), channels, 0x7F000000, bits, flags,
            # bytes per audio packet, frames per audio packet
            rate, channels = self._field(data, e, 32, '>dI')
            bits, flags, bpp, fpp = self._field(data, e, 48, '>IIII')
            t.rate, t.channels, t.bits = int(rate), channels, bits
            kids = e.body + 64
            t.lpcm_flags = flags
        else:
            channels, bits = self._field(data, e, 16, '>HH')
            rate = self._field(data, e, 24, '>I')[0] >> 16
            t.rate, t.channels, t.bits = rate, channels, bits
            kids = e.body + 28 + (16 if version == 1 else 0)
            self._field(data, e, kids - e.body - 4, '>I')
        fourcc = e.type
        children = {}
        self._sound_children(data, kids, e.end, base, children)
        if b'frma' in children:
            fourcc = children[b'frma']
        t.fourcc = fourcc
        codec = AUDIO_FOURCC.get(fourcc)
        if fourcc == b'mp4a':
            codec = OBJECT_TYPES.get(children.get(b'esds_oti'), 'aac')
        elif fourcc in (b'twos', b'sowt') and t.bits != 16:
            # FFmpeg maps these by bits per sample: 8 -> s8, 24 -> s24, 32 -> s32, in the fourcc's byte order
            endian = 'be' if fourcc == b'twos' else 'le'
            codec = {8: 'pcm_s8', 24: 'pcm_s24' + endian, 32: 'pcm_s32' + endian}.get(t.bits, codec)
        elif fourcc == b'in24' and children.get(b'enda'):
            codec = 'pcm_s24le'
        elif fourcc == b'in32' and children.get(b'enda'):
            codec = 'pcm_s32le'
        elif fourcc == b'lpcm':
            flags = getattr(t, 'lpcm_flags', 0)
            kind = 'f' if flags & 1 else ('s' if flags & 4 else 'u')
            codec = 'pcm_%s%d%s' % (kind, t.bits, 'be' if flags & 2 else 'le') if t.bits > 8 else 'pcm_%s8' % kind
        elif fourcc == b'ipcm':
            pcmc = children.get(b'pcmC')
            if pcmc is not None:
                little, size = pcmc
                t.bits = size
                codec = 'pcm_s%d%s' % (size, 'le' if little else 'be')
            else:
                codec = 'none'
        if codec is None:
            codec = fourcc.decode('latin-1').strip()
        t.codec = codec
        if codec == 'alac':
            cookie = children.get(b'alac')
            if cookie is None or len(cookie) < 24:
                t.refusal = 'track {0}: ALAC without its configuration box'.format(t.id)
            else:
                t.config = cookie[:24]
        elif codec == 'flac':
            t.config = children.get(b'dfLa')
            if t.config is None:
                t.refusal = 'track {0}: FLAC without its dfLa box'.format(t.id)
        if codec in PCM_DECODED:
            t.frame_bytes = PCM_DECODED[codec][0] * t.channels

    def _sound_children(self, data, at, end, base, out):
        for c in _boxes(data, at, end, base, self.path):
            if c.type == b'wave':
                self._sound_children(data, c.body, c.end, base, out)
            elif c.type == b'frma':
                out[b'frma'] = self._field(data, c, 0, '4s')[0]
            elif c.type == b'enda':
                out[b'enda'] = bool(self._field(data, c, 0, '>H')[0])
            elif c.type == b'alac':
                body = data[c.body:c.end]
                # inside `wave` QuickTime repeats the box header: version / flags come first either way
                out[b'alac'] = body[4:] if len(body) >= 28 else body
            elif c.type == b'dfLa':
                out[b'dfLa'] = b'fLaC' + data[c.body + 4:c.end]
            elif c.type == b'pcmC':
                flags, size = self._field(data, c, 4, 'BB')
                out[b'pcmC'] = (flags & 1, size)
            elif c.type == b'esds':
                out[b'esds_oti'] = _esds_oti(data[c.body + 4:c.end])

    # -- streams ----------------------------------------------------------------------------------------------------
    def track(self, sid):
        for t in self.tracks:
            if t.id == sid:
                return t
        raise SushiError("Stream with index {0} doesn't exist in {1}".format(sid, self.path))

    def select_audio(self, track=None):
        """The audio track `track` (a stream id; None: the reference's default rule)."""
        t = self.select('audio', track)
        kind = audio_codec(t)
        self.check_edits(t)
        if kind == 'pcm':
            return track_pcm(self.path, t.id, lambda: self.frames(t), t.channels, t.rate, *PCM_DECODED[t.codec])
        if kind == 'flac':
            name = '{0} track {1}'.format(self.path, t.id)
            label, decode = 'FLAC', flac.track_decoder(t.config, name)
            fields = swr.audio_format(flac.FlacFile.from_bytes(t.config, name).bits_per_sample, swr.FLAC)
        else:
            label, decode = 'ALAC', alac.track_decoder(t.config)
            fields = swr.audio_format(alac.bit_depth(t.config), swr.ALAC)
        return track_audio(self.path, t.id, label, lambda: self.frames(t), decode, **fields)

    def script_text(self, track):
        raise SushiError('Unknown script type')

    @property
    def chapters(self):
        """Chapter start times in seconds, as the reference parses them out of ffmpeg's `start %f` text."""
        starts = [s / 1e7 for s in self.chpl]
        for tid in self.chapter_tracks:
            for t in self.tracks:
                if t.track_id != tid or t.kind != 'data' or t.stts is None or not len(t.stts):
                    continue
                times = np.concatenate([[0], np.cumsum(np.repeat(t.stts[:, 1], t.stts[:, 0]))])[:-1]
                for i, v in enumerate(times):
                    s = float(v) / t.timescale
                    if i < len(starts):
                        starts[i] = s
                    else:
                        starts.append(s)
        return [float('%f' % s) for s in starts]

    # -- samples ----------------------------------------------------------------------------------------------------
    def check_edits(self, t):
        """The identity edit list only: none, or one edit at rate 1 from media time 0 covering the whole track."""
        if not t.edits:
            return
        if len(t.edits) == 1:
            dur, mt, rate = t.edits[0]
            total = int(t.stts[:, 0] @ t.stts[:, 1]) if t.stts is not None and len(t.stts) else t.media_duration
            covered = (dur * t.timescale + self.movie_timescale // 2) // self.movie_timescale
            if mt == 0 and rate == 0x10000 and covered >= total:
                return
        raise SushiError('{0}: track {1} has an edit list that trims or shifts it ({2}), which is not supported: '
                         'remux it without one'.format(self.path, t.id, ', '.join(
                             'duration {0} from media time {1} at rate {2:g}'.format(d, m, r / 65536.0)
                             for d, m, r in t.edits)))

    def samples(self, t):
        """(file offsets, sizes) of every sample of track t (PCM: one entry per chunk)."""
        chunks, spc, sizes = t.table
        if chunks is None or spc is None or (sizes is None and not t.frame_bytes):
            raise SushiError('{0}: track {1} has no complete sample table'.format(self.path, t.id))
        chunk_off, chunk_box = chunks
        stsc, stsc_box = spc
        n_chunks = len(chunk_off)
        first = stsc[:, 0]
        if len(stsc) and (first[0] != 1 or np.any(np.diff(first) <= 0) or first[-1] > n_chunks or
                          np.any(stsc[:, 1] == 0)):
            raise SushiError('{0}: stsc box at byte offset {1} names chunks past the {2} of the stco box'.format(
                self.path, stsc_box, n_chunks) if len(stsc) and first[-1] > n_chunks else
                '{0}: stsc box at byte offset {1}: invalid chunk runs'.format(self.path, stsc_box))
        runs = np.diff(np.append(first, n_chunks + 1))
        per_chunk = np.repeat(stsc[:, 1], runs) if len(stsc) else np.zeros(0, np.int64)
        if t.frame_bytes:
            # QuickTime PCM: a sample is one frame; ISO ipcm: a sample is stsz's constant size
            unit = int(sizes[0][0]) if t.fourcc == b'ipcm' and sizes is not None and len(sizes[0]) else t.frame_bytes
            return chunk_off, per_chunk * unit
        size, size_box = sizes
        if int(per_chunk.sum()) != len(size):
            raise SushiError('{0}: track {1}: the stsz box at byte offset {2} lists {3} samples, the stsc box at byte '
                             'offset {4} {5}'.format(self.path, t.id, size_box, len(size), stsc_box,
                                                     int(per_chunk.sum())))
        excl = np.cumsum(size) - size
        chunk_first = np.cumsum(per_chunk) - per_chunk
        within = excl - np.repeat(excl[chunk_first[per_chunk > 0]], per_chunk[per_chunk > 0])
        return np.repeat(chunk_off, per_chunk) + within, size

    def frames(self, t):
        """A FrameTable of track t's samples (PCM: of its chunks), their bytes back to back; `block` holds each
        sample's file offset.  A cut file keeps its whole samples (PCM: the whole sample frames of a partial
        chunk), with a warning."""
        off, size = self.samples(t)
        end = off + size
        past = np.nonzero(end > self.size)[0]
        if len(past):
            k = int(past[0])
            if not self.cut:
                raise SushiError('{0}: track {1}: sample {2} at byte offset {3} lies past the end of the file'.format(
                    self.path, t.id, k, int(off[k])))
            if t.frame_bytes and off[k] < self.size:
                size = size[:k + 1].copy()
                size[k] = (self.size - off[k]) // t.frame_bytes * t.frame_bytes
                off = off[:k + 1]
            else:
                off, size = off[:k], size[:k]
            logging.warning('{0}: the file is cut: track {1} keeps {2} of its samples'.format(self.path, t.id,
                                                                                           'whole sample frames'
                                                                                           if t.frame_bytes else
                                                                                           '{0}'.format(len(off))))
        # one read per run of file-contiguous samples
        if len(off):
            brk = np.nonzero(off[1:] != off[:-1] + size[:-1])[0] + 1
            starts = np.concatenate([[0], brk])
            stops = np.concatenate([brk, [len(off)]])
            pieces = [self._read(int(off[a]), int(off[b - 1] + size[b - 1] - off[a])) for a, b in zip(starts, stops)]
        else:
            pieces = []
        table = FrameTable.__new__(FrameTable)
        table.data = b''.join(pieces)
        table.size = size.astype(np.int64)
        table.offset = (np.cumsum(table.size) - table.size).astype(np.int64)
        table.block = off.astype(np.int64)
        table.time = np.zeros(len(off), np.int64)
        table.duration = np.zeros(len(off), np.int64)
        return table


def _esds_oti(body):
    """The objectTypeIndication of an ES_Descriptor's DecoderConfigDescriptor (None when there is none)."""
    def desc(at):
        tag = body[at]
        at += 1
        n = 0
        for _ in range(4):
            b = body[at]
            at += 1
            n = (n << 7) | (b & 0x7F)
            if not b & 0x80:
                break
        return tag, at, n
    try:
        tag, at, n = desc(0)
        if tag != 3:
            return None
        flags = body[at + 2]
        at += 3
        if flags & 0x80:
            at += 2
        if flags & 0x40:
            at += 1 + body[at]
        if flags & 0x20:
            at += 2
        tag, at, n = desc(at)
        return body[at] if tag == 4 else None
    except IndexError:
        return None


def audio_codec(track):
    """'alac', 'flac' or 'pcm' for an audio track the loader decodes (ALAC, FLAC, 16- or 24-bit integer PCM in either
    byte order); SushiError naming the track and FFmpeg's codec name for anything else."""
    if track.refusal:
        raise SushiError(track.refusal)
    if track.codec in ('alac', 'flac'):
        return track.codec
    if track.codec in PCM_DECODED and track.channels >= 1:
        return 'pcm'
    raise SushiError('Audio track {0} is {1}, which cannot be decoded here (ALAC, FLAC and 16- or 24-bit PCM can): '
                     'convert it to FLAC or WAV first'.format(track.id, track.codec))
