"""Matroska / WebM input: the container walk the reference gets from ffmpeg and mkvextract (demux.py).

`MatroskaFile(path)` reads the EBML header, the segment's Info, Tracks and Chapters and notes where its clusters are;
SeekHead, Cues, Tags and Attachments are skipped.  `frames(ids)` then walks the clusters and reads the payloads of the
requested tracks only: every other block costs one small positioned read of its header, so a video track's payload
is never read.  What comes out:

* tracks with the reference's stream ids (FFmpeg's stream indices: TrackEntry order, 0-based) and `select`, the
  reference's Demuxer._select_stream (demux.py:335-355);
* per requested track, its frames back to back in one buffer with a table of (buffer offset, size, file offset of
  the block, timestamp, duration), after lacing (Xiph, EBML, fixed) and content encodings (header stripping, zlib);
* the chapter start times ffmpeg lists (`Chapter #0.N: start %f`, demux.py:77-78);
* an embedded ASS / SSA / SRT script as text, and a video track's timestamps as a v2 timecodes file.

A block cut short by the end of the file is dropped with a warning and everything before it loads; a size that runs
past its parent, or a lace table that runs past its block, raises SushiError naming the byte offset.  Audio decoding
is not here: WavStream hands a FLAC or PCM track's frames to the GPU (sb_flac_decode_frames / sb_load_pcm).
"""
import io
import logging
import os
import struct
import zlib

import numpy as np

from .common import SushiError, py2_round, select_stream

EBML_MAGIC = b'\x1a\x45\xdf\xa3'

# element ids, marker bits included
ID_EBML, ID_DOCTYPE, ID_DOCTYPE_READ_VERSION = 0x1A45DFA3, 0x4282, 0x4285
ID_SEGMENT = 0x18538067
ID_SEEKHEAD, ID_INFO, ID_TRACKS, ID_CHAPTERS = 0x114D9B74, 0x1549A966, 0x1654AE6B, 0x1043A770
ID_CLUSTER, ID_CUES, ID_TAGS, ID_ATTACHMENTS = 0x1F43B675, 0x1C53BB6B, 0x1254C367, 0x1941A469
ID_VOID, ID_CRC32 = 0xEC, 0xBF
ID_TIMESTAMP_SCALE = 0x2AD7B1
ID_TRACK_ENTRY, ID_TRACK_NUMBER, ID_TRACK_TYPE, ID_CODEC_ID, ID_CODEC_PRIVATE = 0xAE, 0xD7, 0x83, 0x86, 0x63A2
ID_FLAG_DEFAULT, ID_NAME, ID_LANGUAGE, ID_DEFAULT_DURATION = 0x88, 0x536E, 0x22B59C, 0x23E383
ID_AUDIO, ID_SAMPLING_FREQUENCY, ID_CHANNELS, ID_BIT_DEPTH = 0xE1, 0xB5, 0x9F, 0x6264
ID_CONTENT_ENCODINGS, ID_CONTENT_ENCODING, ID_ENCODING_ORDER, ID_ENCODING_SCOPE = 0x6D80, 0x6240, 0x5031, 0x5032
ID_ENCODING_TYPE, ID_COMPRESSION, ID_COMP_ALGO, ID_COMP_SETTINGS, ID_ENCRYPTION = 0x5033, 0x5034, 0x4254, 0x4255, 0x5035
ID_CLUSTER_TIMESTAMP, ID_SIMPLE_BLOCK, ID_BLOCK_GROUP, ID_BLOCK, ID_BLOCK_DURATION = 0xE7, 0xA3, 0xA0, 0xA1, 0x9B
ID_EDITION_ENTRY, ID_CHAPTER_ATOM, ID_CHAPTER_UID, ID_CHAPTER_TIME_START = 0x45B9, 0xB6, 0x73C4, 0x91

# what ends a cluster of unknown size: the next element of the segment's level
SEGMENT_CHILDREN = {ID_SEEKHEAD, ID_INFO, ID_TRACKS, ID_CHAPTERS, ID_CLUSTER, ID_CUES, ID_TAGS, ID_ATTACHMENTS}
TRACK_KINDS = {1: 'video', 2: 'audio', 17: 'subtitles'}
# FFmpeg gives a stream (and so a stream id) only to TrackEntries of these types that have a CodecID
STREAM_TYPES = (1, 2, 17, 0x21)
# the reference's subtitle types (demux.py:82-86): ffmpeg's codec names ssa / ass / subrip
SCRIPT_TYPES = {'S_TEXT/ASS': '.ass', 'S_TEXT/SSA': '.ass', 'S_TEXT/UTF8': '.srt'}
HEAD = 32           # bytes read for an element header: id (4) + size (8) + a block's track, timestamp and flags (11)


def read_id(buf, at):
    """(element id with its marker bits, length) of the id at buf[at], or None when buf ends inside it."""
    if at >= len(buf):
        return None
    b = buf[at]
    n = 1 if b & 0x80 else 2 if b & 0x40 else 3 if b & 0x20 else 4 if b & 0x10 else 0
    if n == 0:
        raise ValueError('invalid element id')
    if at + n > len(buf):
        return None
    return int.from_bytes(buf[at:at + n], 'big'), n


def read_vint(buf, at):
    """(value, length) of the variable-size integer at buf[at]; the value is None for the reserved all-ones value (an
    unknown size).  None when buf ends inside it."""
    if at >= len(buf):
        return None
    b = buf[at]
    if b == 0:
        raise ValueError('invalid variable-size integer')
    n = 9 - b.bit_length()
    if at + n > len(buf):
        return None
    v = int.from_bytes(buf[at:at + n], 'big') & ((1 << (7 * n)) - 1)
    return (None if v == (1 << (7 * n)) - 1 else v), n


def _uint(b):
    return int.from_bytes(b, 'big') if b else 0


def _float(b):
    if len(b) == 4:
        return struct.unpack('>f', b)[0]
    if len(b) == 8:
        return struct.unpack('>d', b)[0]
    return 0.0


def _text(b):
    return b.split(b'\0', 1)[0].decode('utf-8', 'replace')


def children(data, where=0):
    """(id, payload, file offset of the element) of every child of a master element held in memory, Void and CRC-32
    skipped; `where` is the file offset of data[0] (for messages)."""
    at, end = 0, len(data)
    while at < end:
        try:
            head = read_id(data, at)
            size = read_vint(data, at + head[1]) if head else None
        except ValueError as e:
            raise SushiError('Matroska element at byte {0}: {1}'.format(where + at, e))
        if head is None or size is None or size[0] is None:
            raise SushiError('Matroska element at byte {0} runs past its parent'.format(where + at))
        body = at + head[1] + size[1]
        if body + size[0] > end:
            raise SushiError('Matroska element at byte {0} runs past its parent'.format(where + at))
        if head[0] not in (ID_VOID, ID_CRC32):
            yield head[0], data[body:body + size[0]], where + at
        at = body + size[0]


class Track(object):
    """One TrackEntry.  `id` is the stream id (TrackEntry order); `refusal` says why its frames cannot be read."""

    def __init__(self, sid):
        self.id = sid
        self.number = self.type = None
        self.codec_id, self.codec_private = '', b''
        self.default, self.name, self.language = True, '', 'eng'
        self.default_duration = 0
        self.sampling_frequency, self.channels, self.bit_depth = 8000.0, 1, 0
        self.encodings = []             # (order, scope, kind, algo, settings) in file order
        self.refusal = None

    @property
    def kind(self):
        return TRACK_KINDS.get(self.type, 'other')

    @property
    def title(self):
        return self.name

    @property
    def info(self):
        """What a candidate list shows of the stream (ffmpeg's info line does not exist here)."""
        parts = [self.codec_id or 'no codec', self.language]
        if self.kind == 'audio':
            parts += ['{0} channels'.format(self.channels), '{0:g} Hz'.format(self.sampling_frequency)]
        return ', '.join(parts) + (' (default)' if self.default else '')

    @property
    def script_type(self):
        return SCRIPT_TYPES.get(self.codec_id, self.codec_id)

    def decode_frame(self, data):
        """A frame's bytes after the track's content encodings (the last one applied first)."""
        for _, scope, _, algo, settings in sorted(self.encodings, key=lambda e: -e[0]):
            if not scope & 1:
                continue
            if algo == 3:
                data = settings + data
            else:
                data = zlib.decompress(data)
        return data


class FrameTable(object):
    """A track's frames: `data` holds their bytes back to back, frame i at data[offset[i]:offset[i] + size[i]]; `block`
    is the file offset of the (Simple)Block holding it, `time` and `duration` are in nanoseconds."""

    def __init__(self, pieces, rows):
        self.data = b''.join(pieces)
        rows = np.array(rows, np.int64).reshape(-1, 4)
        self.size = rows[:, 0].copy()
        self.offset = np.concatenate([[0], np.cumsum(self.size)[:-1]]).astype(np.int64) if len(rows) else self.size.copy()
        self.block, self.time, self.duration = rows[:, 1].copy(), rows[:, 2].copy(), rows[:, 3].copy()

    def __len__(self):
        return len(self.size)

    def refuse_empty(self, path, what):
        """SushiError naming the first empty frame (a zero-size lace) and the file offset of its block."""
        empty = np.nonzero(self.size == 0)[0]
        if len(empty):
            f = int(empty[0])
            raise SushiError('{0}: {1} frame {2} at byte offset {3}: empty frame'.format(path, what, f, int(self.block[f])))

    def frame(self, i):
        return self.data[self.offset[i]:self.offset[i] + self.size[i]]


class _Source(object):
    """Positioned reads of the file (one pread each when it has a descriptor), counted."""

    def __init__(self, f):
        self.f = f
        f.seek(0, os.SEEK_END)
        self.size = f.tell()
        self.bytes_read = 0
        try:
            self.fd = f.fileno() if isinstance(f, io.FileIO) else None
        except (AttributeError, OSError):
            self.fd = None

    def read(self, pos, n):
        n = max(0, min(n, self.size - pos))
        if self.fd is not None:
            b = os.pread(self.fd, n, pos)
        else:
            self.f.seek(pos)
            b = self.f.read(n)
        self.bytes_read += len(b)
        return b


def is_matroska(path):
    """True when the file starts with an EBML header (False when it cannot be read: the WAV reader reports that)."""
    try:
        with open(path, 'rb') as f:
            return f.read(4) == EBML_MAGIC
    except OSError:
        return False


class MatroskaFile(object):
    """The container structure of a Matroska / WebM file.  `fileobj` (opened unbuffered by default) is any object
    with seek / read; the walk only ever reads through it."""

    def __init__(self, path, fileobj=None):
        self.path = path
        self._own = fileobj is None
        self._src = _Source(open(path, 'rb', buffering=0) if fileobj is None else fileobj)
        self.timestamp_scale = 1000000
        self.tracks, self.chapter_starts = [], []
        self._clusters = []                 # (offset, declared end or None)
        self._tables = {}                   # (stream id, payloads read) -> FrameTable
        try:
            self._read_header()
        except Exception:
            self.close()
            raise

    def close(self):
        if self._own and self._src is not None:
            self._src.f.close()
        self._src = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def bytes_read(self):
        """Bytes read from the file so far."""
        return self._src.bytes_read

    # -- element headers read from the file -------------------------------------------------------------------------
    def _header(self, pos, extra=0):
        """(id, id length + size length, size or None, the bytes read) of the element at `pos`, or None when the file
        ends inside its header.  `extra` more bytes are read with it (the start of a block's payload)."""
        head = self._src.read(pos, 12 + extra)
        try:
            i = read_id(head, 0)
            s = read_vint(head, i[1]) if i else None
        except ValueError as e:
            raise SushiError('{0}: Matroska element at byte {1}: {2}'.format(self.path, pos, e))
        if i is None or s is None:
            return None
        return i[0], i[1] + s[1], s[0], head

    def _cut(self, pos, elem_end, parent_end):
        """True when the file ends inside the element at `pos` (ending at elem_end) and its parent, whose declared
        end is parent_end (None for an unknown size), is cut too: a truncated file.  An element that runs past a
        parent ending inside the file is damage: SushiError naming its offset."""
        if elem_end > self._src.size and (parent_end is None or parent_end > self._src.size):
            return True
        if parent_end is not None and elem_end > parent_end:
            self._past_parent(pos, parent_end)
        return False

    def _past_parent(self, pos, parent_end):
        raise SushiError('{0}: Matroska element at byte {1} runs past its parent (which ends at byte {2})'.format(
            self.path, pos, parent_end))

    def _read_header(self):
        src = self._src
        h = self._header(0)
        if h is None or h[0] != ID_EBML or h[2] is None:
            raise SushiError('{0}: not an EBML file'.format(self.path))
        doctype, read_version = 'matroska', 1
        for eid, body, _ in children(src.read(h[1], h[2]), where=h[1]):
            if eid == ID_DOCTYPE:
                doctype = _text(body)
            elif eid == ID_DOCTYPE_READ_VERSION:
                read_version = _uint(body)
        if doctype not in ('matroska', 'webm') or read_version > 4:
            raise SushiError('{0}: unsupported EBML document type {1} version {2}'.format(self.path, doctype, read_version))
        pos = h[1] + h[2]
        while True:
            h = self._header(pos)
            if h is None:
                raise SushiError('{0}: no Matroska segment'.format(self.path))
            if h[0] == ID_SEGMENT:
                break
            if h[2] is None:
                raise SushiError('{0}: element of unknown size at byte {1}'.format(self.path, pos))
            pos += h[1] + h[2]
        self._segment = pos + h[1]
        self._segment_end = None if h[2] is None else pos + h[1] + h[2]       # declared; None for an unknown size
        have_tracks = False
        pos = self._segment
        end = self._segment_end
        while pos < (src.size if end is None else min(end, src.size)):
            h = self._header(pos)
            if h is None:
                logging.warning('{0}: file ends inside the element header at byte {1}'.format(self.path, pos))
                break
            eid, hl, size, _ = h
            if eid == ID_CLUSTER and size is None:
                self._clusters.append((pos, None))
                pos = self._walk_cluster(pos + hl, None, end, None)
                if pos is None:
                    break
                continue
            if size is None:
                raise SushiError('{0}: element at byte {1} has an unknown size'.format(self.path, pos))
            if self._cut(pos, pos + hl + size, end):
                # the file ends inside this element: a cluster loads up to its cut block, anything after is gone
                if eid in (ID_INFO, ID_TRACKS, ID_CHAPTERS):
                    raise SushiError('{0}: the file ends inside the element at byte {1}'.format(self.path, pos))
                if eid == ID_CLUSTER:
                    self._clusters.append((pos, pos + hl + size))
                else:
                    logging.warning('{0}: file ends inside the element at byte {1}; it is skipped'.format(
                        self.path, pos))
                break
            if eid == ID_CLUSTER:
                self._clusters.append((pos, pos + hl + size))
            elif eid in (ID_INFO, ID_TRACKS, ID_CHAPTERS):
                body = src.read(pos + hl, size)
                if eid == ID_INFO:
                    for cid, b, _ in children(body, where=pos + hl):
                        if cid == ID_TIMESTAMP_SCALE:
                            self.timestamp_scale = _uint(b)
                elif eid == ID_TRACKS:
                    self._read_tracks(body, pos + hl)
                    have_tracks = True
                else:
                    self._read_chapters(body, pos + hl)
            pos += hl + size
        if not have_tracks:
            raise SushiError('{0}: Matroska file without tracks'.format(self.path))

    def _read_tracks(self, body, where):
        for eid, entry, at in children(body, where=where):
            if eid != ID_TRACK_ENTRY:
                continue
            t = Track(len(self.tracks))
            for cid, b, cat in children(entry, where=at):
                if cid == ID_TRACK_NUMBER:
                    t.number = _uint(b)
                elif cid == ID_TRACK_TYPE:
                    t.type = _uint(b)
                elif cid == ID_CODEC_ID:
                    t.codec_id = _text(b)
                elif cid == ID_CODEC_PRIVATE:
                    t.codec_private = bytes(b)
                elif cid == ID_FLAG_DEFAULT:
                    t.default = bool(_uint(b))
                elif cid == ID_NAME:
                    t.name = _text(b)
                elif cid == ID_LANGUAGE:
                    t.language = _text(b)
                elif cid == ID_DEFAULT_DURATION:
                    t.default_duration = _uint(b)
                elif cid == ID_AUDIO:
                    for aid, ab, _ in children(b):
                        if aid == ID_SAMPLING_FREQUENCY:
                            t.sampling_frequency = _float(ab)
                        elif aid == ID_CHANNELS:
                            t.channels = _uint(ab)
                        elif aid == ID_BIT_DEPTH:
                            t.bit_depth = _uint(ab)
                elif cid == ID_CONTENT_ENCODINGS:
                    self._read_encodings(t, b)
            for _, scope, kind, algo, settings in t.encodings:
                if scope & 2 and kind == 0 and t.codec_private:
                    try:
                        t.codec_private = settings + t.codec_private if algo == 3 else zlib.decompress(t.codec_private)
                    except zlib.error as e:
                        raise SushiError('{0}: CodecPrivate of track {1}: {2}'.format(self.path, t.id, e))
            if t.type not in STREAM_TYPES or not t.codec_id:
                continue                            # no stream: FFmpeg skips it, so it takes no stream id
            self.tracks.append(t)

    def _read_encodings(self, t, body):
        for eid, enc, _ in children(body):
            if eid != ID_CONTENT_ENCODING:
                continue
            order, scope, kind, algo, settings = 0, 1, 0, 0, b''
            for cid, b, _ in children(enc):
                if cid == ID_ENCODING_ORDER:
                    order = _uint(b)
                elif cid == ID_ENCODING_SCOPE:
                    scope = _uint(b)
                elif cid == ID_ENCODING_TYPE:
                    kind = _uint(b)
                elif cid == ID_ENCRYPTION:
                    kind = 1
                elif cid == ID_COMPRESSION:
                    for k, v, _ in children(b):
                        if k == ID_COMP_ALGO:
                            algo = _uint(v)
                        elif k == ID_COMP_SETTINGS:
                            settings = bytes(v)
            if kind != 0:
                t.refusal = 'track {0} is encrypted'.format(t.id)
            elif algo not in (0, 3):
                t.refusal = 'track {0} is compressed with {1}, which is not supported'.format(
                    t.id, {1: 'bzlib', 2: 'lzo'}.get(algo, 'algorithm %d' % algo))
            t.encodings.append((order, scope, kind, algo, settings))

    def _read_chapters(self, body, where):
        """FFmpeg's rule: the top-level atoms of every edition in file order (nested atoms ignored); an atom needs a
        start and a nonzero ChapterUID, and is kept when no start was kept yet, the last kept start was 0, or it starts
        later than the last kept start."""
        max_start = 0
        for eid, edition, at in children(body, where=where):
            if eid != ID_EDITION_ENTRY:
                continue
            for aid, atom, aat in children(edition, where=at):
                if aid != ID_CHAPTER_ATOM:
                    continue
                uid, start = 0, None
                for cid, b, _ in children(atom, where=aat):
                    if cid == ID_CHAPTER_UID:
                        uid = _uint(b)
                    elif cid == ID_CHAPTER_TIME_START:
                        start = _uint(b)
                if start is not None and uid and (max_start == 0 or start > max_start):
                    self.chapter_starts.append(start)
                    max_start = start

    @property
    def chapters(self):
        """Chapter start times in seconds, as the reference parses them out of ffmpeg's `start %f` text."""
        return [float('%f' % (s / 1e9)) for s in self.chapter_starts]

    # -- the clusters -----------------------------------------------------------------------------------------------
    def _walk_cluster(self, pos, end, segment_end, visit):
        """Walk a cluster's children from `pos`.  `end` is the cluster's declared end, None for an unknown size (the
        cluster then ends at the next element of the segment's level or at segment_end, the segment's declared end or
        None for an unknown size).  visit(pos, header length, size, cluster time, BlockDuration, first payload bytes)
        gets every block.  Returns where the walk stopped (the cluster's end), or None when the file ended inside an
        element."""
        src = self._src
        parent = end if end is not None else segment_end
        limit = src.size if parent is None else min(parent, src.size)
        cluster_time = 0
        while pos < limit:
            h = self._header(pos, HEAD if visit is not None else 0)
            if h is None:
                logging.warning('{0}: file ends inside the element header at byte {1}; the rest is dropped'.format(
                    self.path, pos))
                return None
            eid, hl, size, head = h
            if end is None and eid in SEGMENT_CHILDREN:
                return pos
            if size is None:
                raise SushiError('{0}: element at byte {1} has an unknown size'.format(self.path, pos))
            elem_end = pos + hl + size
            if self._cut(pos, elem_end, parent):
                logging.warning('{0}: file ends inside the element at byte {1}; it and the rest are dropped'.format(
                    self.path, pos))
                return None
            if visit is not None:
                if eid == ID_CLUSTER_TIMESTAMP:
                    cluster_time = _uint(src.read(pos + hl, size))
                elif eid == ID_SIMPLE_BLOCK:
                    visit(pos, hl, size, cluster_time, None, head[hl:hl + min(size, HEAD)])
                elif eid == ID_BLOCK_GROUP:
                    block, duration = None, None
                    for cid, b, at in self._children_at(pos + hl, elem_end):
                        if cid == ID_BLOCK:
                            block = at
                        elif cid == ID_BLOCK_DURATION:
                            duration = _uint(src.read(b[0], b[1]))
                    if block is not None:
                        visit(block[0], block[1], block[2], cluster_time, duration, None)
            pos = elem_end
        return pos

    def _children_at(self, pos, end):
        """(id, (payload offset, size), (offset, header length, size)) of every child of the element body [pos, end)
        in the file, payloads not read."""
        while pos < end:
            h = self._header(pos)
            if h is None or h[2] is None or pos + h[1] + h[2] > end:
                self._past_parent(pos, end)
            if h[0] not in (ID_VOID, ID_CRC32):
                yield h[0], (pos + h[1], h[2]), (pos, h[1], h[2])
            pos += h[1] + h[2]

    def frames(self, ids, payloads=True):
        """{stream id: FrameTable} of the requested tracks, in block order.  With payloads=False only the block
        headers are read: the tables have times and no bytes (sizes are 0).  Tables already read (by prefetch or an
        earlier call) are not read again."""
        ids = list(ids)
        missing = [sid for sid in ids if (sid, True) not in self._tables and (sid, payloads) not in self._tables]
        if missing:
            self.prefetch(missing if payloads else (), () if payloads else missing)
        return {sid: self._tables.get((sid, True)) or self._tables[(sid, payloads)] for sid in ids}

    def release(self, ids):
        """Forget the tables of these tracks (their payloads can be large)."""
        for sid in ids:
            self._tables.pop((sid, True), None)
            self._tables.pop((sid, False), None)

    def prefetch(self, payload_ids=(), time_ids=()):
        """One walk over the clusters that reads the frames of every track in payload_ids and the block times of
        every track in time_ids (their payloads are not read); later frames() calls take the tables from here."""
        by_number, wants = {}, {}
        for sid, payloads in [(s, False) for s in time_ids] + [(s, True) for s in payload_ids]:
            t = self.track(sid)
            if t.refusal:
                raise SushiError('{0}: {1}'.format(self.path, t.refusal))
            by_number[t.number] = t
            wants[t.id] = payloads
        if not by_number:
            return
        pieces = {t.id: [] for t in by_number.values()}
        rows = {t.id: [] for t in by_number.values()}
        scale = self.timestamp_scale
        src = self._src

        def lace_ticks(t, duration, count):
            # FFmpeg's arithmetic: the block lasts BlockDuration, or DefaultDuration per lace, in whole ticks, and each
            # lace a whole share of it.  Laced frames after the first advance by that share
            block = duration if duration is not None else t.default_duration * count // scale
            return block // count

        def visit(pos, hl, size, cluster_time, duration, head):
            if head is None:
                head = src.read(pos + hl, min(size, HEAD))
            try:
                tn = read_vint(head, 0)
            except ValueError:
                tn = None
            if tn is None or tn[0] not in by_number:
                return
            t = by_number[tn[0]]
            at = tn[1]
            if at + 3 > size:
                raise SushiError('{0}: block at byte {1} is too short for its header'.format(self.path, pos))
            rel = struct.unpack('>h', head[at:at + 2])[0]
            lacing = (head[at + 2] >> 1) & 3
            at += 3
            if not wants[t.id]:
                count = 1 if lacing == 0 or at >= len(head) else head[at] + 1
                step = lace_ticks(t, duration, count)
                rows[t.id].extend((0, pos, (cluster_time + rel + k * step) * scale, step * scale) for k in range(count))
                return
            body = src.read(pos + hl, size)
            sizes = self._laces(body, at, lacing, pos)
            at = size - sum(sizes)
            step = lace_ticks(t, duration, len(sizes))
            for k, n in enumerate(sizes):
                try:
                    data = t.decode_frame(body[at:at + n])
                except zlib.error as e:
                    raise SushiError('{0}: block at byte {1}: {2}'.format(self.path, pos, e))
                at += n
                pieces[t.id].append(data)
                rows[t.id].append((len(data), pos, (cluster_time + rel + k * step) * scale, step * scale))

        for cpos, cend in self._clusters:
            h = self._header(cpos)
            if self._walk_cluster(cpos + h[1], cend, self._segment_end, visit) is None:
                break
        for sid in pieces:
            self._tables[(sid, wants[sid])] = FrameTable(pieces[sid], rows[sid])

    def _laces(self, body, at, lacing, pos):
        """Frame sizes of a block whose lace header starts at body[at] (after the flags byte)."""
        size = len(body)
        if lacing == 0:
            return [size - at]
        bad = SushiError('{0}: the lace table of the block at byte {1} runs past its block'.format(self.path, pos))
        if at >= size:
            raise bad
        count = body[at] + 1
        at += 1
        sizes = []
        if lacing == 1:                                    # Xiph: 255s then a byte below 255
            for _ in range(count - 1):
                n = 0
                while True:
                    if at >= size:
                        raise bad
                    b = body[at]
                    at += 1
                    n += b
                    if b != 255:
                        break
                sizes.append(n)
        elif lacing == 3:                                  # EBML: a size, then signed differences
            try:
                v = read_vint(body, at)
            except ValueError:
                v = None
            if v is None or v[0] is None:
                raise bad
            sizes.append(v[0])
            at += v[1]
            for _ in range(count - 2):
                try:
                    v = read_vint(body, at)
                except ValueError:
                    v = None
                if v is None or v[0] is None:
                    raise bad
                sizes.append(sizes[-1] + v[0] - ((1 << (7 * v[1] - 1)) - 1))
                at += v[1]
        else:                                              # fixed: equal sizes
            if (size - at) % count:
                raise SushiError('{0}: the fixed-size laces of the block at byte {1} do not divide it evenly'.format(
                    self.path, pos))
            return [(size - at) // count] * count
        rest = size - at - sum(sizes)
        if rest < 0 or any(s < 0 for s in sizes):
            raise bad
        return sizes + [rest]

    # -- streams ----------------------------------------------------------------------------------------------------
    def track(self, sid):
        for t in self.tracks:
            if t.id == sid:
                return t
        raise SushiError("Stream with index {0} doesn't exist in {1}".format(sid, self.path))

    def streams(self, kind):
        return [t for t in self.tracks if t.kind == kind]

    def select(self, kind, idx):
        """The reference's Demuxer._select_stream (demux.py:335-355): kind is 'audio', 'subtitles' or 'video'."""
        return select_stream(self.streams(kind), kind, idx, self.path)

    # -- side products ----------------------------------------------------------------------------------------------
    def script_text(self, track):
        """The script of a subtitle track as the file the reference's ffmpeg call writes: ASS / SSA as CodecPrivate
        and one Dialogue line per block in ReadOrder (times rounded to centiseconds), UTF-8 as numbered SRT entries
        with millisecond times and the text as it is."""
        kind = SCRIPT_TYPES.get(track.codec_id)
        if kind is None:
            raise SushiError('Unknown script type')
        table = self.frames([track.id])[track.id]
        if kind == '.srt':
            out = []
            for i in range(len(table)):
                a, b = table.time[i], table.time[i] + table.duration[i]
                out.append('{0}\n{1} --> {2}\n{3}\n'.format(i + 1, _srt_time(a), _srt_time(b),
                                                           table.frame(i).decode('utf-8', 'replace')))
            return '\n'.join(out)
        lines = []
        for i in range(len(table)):
            fields = table.frame(i).decode('utf-8', 'replace').split(',', 8)
            if len(fields) < 9:
                raise SushiError('{0}: subtitle block at byte {1} is not an ASS event'.format(self.path, table.block[i]))
            a, b = table.time[i], table.time[i] + table.duration[i]
            lines.append((int(fields[0]), 'Dialogue: {0},{1},{2},{3}'.format(fields[1], _ass_time(a), _ass_time(b),
                                                                            ','.join(fields[2:]))))
        lines.sort(key=lambda x: x[0])
        head = track.codec_private.decode('utf-8', 'replace').rstrip('\r\n\0')
        return head + '\n' + ''.join(line + '\n' for _, line in lines)

    def timecodes_text(self):
        """The frame times of the first video track as mkvextract's timestamps_v2 file: milliseconds, ascending."""
        video = self.streams('video')
        if not video:
            raise SushiError("{0} doesn't have any video".format(self.path))
        table = self.frames([video[0].id], payloads=False)[video[0].id]
        return '# timestamp format v2\n' + ''.join(_ms(t) + '\n' for t in np.sort(table.time))


def audio_codec(track):
    """'flac', 'truehd', 'alac' or 'pcm' for an audio track the GPU loader decodes (FLAC, Dolby TrueHD, ALAC, whose
    CodecPrivate is the ALACSpecificConfig, little-endian integer PCM of 16 or 24 bits);
    SushiError naming the track and its codec for anything else."""
    if track.refusal:
        raise SushiError(track.refusal)
    if track.codec_id == 'A_FLAC':
        return 'flac'
    if track.codec_id == 'A_TRUEHD':
        return 'truehd'
    if track.codec_id == 'A_ALAC' and len(track.codec_private) >= 24:
        return 'alac'
    if track.codec_id == 'A_PCM/INT/LIT' and track.bit_depth in (16, 24) and track.channels >= 1:
        return 'pcm'
    what = track.codec_id + (' at {0} bits'.format(track.bit_depth) if track.codec_id.startswith('A_PCM') else '')
    raise SushiError('Audio track {0} is {1}, which cannot be decoded here (FLAC, TrueHD, ALAC and 16- or '
                     '24-bit little-endian PCM can): convert it to FLAC or WAV first'.format(track.id, what))


def _ass_time(ns):
    cs = py2_round(ns / 1e7)
    return '{0}:{1:02d}:{2:02d}.{3:02d}'.format(int(cs // 360000), int((cs // 6000) % 60), int((cs // 100) % 60),
                                                int(cs % 100))


def _srt_time(ns):
    ms = py2_round(ns / 1e6)
    return '{0:02d}:{1:02d}:{2:02d},{3:03d}'.format(int(ms // 3600000), int((ms // 60000) % 60),
                                                    int((ms // 1000) % 60), int(ms % 1000))


def _ms(ns):
    ns = int(ns)
    if ns % 1000000 == 0:
        return str(ns // 1000000)
    return ('%.6f' % (ns / 1e6)).rstrip('0')
