"""MPEG program streams on the host: VCD and SVCD `.mpg`, DVD `.vob`, DVB recorders' `.mpg` (and `.mpeg`, `.m2p`).

The host reads only the head of the file (FFmpeg's probesize), following the packet chain by length, and lists the
streams as FFmpeg's `mpeg` demuxer lists them after probing: in the order their first packet appears, with FFmpeg's
stream id (the PES stream id with 0x100 added; for private stream 1 the substream id) and codec name:
  - 0xC0-0xDF MPEG audio `mp2`; 0xE0-0xEF video, `mpeg2video` when a sequence extension follows the first sequence
    header and `mpeg1video` when not (FFmpeg's parser decides so); a PSM entry gives the codec of other stream types;
  - private stream 1 substreams: 0x20-0x3F `dvd_subtitle`, 0x80-0x87 and 0xC0-0xCF `ac3`, 0x88-0x8F and 0x98-0x9F `dts`,
    0xA0-0xAF `pcm_dvd`, 0xB0-0xBF `truehd`;
  - private stream 2 (DVD nav packs) a data stream `dvd_nav_packet`; padding, the PSM and the system header none.
A video stream with neither a PSM entry nor a sequence header at its start is listed without a codec, where FFmpeg
probes its content.  Streams that first appear past the head are not listed.  The audio itself is demuxed and
decoded on the GPU (sb_ps_*): the host reads the file in large chunks and hands them over, and does no per-packet work.
"""
import logging
import os
import struct

from . import _native, swr
from .common import Audio, Container, SushiError

PS_EXTENSIONS = ('.mpg', '.mpeg', '.m2p', '.vob')
PROBE_SIZE = 5000000             # FFmpeg's default probesize
# bytes of file each sb_ps_feed call takes, through one page-locked buffer
CHUNK_BYTES = 64 << 20

PSM_TYPES = {0x01: ('video', None), 0x02: ('video', None), 0x03: ('audio', 'mp2'), 0x04: ('audio', 'mp2'),
             0x0F: ('audio', 'aac'), 0x10: ('video', 'mpeg4'), 0x1B: ('video', 'h264'), 0x24: ('video', 'hevc'),
             0x81: ('audio', 'ac3')}
LAYERS = {1: 'layer III (MP3)', 2: 'layer II', 3: 'layer I (MP1)'}


def is_program_stream(path):
    """True for a program stream's file name; ProgramStream then decides from the content."""
    return str(path).lower().endswith(PS_EXTENSIONS)


def substream_codec(sub):
    """(kind, codec) of a private stream 1 substream id as FFmpeg's mpeg demuxer names it, or None (skipped)"""
    if 0x20 <= sub <= 0x3F:
        return 'subtitles', 'dvd_subtitle'
    if 0x80 <= sub <= 0x87 or 0xC0 <= sub <= 0xCF:
        return 'audio', 'ac3'
    if 0x88 <= sub <= 0x8F or 0x98 <= sub <= 0x9F:
        return 'audio', 'dts'
    if 0xA0 <= sub <= 0xAF:
        return 'audio', 'pcm_dvd'
    if 0xB0 <= sub <= 0xBF:
        return 'audio', 'truehd'
    return None


def pes_payload(pk):
    """The payload of the PES packet pk (MPEG-1 or MPEG-2 header), or None for a header FFmpeg skips"""
    end, at = len(pk), 6
    while at < end and pk[at] == 0xFF:
        at += 1
    if at < end and pk[at] & 0xC0 == 0x40:
        at += 2
    if at >= end:
        return None
    c = pk[at]
    if c & 0xE0 == 0x20:
        at += 10 if c & 0x10 else 5
    elif c & 0xC0 == 0x80:
        if at + 3 > end:
            return None
        at += 3 + pk[at + 2]
    elif c == 0x0F:
        at += 1
    else:
        return None
    return pk[at:] if at <= end else None


def first_header(data):
    """The first four bytes of `data` FFmpeg's MPEG audio parser takes for a header (sb_mp2.cuh frame_table), or None"""
    for b in range(len(data) - 3):
        h = int.from_bytes(data[b:b + 4], 'big')
        bi = (h >> 12) & 15
        if (h & 0xFFE00000) == 0xFFE00000 and (h >> 19) & 3 != 1 and (h >> 17) & 3 and bi not in (0, 15) and \
                (h >> 10) & 3 != 3:
            return h
    return None


class Stream(object):
    """One stream as FFmpeg lists it: `id` its index, `stream_id` FFmpeg's id, `pes_id` the PES stream id carrying it,
    `kind` ('audio', 'video', 'subtitles' or 'data'), `codec` FFmpeg's codec name ('none' when there is none)."""

    def __init__(self, sid, stream_id, pes_id, kind, codec):
        self.id, self.stream_id, self.pes_id, self.kind, self.codec = sid, stream_id, pes_id, kind, codec
        self.default = False
        self.title = ''
        self.head = b''                   # its payload bytes in the head (MPEG audio and video: the first 64 kB)

    @property
    def info(self):
        return '{0}, stream id 0x{1:x}'.format(self.codec, self.stream_id)

    @property
    def script_type(self):
        return self.codec

    @property
    def layer(self):
        """2 for layer II (the MPEG audio header's layer field: 1 layer III, 2 layer II, 3 layer I), None unknown"""
        h = first_header(self.head)
        return None if h is None else (h >> 17) & 3


class ProgramStream(Container):
    """The head of a program stream and its stream list.  `chapters` is always empty (FFmpeg's mpeg demuxer gives
    none)."""
    no_timecodes = 'a program stream'           # what the command line says video timestamps cannot be read from

    def __init__(self, path):
        self.path = path
        self.size = os.path.getsize(path)
        with open(path, 'rb') as f:
            head = f.read(PROBE_SIZE)
        if head[:4] != b'\x00\x00\x01\xba' or len(head) < 12 or not (head[4] & 0xC0 == 0x40 or head[4] & 0xF0 == 0x20):
            raise SushiError('{0}: not a program stream (no pack header at its start)'.format(path))
        self.chapters = []
        self.tracks = []
        self._read_head(head)

    def _read_head(self, head):
        psm, found, at = {}, {}, 0
        while at + 4 <= len(head) and head[at:at + 3] == b'\x00\x00\x01' and head[at + 3] >= 0xB9:
            code = head[at + 3]
            if code == 0xB9:
                at += 4
                continue
            if code == 0xBA:
                if at + 14 > len(head):
                    break
                at += 14 + (head[at + 13] & 7) if head[at + 4] & 0xC0 == 0x40 else 12
                continue
            if at + 6 > len(head):
                break
            n = 6 + struct.unpack_from('>H', head, at + 4)[0]
            pk = head[at:at + n]
            at += n
            if code == 0xBC and len(pk) == n:
                info = struct.unpack_from('>H', pk, 8)[0]
                end = n - 4
                k = 10 + info + 2
                while k + 4 <= end:
                    psm[pk[k + 1]] = pk[k]
                    k += 4 + struct.unpack_from('>H', pk, k + 2)[0]
                continue
            if code in (0xBB, 0xBE) or code >= 0xF0:
                continue
            if code == 0xBF:
                key, kind, codec = 0x1BF, 'data', 'dvd_nav_packet'
                payload = b''
            else:
                payload = pes_payload(pk)
                if payload is None:
                    continue
                if code == 0xBD:
                    if not payload:
                        continue
                    named = substream_codec(payload[0])
                    if named is None:
                        continue
                    key, (kind, codec) = payload[0], named
                elif 0xC0 <= code <= 0xEF:
                    key = 0x100 | code
                    kind, codec = ('audio', 'mp2') if code < 0xE0 else ('video', None)
                    if code in psm and psm[code] in PSM_TYPES:
                        kind, named = PSM_TYPES[psm[code]]
                        codec = named or codec
                else:
                    continue
            s = found.get(key)
            if s is None:
                s = found[key] = Stream(len(self.tracks), key, code, kind, codec)
                self.tracks.append(s)
            if code != 0xBD and len(s.head) < 65536:
                s.head += payload
        for s in self.tracks:
            if s.kind == 'video' and s.codec is None:
                seq = s.head.find(b'\x00\x00\x01\xb3')
                if seq < 0:
                    s.codec = 'none'
                else:
                    ext = s.head.find(b'\x00\x00\x01\xb5', seq)
                    s.codec = 'mpeg2video' if ext >= 0 and s.head[ext + 4] >> 4 == 1 else 'mpeg1video'

    def select_audio(self, track=None):
        s = self.select('audio', track)
        audio_codec(s)
        return Audio('MP2', s.id, self.path, decode=lambda device: self._decode(device, s),
                     **swr.audio_format(16, swr.PLAIN))

    def _decode(self, device, s):
        """The MP2 stream `s`, demuxed and decoded on the GPU (sb_ps_*) from chunks of CHUNK_BYTES."""
        h, cut, _ = _native.demux_file(device, 'sb_ps', (s.pes_id, -1), self.path, CHUNK_BYTES)
        if cut:
            logging.warning('{0}: stream {1} is cut short at the end of the file; its whole frames are kept, and a last '
                            'frame cut short is decoded with zeros'.format(self.path, s.id))
        return h


def audio_codec(stream):
    """'mp2' for an MPEG audio stream whose first header is layer II; SushiError naming the stream and FFmpeg's codec
    name (or the layer) for anything else."""
    if stream.codec == 'mp2':
        layer = stream.layer
        if layer == 2:
            return 'mp2'
        what = 'MPEG audio {0}'.format(LAYERS[layer]) if layer in LAYERS else 'MPEG audio with no frame header in the ' \
            'first {0} bytes'.format(PROBE_SIZE)
    else:
        what = stream.codec
    raise SushiError('Audio track {0} is {1}, which cannot be decoded here (MP2 can): convert it to FLAC or WAV '
                     'first'.format(stream.id, what))
