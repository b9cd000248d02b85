"""MPEG transport streams on the host: Blu-ray BDAV streams (`.m2ts`, 192-byte packets carrying a 4-byte arrival time
stamp) and plain 188-byte streams (`.ts`, `.mts`, `.m2t`).

The host reads only the head of the file: the packet size, the PAT and the first PMT, which give the stream list
(ids, kinds and codec names as FFmpeg's mpegts demuxer gives them).  The audio itself is demuxed and decoded on the
GPU (sb_ts_*): the host reads the file in large chunks and hands them over, and does no per-packet work.

What is kept of FFmpeg's stream rules:
  - streams come in PMT order, one per elementary stream;
  - stream types are looked up in FFmpeg's ISO table, then, under an `HDMV` (or `HDPR`) registration descriptor in the
    PMT's program info, in its HDMV table (0x80 pcm_bluray, 0x81 ac3, 0x82 / 0x85 / 0x86 / 0xA2 dts, 0x83 truehd, 0x84 /
    0xA1 eac3, 0x90 hdmv_pgs_subtitle, 0x92 hdmv_text_subtitle), then in its table of other private types (0x81 ac3,
    0x8A dts); anything else is a data stream with no codec, which still takes an id;
  - an HDMV stream of type 0x83 gets a second stream right after it, `ac3`: FFmpeg routes the PES packets whose
    stream_id_extension is 0x76 (the AC-3 sub-stream) to it and every other one to the TrueHD stream;
  - no stream is flagged default.
Only the first PMT version is read: streams a later PMT announces are not listed.  Elementary-stream descriptors
(languages, stream-level registrations) are not read.  A PAT listing more than one program is refused.
"""
import logging
import os

from . import _native, swr
from .common import Audio, Container, SushiError

TS_EXTENSIONS = ('.m2ts', '.mts', '.m2t', '.ts')
PROBE_SIZE = 5000000             # FFmpeg's default probesize: the PAT and the PMT must lie in this many bytes
SYNC = 0x47
# bytes of file each sb_ts_feed call takes (rounded down to whole packets), through one page-locked buffer
CHUNK_BYTES = 64 << 20

ISO_TYPES = {0x01: ('video', 'mpeg2video'), 0x02: ('video', 'mpeg2video'), 0x03: ('audio', 'mp3'),
             0x04: ('audio', 'mp3'), 0x0F: ('audio', 'aac'), 0x10: ('video', 'mpeg4'), 0x11: ('audio', 'aac_latm'),
             0x1B: ('video', 'h264'), 0x1C: ('audio', 'aac'), 0x20: ('video', 'h264'), 0x21: ('video', 'jpeg2000'),
             0x24: ('video', 'hevc'), 0x33: ('video', 'vvc'), 0x42: ('video', 'cavs'), 0xD1: ('video', 'dirac'),
             0xD2: ('video', 'avs2'), 0xD4: ('video', 'avs3'), 0xEA: ('video', 'vc1')}
HDMV_TYPES = {0x80: ('audio', 'pcm_bluray'), 0x81: ('audio', 'ac3'), 0x82: ('audio', 'dts'), 0x83: ('audio', 'truehd'),
              0x84: ('audio', 'eac3'), 0x85: ('audio', 'dts'), 0x86: ('audio', 'dts'), 0xA1: ('audio', 'eac3'),
              0xA2: ('audio', 'dts'), 0x90: ('subtitles', 'hdmv_pgs_subtitle'),
              0x92: ('subtitles', 'hdmv_text_subtitle')}
MISC_TYPES = {0x81: ('audio', 'ac3'), 0x8A: ('audio', 'dts')}
# stream types 0x03 and 0x04 are listed as `mp3` until FFmpeg's parser reads a frame header; the GPU decodes layer II
# and refuses layer I and III by name
DECODED = {'pcm_bluray': ('BD-LPCM', _native.SB_TS_PCM_BLURAY), 'truehd': ('TrueHD', _native.SB_TS_TRUEHD),
           'mp3': ('MP2', _native.SB_TS_MP2)}


def is_transport_stream(path):
    """True for a transport stream's file name; TransportStream then decides from the content."""
    return str(path).lower().endswith(TS_EXTENSIONS)


def crc32_mpeg(data):
    """The CRC-32 of MPEG-2 sections (polynomial 0x04C11DB7, initial value 0xFFFFFFFF, no reflection)."""
    crc = 0xFFFFFFFF
    for b in data:
        crc ^= b << 24
        for _ in range(8):
            crc = ((crc << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if crc & 0x80000000 else (crc << 1) & 0xFFFFFFFF
    return crc


class Stream(object):
    """One stream as FFmpeg lists it: `id` its index, `pid`, `stream_type`, `kind` ('audio', 'video', 'subtitles' or
    'other'), `codec` FFmpeg's codec name ('none' when there is none)."""

    def __init__(self, sid, pid, stream_type, kind, codec):
        self.id, self.pid, self.stream_type, self.kind, self.codec = sid, pid, stream_type, kind, codec
        self.default = False
        self.title = ''

    @property
    def info(self):
        return '{0}, PID 0x{1:04x}, stream type 0x{2:02x}'.format(self.codec, self.pid, self.stream_type)

    @property
    def script_type(self):
        return self.codec


class TransportStream(Container):
    """The head of a transport stream: packet size, program and stream list.  `chapters` is always empty (FFmpeg's
    mpegts demuxer gives none)."""
    no_timecodes = 'a transport stream'         # what the command line says video timestamps cannot be read from

    def __init__(self, path):
        self.path = path
        self.size = os.path.getsize(path)
        with open(path, 'rb') as f:
            head = f.read(PROBE_SIZE)
        self.packet_size = self._packet_size(head)
        self.chapters = []
        self._read_tables(head)

    def _packet_size(self, head):
        for size in (192, 188):
            n = min(len(head) // size, 32)
            if n >= 1 and all(head[k * size + size - 188] == SYNC for k in range(n)):
                return size
        raise SushiError('{0}: not a transport stream (no 0x47 sync byte every 188 or 192 bytes)'.format(self.path))

    def _packets(self, head):
        """(byte offset, PID, payload-unit start, payload) of each whole packet in `head`."""
        p = self.packet_size
        for at in range(0, len(head) - p + 1, p):
            pk = head[at + p - 188:at + p]
            if pk[0] != SYNC:
                raise SushiError('{0}: transport stream packet at byte offset {1}: lost sync'.format(self.path, at))
            afc = (pk[3] >> 4) & 3
            off = 4 + (1 + pk[4] if afc & 2 else 0)
            if not afc & 1 or off >= 188:
                continue
            yield at, ((pk[1] & 0x1F) << 8) | pk[2], (pk[1] >> 6) & 1, pk[off:]

    def _section(self, head, pid, table_id):
        """(bytes, byte offset of the packet it starts in) of the first whole section of `table_id` on `pid`."""
        buf, start = None, None
        for at, p, pusi, payload in self._packets(head):
            if p != pid:
                continue
            if pusi:
                pointer = payload[0]
                if buf is not None:
                    buf += payload[1:1 + pointer]
                    found = self._complete(buf, table_id, start)
                    if found:
                        return found
                buf, start = bytearray(payload[1 + pointer:]), at
            elif buf is not None:
                buf += payload
            if buf is not None:
                found = self._complete(buf, table_id, start)
                if found:
                    return found
                if len(buf) >= 3 and buf[0] != table_id and buf[0] != 0xFF:
                    buf = None                                    # another table on this PID: wait for the next start
        raise SushiError('{0}: no {1} on PID {2} in the first {3} bytes'.format(
            self.path, 'PAT' if table_id == 0 else 'PMT', pid, PROBE_SIZE))

    def _complete(self, buf, table_id, start):
        if len(buf) < 3 or buf[0] != table_id:
            return None
        n = 3 + (((buf[1] & 0x0F) << 8) | buf[2])
        if len(buf) < n:
            return None
        section = bytes(buf[:n])
        if n < 12 or crc32_mpeg(section) != 0:
            raise SushiError('{0}: {1} section at byte offset {2}: CRC-32 mismatch'.format(
                self.path, 'PAT' if table_id == 0 else 'PMT', start))
        return section, start

    def _read_tables(self, head):
        pat, _ = self._section(head, 0, 0x00)
        programs = []
        for k in range(8, len(pat) - 4, 4):
            number = (pat[k] << 8) | pat[k + 1]
            if number:
                programs.append(((pat[k + 2] & 0x1F) << 8) | pat[k + 3])
        if len(programs) != 1:
            raise SushiError('{0}: the transport stream has {1} programs; only one program is supported'.format(
                self.path, len(programs)))
        pmt, _ = self._section(head, programs[0], 0x02)
        info_len = ((pmt[10] & 0x0F) << 8) | pmt[11]
        hdmv = False
        at = 12
        while at + 2 <= 12 + info_len:
            tag, n = pmt[at], pmt[at + 1]
            if tag == 0x05 and pmt[at + 2:at + 6] in (b'HDMV', b'HDPR'):
                hdmv = True
            at += 2 + n
        self.hdmv = hdmv
        self.tracks = []
        at = 12 + info_len
        while at + 5 <= len(pmt) - 4:
            stype, pid = pmt[at], ((pmt[at + 1] & 0x1F) << 8) | pmt[at + 2]
            es_len = ((pmt[at + 3] & 0x0F) << 8) | pmt[at + 4]
            at += 5 + es_len
            kind, codec = ISO_TYPES.get(stype) or (hdmv and HDMV_TYPES.get(stype)) or MISC_TYPES.get(stype) or \
                ('other', 'none')
            self.tracks.append(Stream(len(self.tracks), pid, stype, kind, codec))
            if hdmv and stype == 0x83:
                self.tracks.append(Stream(len(self.tracks), pid, stype, 'audio', 'ac3'))

    def select_audio(self, track=None):
        s = self.select('audio', track)
        label = DECODED[audio_codec(s)][0]
        # BD-LPCM's bit depth is in its PES headers, read on the GPU; TrueHD decodes to S32, MP2 to S16
        fields = swr.audio_format(16, swr.PLAIN) if label == 'MP2' else {'fmt': 'S32' if label == 'TrueHD' else None}
        return Audio(label, s.id, self.path, decode=lambda device: self._decode(device, s), **fields)

    def _decode(self, device, s):
        """The BD-LPCM, TrueHD or MP2 stream `s`, demuxed and decoded on the GPU (sb_ts_*) from chunks of CHUNK_BYTES."""
        h, cut, dropped = _native.demux_file(device, 'sb_ts', (self.packet_size, s.pid, DECODED[s.codec][1]), self.path,
                                             CHUNK_BYTES, self.packet_size)
        if dropped:
            logging.warning('{0}: the file ends inside the transport stream packet at byte offset {1}; that '
                            'packet is dropped'.format(self.path, self.size - dropped))
        if cut:
            logging.warning('{0}: the last PES packet of stream {1} is cut short; its whole sample frames are '
                            'kept'.format(self.path, s.id))
        return h


def audio_codec(stream):
    """'pcm_bluray', 'truehd' or 'mp3' (MPEG audio: layer II is decoded) for a stream the GPU decodes; SushiError naming the stream and FFmpeg's codec name
    for anything else."""
    if stream.codec in DECODED:
        return stream.codec
    raise SushiError('Audio track {0} is {1}, which cannot be decoded here (BD-LPCM, TrueHD and MP2 can): convert it to '
                     'FLAC or WAV first'.format(stream.id, stream.codec))
