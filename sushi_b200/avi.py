"""AVI files on the host (`.avi`): old TV captures (VirtualDub, AviUtl, Huffyuv or Ut Video with PCM audio) and DVB
captures cut to AVI (MP2 audio), OpenDML files over 1 GiB included.

The host reads only headers, one small read each: the top-level RIFF chain (`RIFF AVI `, then any OpenDML `RIFF
AVIX` continuations), the `hdrl` list, and the file extents of every `LIST movi`.  The streams are listed as FFmpeg's
`avi` demuxer lists them: stream id the index of the `strl` in header order, kind from `strh.fccType` (`vids`, `auds`,
`txts`), and codec names from the video format's compression FOURCC and the audio format's `wFormatTag` (for
WAVEFORMATEXTENSIBLE, its sub-format GUID).  The audio itself is demuxed on the GPU (sb_avi_*): the host reads the file
in large chunks and hands them over, and does no per-chunk work.  16- and 24-bit little-endian PCM loads as container
PCM does; MP2 (confirmed by the layer of its first frame header) is decoded; everything else is refused by name.
Chunk timestamps, `dwStart` and `dwInitialFrames` shift nothing: the decoded samples are placed back to back."""
import logging
import os
import struct

import numpy as np

from . import _native, swr
from .common import Audio, Container, SushiError
from .mpegps import LAYERS, first_header

AVI_EXTENSIONS = ('.avi',)
# bytes of file each sb_avi_feed call takes, through one page-locked buffer
CHUNK_BYTES = 64 << 20
HEAD_BYTES = 1 << 20             # bytes of the first movi list read for an MP2 stream's first frame header
SB_AVI_PCM, SB_AVI_MP2 = 0, 1
PCM_GUID_TAIL = bytes.fromhex('000000001000800000aa00389b71')

# FFmpeg's codec names of the WAVE format tags (libavformat riff.c), PCM and float by their bit depth below
WAV_TAGS = {0x0002: 'adpcm_ms', 0x0006: 'pcm_alaw', 0x0007: 'pcm_mulaw', 0x0011: 'adpcm_ima_wav', 0x0050: 'mp2',
            0x0055: 'mp3', 0x0092: 'ac3', 0x00FF: 'aac', 0x0160: 'wmav1', 0x0161: 'wmav2', 0x0162: 'wmapro',
            0x0163: 'wmalossless', 0x1610: 'aac', 0x2000: 'ac3', 0x2001: 'dts', 0xF1AC: 'flac'}
PCM_BY_BYTES = {1: 'pcm_u8', 2: 'pcm_s16le', 3: 'pcm_s24le', 4: 'pcm_s32le', 8: 'pcm_s64le'}
FLOAT_BY_BYTES = {4: 'pcm_f32le', 8: 'pcm_f64le'}
# FFmpeg's codec names of common video compression FOURCCs (libavformat riff.c); BI_RGB is rawvideo
BMP_TAGS = {b'H264': 'h264', b'h264': 'h264', b'X264': 'h264', b'x264': 'h264', b'AVC1': 'h264', b'avc1': 'h264',
            b'XVID': 'mpeg4', b'xvid': 'mpeg4', b'DIVX': 'mpeg4', b'divx': 'mpeg4', b'DX50': 'mpeg4', b'FMP4': 'mpeg4',
            b'MJPG': 'mjpeg', b'HFYU': 'huffyuv', b'FFVH': 'ffvhuff', b'FFV1': 'ffv1', b'ULRG': 'utvideo',
            b'ULRA': 'utvideo', b'ULY0': 'utvideo', b'ULY2': 'utvideo', b'ULY4': 'utvideo', b'ULH0': 'utvideo',
            b'ULH2': 'utvideo', b'ULH4': 'utvideo', b'MPG2': 'mpeg2video', b'mpg2': 'mpeg2video',
            b'MPG1': 'mpeg1video', b'DIB ': 'rawvideo', b'\0\0\0\0': 'rawvideo', b'HEVC': 'hevc', b'H265': 'hevc'}


def is_avi(path):
    """True for a file that starts `RIFF`, a size, `AVI `"""
    try:
        with open(path, 'rb') as f:
            head = f.read(12)
    except (OSError, TypeError):
        return False
    return head[:4] == b'RIFF' and head[8:12] == b'AVI '


def wav_codec(strf):
    """(FFmpeg's codec name, format tag, bits, channel mask or None) of a WAVEFORMATEX or WAVEFORMATEXTENSIBLE"""
    if len(strf) < 16:
        return 'none', None, 0, None
    tag, _, _, _, _, bits = struct.unpack_from('<HHIIHH', strf, 0)
    mask = None
    if tag == 0xFFFE and len(strf) >= 40 and struct.unpack_from('<H', strf, 16)[0] >= 22:
        valid, mask = struct.unpack_from('<HI', strf, 18)
        if strf[26:40] != PCM_GUID_TAIL:
            return 'none', tag, bits, mask
        tag = struct.unpack_from('<H', strf, 24)[0]
        bits = valid or bits
    if tag == 1:
        return PCM_BY_BYTES.get((bits + 7) >> 3, 'none'), tag, bits, mask
    if tag == 3:
        return FLOAT_BY_BYTES.get((bits + 7) >> 3, 'none'), tag, bits, mask
    return WAV_TAGS.get(tag, 'none'), tag, bits, mask


class Stream(object):
    """One stream as FFmpeg lists it: `id` its index, `kind` ('video', 'audio', 'subtitles' or 'data'), `codec`
    FFmpeg's codec name ('none' when there is none); audio also `channels`, `rate`, `bits`, `block_align` and `mask`
    (WAVEFORMATEXTENSIBLE's dwChannelMask, or None)."""

    def __init__(self, sid, kind, codec):
        self.id, self.kind, self.codec = sid, kind, codec
        self.default = False
        self.title = ''
        self.channels = self.rate = self.bits = self.block_align = 0
        self.mask = None
        self.head = b''                   # MP2: its first payload bytes in the first movi list

    @property
    def info(self):
        return self.codec

    @property
    def script_type(self):
        return self.codec

    @property
    def layer(self):
        h = first_header(self.head)
        return None if h is None else (h >> 17) & 3


class AviFile(Container):
    """The headers of an AVI file: its stream list and the extents of its movi lists.  `chapters` is always empty
    (FFmpeg's avi demuxer gives none)."""
    no_timecodes = 'an AVI file'                # what the command line says video timestamps cannot be read from

    def __init__(self, path):
        self.path = path
        self.size = os.path.getsize(path)
        self.chapters = []
        self.tracks = []
        self.movi = []                          # [(first chunk's file offset, the list's end)]
        with open(path, 'rb') as f:
            head = f.read(12)
            if head[:4] != b'RIFF' or head[8:12] != b'AVI ':
                raise SushiError('{0}: not an AVI file (no RIFF AVI header at its start)'.format(path))
            self._read_riffs(f)

    def _read_riffs(self, f):
        at, hdrl = 0, False
        while at + 12 <= self.size:
            f.seek(at)
            h = f.read(12)
            size = struct.unpack_from('<I', h, 4)[0]
            if h[:4] != b'RIFF' or h[8:12] not in (b'AVI ', b'AVIX'):
                break
            end = min(self.size, at + 8 + size)
            k = at + 12
            while k + 12 <= end:
                f.seek(k)
                c = f.read(12)
                n = struct.unpack_from('<I', c, 4)[0]
                if c[:4] == b'LIST' and c[8:12] == b'hdrl' and not hdrl:
                    f.seek(k + 12)
                    self._read_hdrl(f.read(max(0, n - 4)))
                    hdrl = True
                elif c[:4] == b'LIST' and c[8:12] == b'movi':
                    self.movi.append((k + 12, k + 8 + n))
                k += 8 + n + (n & 1)
            at += 8 + size + (size & 1)
        if not hdrl:
            raise SushiError('{0}: not an AVI file (no hdrl list)'.format(self.path))
        self.movi = [(a, b) for a, b in self.movi if b > a]
        if any(s.codec == 'mp2' for s in self.tracks) and self.movi:
            f.seek(self.movi[0][0])
            self._read_head(f.read(min(HEAD_BYTES, self.movi[0][1] - self.movi[0][0])))

    def _read_hdrl(self, body):
        at = 0
        while at + 8 <= len(body):
            fourcc, n = body[at:at + 4], struct.unpack_from('<I', body, at + 4)[0]
            if fourcc == b'LIST' and body[at + 8:at + 12] == b'strl':
                self._read_strl(body[at + 12:at + 8 + n])
            at += 8 + n + (n & 1)

    def _read_strl(self, body):
        strh = strf = None
        at = 0
        while at + 8 <= len(body):
            fourcc, n = body[at:at + 4], struct.unpack_from('<I', body, at + 4)[0]
            data = body[at + 8:at + 8 + n]
            if fourcc == b'strh':
                strh = data
            elif fourcc == b'strf':
                strf = data
            at += 8 + n + (n & 1)
        fcc = strh[:4] if strh and len(strh) >= 4 else b''
        sid = len(self.tracks)
        if fcc == b'vids':
            comp = strf[16:20] if strf and len(strf) >= 20 else b''
            s = Stream(sid, 'video', BMP_TAGS.get(comp, 'none'))
        elif fcc == b'auds':
            codec, _, bits, mask = wav_codec(strf or b'')
            s = Stream(sid, 'audio', codec)
            if strf and len(strf) >= 16:
                _, s.channels, s.rate, _, s.block_align, _ = struct.unpack_from('<HHIIHH', strf, 0)
            s.bits, s.mask = bits, mask
        elif fcc == b'txts':
            s = Stream(sid, 'subtitles', 'none')
        else:
            s = Stream(sid, 'data', 'none')
        self.tracks.append(s)

    def _read_head(self, data):
        """the first payload bytes of each MP2 stream, following the chunks of the first movi list by size"""
        want = {b'%02dwb' % s.id: s for s in self.tracks if s.codec == 'mp2'}
        at = 0
        while at + 12 <= len(data):
            fourcc, n = data[at:at + 4], struct.unpack_from('<I', data, at + 4)[0]
            if fourcc == b'LIST':
                at += 12
                continue
            s = want.get(fourcc)
            if s is not None and len(s.head) < 65536:
                s.head += data[at + 8:at + 8 + n]
            at += 8 + n + (n & 1)

    def select_audio(self, track=None):
        s = self.select('audio', track)
        codec = audio_codec(s)
        if codec == 'mp2':
            return Audio('MP2', s.id, self.path, decode=lambda device: self._decode(device, s, SB_AVI_MP2),
                         **swr.audio_format(16, swr.PLAIN))
        layout = dict(swr.DEFAULT)
        if s.mask and bin(s.mask).count('1') == s.channels:
            layout[s.channels] = s.mask
        return Audio('PCM', s.id, self.path, decode=lambda device: self._decode(device, s, SB_AVI_PCM),
                     **swr.audio_format(24 if s.codec == 'pcm_s24le' else 16, layout))

    def _decode(self, device, s, codec):
        """Stream `s`, demuxed on the GPU (sb_avi_*) from chunks of CHUNK_BYTES and, for MP2, decoded there."""
        config = np.array([s.channels, 24 if s.codec == 'pcm_s24le' else 16, s.rate], np.int32)
        ext = np.array(self.movi or [(0, 0)], np.int64).reshape(-1)
        h, cut, _ = _native.demux_file(device, 'sb_avi', (s.id, codec, config.ctypes.data_as(_native.c_i32p),
                                                          ext.ctypes.data_as(_native.c_i64p), len(self.movi)),
                                       self.path, CHUNK_BYTES)
        if cut:
            logging.warning('{0}: stream {1} is cut short at the end of the file; the bytes of its last chunk that '
                            'exist are kept{2}'.format(self.path, s.id, ', and a last frame cut short is decoded with '
                                                       'zeros' if codec == SB_AVI_MP2 else ''))
        return h


def audio_codec(stream):
    """'mp2' for an MP2 stream whose first header is layer II, 'pcm' for 16- or 24-bit little-endian PCM of 1 to 8
    channels; SushiError naming the stream and FFmpeg's codec name (or the layer) for anything else."""
    if stream.codec == 'mp2':
        layer = stream.layer
        if layer == 2:
            return 'mp2'
        what = 'MPEG audio {0}'.format(LAYERS[layer]) if layer in LAYERS else 'MPEG audio with no frame header in the ' \
            'first {0} bytes of its first movi list'.format(HEAD_BYTES)
    elif stream.codec in ('pcm_s16le', 'pcm_s24le') and 1 <= stream.channels <= 8:
        width = 2 if stream.codec == 'pcm_s16le' else 3
        if stream.block_align == stream.channels * width:
            return 'pcm'
        what = '{0} with nBlockAlign {1} for {2} channels'.format(stream.codec, stream.block_align, stream.channels)
    elif stream.codec in ('pcm_s16le', 'pcm_s24le'):
        what = '{0} with {1} channels'.format(stream.codec, stream.channels)
    else:
        what = stream.codec
    raise SushiError('Audio track {0} is {1}, which cannot be decoded here (16- and 24-bit PCM of 1 to 8 channels can, '
                     'and MP2): convert it to FLAC or WAV first'.format(stream.id, what))
