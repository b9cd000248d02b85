"""Seeded writer of AVI files for the tests, with PCM audio and MP2 audio from tests/mp2_cases.py.

A case is a header (`avih`, one `strl` per stream with `strh`, `strf` and, in OpenDML cases, an `indx` super index,
and `LIST odml`) and the chunks of its streams in file order, laid out in one `movi` list or, in OpenDML cases, in the
`movi` of `RIFF AVI ` and of each `RIFF AVIX` that follows, each ending with one `ix##` standard index per stream.
Video chunks are random bytes under `00dc` / `00db`; optional `JUNK` chunks, `LIST rec ` grouping, odd sizes with their
pad byte, zero-size chunks, an `idx1` index and a GAB2-style `txts` stream.  PCM chunks hold whole sample frames
unless a case says otherwise; MP2 is CBR (`dwSampleSize` 1, chunks cut anywhere, frames straddling them) or VBR (one
frame per chunk, `nBlockAlign` 1152).

`good_cases()` the cases that load, `refused_cases()` the ones refused by name (with the reason), `damaged_cases()`
copies with one fault each and the byte offset the refusal names, `cut_case()` a copy cut inside an audio chunk.
What FFmpeg does with each is decided by tests/test_avi_cases.py against FFmpeg's `avi` demuxer:
  - chunks of a PCM stream that are not a whole number of sample frames (`partial_pcm_frames`): FFmpeg's decoder
    drops the partial frame of each packet; here they are refused by name."""
import struct

import numpy as np

from tests import mp2_cases as mc

AVIF_HASINDEX, AVIF_ISINTERLEAVED = 0x10, 0x100
PCM_GUID_TAIL = bytes.fromhex('000000001000800000aa00389b71')


def chunk(fourcc, data, pad=True):
    return fourcc + struct.pack('<I', len(data)) + data + (b'\0' if pad and len(data) & 1 else b'')


def riff_list(kind, body):
    return b'LIST' + struct.pack('<I', len(body) + 4) + kind + body


def waveformat(tag, channels, rate, bits, block_align=None, extensible=None, extra=b''):
    """WAVEFORMATEX (cbSize and what follows it; `extensible` (valid bits, channel mask, sub-format tag) makes it
    WAVEFORMATEXTENSIBLE)"""
    ba = channels * bits // 8 if block_align is None else block_align
    head = struct.pack('<HHIIHH', tag, channels, rate, rate * ba if ba else 24000, ba, bits)
    if extensible is not None:
        valid, mask, sub = extensible
        extra = struct.pack('<HI', valid, mask) + struct.pack('<H', sub) + PCM_GUID_TAIL
    return head + struct.pack('<H', len(extra)) + extra


def mp2_waveformat(case, vbr):
    """MPEGLAYER3WAVEFORMAT-style MP2 header as muxers write it (wFormatTag 0x50, MPEG1WAVEFORMAT extension)"""
    br = mc.KBPS[case.specs[0].lsf][case.specs[0].bitrate_index] * 1000
    ext = struct.pack('<HIHHHHII', 2, br, case.channels, 1, 0, 0, 0, 0)
    return struct.pack('<HHIIHH', 0x50, case.channels, case.rate, br // 8, 1152 if vbr else 1, 0) + \
        struct.pack('<H', len(ext)) + ext


class Stream(object):
    """One stream: `kind` 'vids', 'auds' or 'txts', `strf` its format chunk, `chunks` its payloads in order, `suffix`
    the two letters after its index in chunk FOURCCs.  For audio `codec` ('pcm', 'mp2' or FFmpeg's name of a refused
    one), `channels`, `bits`, `rate` and, for MP2, `case` (mp2_cases)."""

    def __init__(self, kind, strf, chunks, suffix=None, handler=b'\0\0\0\0', scale=1, rate=25, sample_size=0,
                 start=0, initial=0, codec=None, channels=0, bits=0, case=None, mask=None):
        self.kind, self.strf, self.chunks = kind, strf, chunks
        self.suffix = suffix or {'vids': b'dc', 'auds': b'wb', 'txts': b'tx'}[kind]
        self.handler, self.scale, self.rate, self.sample_size = handler, scale, rate, sample_size
        self.start, self.initial = start, initial
        self.codec, self.channels, self.bits, self.case, self.mask = codec, channels, bits, case, mask
        self.offsets = []                  # file offset of each of its chunks' headers
        self.es = b''.join(chunks)

    def strh(self):
        return struct.pack('<4s4sIHHIIIIIIIIhhhh', self.kind.encode(), self.handler, 0, 0, 0, self.initial, self.scale,
                           self.rate, self.start, len(self.chunks), 0, 0xFFFFFFFF, self.sample_size, 0, 0, 320, 240)


def pcm_stream(rng, channels, bits, rate, frames_per_chunk, extensible=None, chunk_frames=None):
    """A PCM stream of random samples in chunks of frames_per_chunk frames (a list is cycled)"""
    width = bits // 8
    sizes = frames_per_chunk if isinstance(frames_per_chunk, list) else [frames_per_chunk]
    chunks = []
    for k in range(len(sizes) if chunk_frames is None else chunk_frames):
        n = sizes[k % len(sizes)]
        chunks.append(rng.integers(0, 256, n * channels * width, dtype=np.uint8).tobytes())
    tag = 0xFFFE if extensible is not None else 1
    strf = waveformat(tag, channels, rate, bits, extensible=extensible)
    return Stream('auds', strf, chunks, scale=channels * width, rate=rate * channels * width,
                  sample_size=channels * width, codec='pcm', channels=channels, bits=bits,
                  mask=extensible[1] if extensible else None)


def mp2_stream(case, vbr, rng=None, cuts=None):
    """An MP2 stream: VBR one frame per chunk; CBR the frames joined and cut into chunks of random sizes"""
    if vbr:
        chunks = list(case.frames)
    else:
        data, chunks, at = case.data, [], 0
        while at < len(data):
            n = int(rng.integers(1, 3000))
            chunks.append(data[at:at + n])
            at += n
    return Stream('auds', mp2_waveformat(case, vbr), chunks, scale=1152 if vbr else 1,
                  rate=case.rate if vbr else mc.KBPS[case.specs[0].lsf][case.specs[0].bitrate_index] * 125,
                  sample_size=0 if vbr else 1, codec='mp2', channels=case.channels, bits=16, case=case)


def video_stream(rng, n, suffix=b'dc', sizes=(500, 4000)):
    strf = struct.pack('<IiiHHIIiiII', 40, 320, 240, 1, 24, 0x34363258 if suffix == b'dc' else 0, 320 * 240 * 3, 0, 0,
                       0, 0)
    chunks = [rng.integers(0, 256, int(rng.integers(*sizes)), dtype=np.uint8).tobytes() for _ in range(n)]
    return Stream('vids', strf, chunks, suffix=suffix, handler=b'H264' if suffix == b'dc' else b'\0\0\0\0')


def text_stream(n):
    """GAB2 subtitle stream (as FFmpeg reads it: a `GAB2` header, then a name and an SRT file); its chunks are empty
    after the first"""
    name = 'English'.encode('utf-16-le') + b'\0\0'
    srt = b'1\r\n00:00:01,000 --> 00:00:02,000\r\nhello\r\n\r\n'
    body = b'GAB2\0' + struct.pack('<HI', 2, len(name)) + name + struct.pack('<HI', 4, len(srt)) + srt
    return Stream('txts', b'', [body] + [b''] * (n - 1))


def interleave(streams, rng, per=None):
    """file order: stream s's chunks spread over the file by their share (per: chunks of each stream in each round)"""
    left = [list(range(len(s.chunks))) for s in streams]
    order = []
    while any(left):
        for i, s in enumerate(streams):
            take = 1 if per is None else per[i]
            for _ in range(take):
                if left[i]:
                    order.append((i, left[i].pop(0)))
    return order


class AviCase(object):
    """`order` [(stream, chunk)] in file order.  `segments` > 1 writes OpenDML (RIFF AVIX, indx, ix##), `rec` groups
    every `rec` chunks in LIST rec, `junk` puts a JUNK chunk every `junk` chunks, `idx1` writes the legacy index."""

    def __init__(self, name, streams, order, segments=1, rec=0, junk=0, idx1=True):
        self.name, self.streams, self.order = name, streams, order
        self.segments, self.rec, self.junk, self.idx1 = segments, rec, junk, idx1
        header = self._header(None)
        data, ix = self._layout(header)
        self.data, _ = self._layout(self._header(ix))
        assert len(self.data) == len(data)

    def audio(self):
        return [(i, s) for i, s in enumerate(self.streams) if s.kind == 'auds']

    def _header(self, ix):
        n = len(self.streams)
        avih = struct.pack('<IIIIIIIIII16x', 40000, 0, 0, AVIF_HASINDEX | AVIF_ISINTERLEAVED,
                           len([1 for s, _ in self.order if self.streams[s].kind == 'vids']), 0, n, 0, 320, 240)
        body = chunk(b'avih', avih)
        for i, s in enumerate(self.streams):
            strl = chunk(b'strh', s.strh()) + chunk(b'strf', s.strf)
            if self.segments > 1:
                entries = b''
                for k in range(self.segments):
                    off, size, dur = ix[(i, k)] if ix else (0, 0, 0)
                    entries += struct.pack('<QII', off, size, dur)
                strl += chunk(b'indx', struct.pack('<HBBI4s12x', 4, 0, 0, self.segments,
                                                   b'%02d' % i + s.suffix) + entries)
            body += riff_list(b'strl', strl)
        if self.segments > 1:
            body += riff_list(b'odml', chunk(b'dmlh', struct.pack('<I', len(self.order)) + bytes(244)))
        return riff_list(b'hdrl', body) + chunk(b'JUNK', bytes(100))

    def _layout(self, header):
        for s in self.streams:
            s.offsets = []
        segs = np.array_split(np.arange(len(self.order)), self.segments)
        out = bytearray()
        ix = {}
        idx1 = b''
        for k, seg in enumerate(segs):
            start = len(out)
            out += b'RIFF\0\0\0\0' + (b'AVI ' if k == 0 else b'AVIX')
            if k == 0:
                out += header
            movi = len(out)
            out += b'LIST\0\0\0\0movi'
            rec_at, per_stream = None, {}
            for j, o in enumerate(seg):
                s, c = self.order[o]
                st = self.streams[s]
                if self.rec and j % self.rec == 0:
                    if rec_at is not None:
                        struct.pack_into('<I', out, rec_at + 4, len(out) - rec_at - 8)
                    rec_at = len(out)
                    out += b'LIST\0\0\0\0rec '
                if self.junk and j % self.junk == self.junk - 1:
                    out += chunk(b'JUNK', bytes(j * 7 % 41))
                fourcc = b'%02d' % s + st.suffix
                st.offsets.append(len(out))
                per_stream.setdefault(s, []).append((len(out), len(st.chunks[c])))
                if k == 0:
                    idx1 += struct.pack('<4sIII', fourcc, 0x10, len(out) - movi - 8, len(st.chunks[c]))
                out += chunk(fourcc, st.chunks[c])
            if rec_at is not None:
                struct.pack_into('<I', out, rec_at + 4, len(out) - rec_at - 8)
            if self.segments > 1:
                for s in range(len(self.streams)):
                    st = self.streams[s]
                    ents = per_stream.get(s, [])
                    base = movi
                    body = struct.pack('<HBBI4sQI', 2, 0, 1, len(ents), b'%02d' % s + st.suffix, base, 0)
                    body += b''.join(struct.pack('<II', o + 8 - base, n) for o, n in ents)
                    ix[(s, k)] = (len(out), len(body) + 8, len(ents) if st.kind != 'auds' else
                                  sum(n for _, n in ents) // max(1, st.sample_size or 1))
                    out += chunk(b'ix%02d' % s, body)
            struct.pack_into('<I', out, movi + 4, len(out) - movi - 8)
            if k == 0 and self.idx1:
                out += chunk(b'idx1', idx1)
            struct.pack_into('<I', out, start + 4, len(out) - start - 8)
        return bytes(out), ix

    def movi_extents(self, data=None):
        """[(start, end)]: the file offsets of every movi list's first chunk and of its declared end"""
        data = self.data if data is None else data
        out, at = [], 0
        while at + 12 <= len(data):
            size = struct.unpack_from('<I', data, at + 4)[0]
            body, end = at + 12, min(len(data), at + 8 + size)
            while body + 12 <= end:
                n = struct.unpack_from('<I', data, body + 4)[0]
                if data[body:body + 4] == b'LIST' and data[body + 8:body + 12] == b'movi':
                    out.append((body + 12, body + 8 + n))
                body += 8 + n + (n & 1)
            at += 8 + size + (size & 1)
        return out

    def write(self, directory, data=None, suffix='.avi'):
        path = str(directory / (self.name + suffix))
        with open(path, 'wb') as f:
            f.write(self.data if data is None else data)
        return path

    def __repr__(self):
        return self.name


def _mp2(name, seed, n, **kw):
    return mc.stream(name, seed, n, **kw)


def good_cases():
    cases = []
    rng = np.random.default_rng([41])
    # 16-bit stereo PCM beside video, a chunk every frame (40 ms)
    v = video_stream(rng, 60)
    a = pcm_stream(rng, 2, 16, 48000, 1920, chunk_frames=60)
    cases.append(AviCase('pcm16_every_frame', [v, a], interleave([v, a], rng)))
    # 24-bit 5.1 PCM (WAVEFORMATEXTENSIBLE) at 0.5 s, uncompressed video chunks, JUNK and odd video sizes
    v = video_stream(rng, 40, suffix=b'db', sizes=(301, 1501))
    a = pcm_stream(rng, 6, 24, 48000, 24000, extensible=(24, 0x3F, 1), chunk_frames=4)
    cases.append(AviCase('pcm24_51_half_second', [v, a], interleave([v, a], rng, per=[12, 1]), junk=5))
    # 16-bit mono, extensible without a channel mask, zero-size chunks, LIST rec grouping, no idx1
    v = video_stream(rng, 30)
    a = pcm_stream(rng, 1, 16, 44100, [1764, 0, 1763, 1], extensible=(16, 0, 1), chunk_frames=30)
    cases.append(AviCase('pcm16_mono_rec', [v, a], interleave([v, a], rng), rec=2, idx1=False))
    # audio-first preload, then interleave; two audio streams (8-channel 16-bit and stereo 24-bit)
    v = video_stream(rng, 30)
    a = pcm_stream(rng, 8, 16, 48000, [1920, 960], chunk_frames=40)
    b = pcm_stream(rng, 2, 24, 44100, 1764, chunk_frames=35)
    order = [(1, k) for k in range(10)] + interleave([v, a, b], rng)
    order = order[:10] + [(s, c) for s, c in order[10:] if not (s == 1 and c < 10)]
    cases.append(AviCase('two_audio_preload', [v, a, b], order))
    # OpenDML: three RIFF segments, indx super indexes, ix## chunks in each movi
    v = video_stream(rng, 60)
    a = pcm_stream(rng, 2, 24, 48000, 1920, chunk_frames=60)
    cases.append(AviCase('odml_pcm24', [v, a], interleave([v, a], rng), segments=3))
    # MP2 CBR (dwSampleSize 1, frames straddling chunks) and VBR (one frame per chunk), with a GAB2 text stream
    cbr = _mp2('avi_cbr', 401, 40, rate_index=1, bitrate_index=10, mode=0)
    v = video_stream(rng, 30)
    a = mp2_stream(cbr, False, rng)
    t = text_stream(2)
    cases.append(AviCase('mp2_cbr_subs', [v, a, t], interleave([v, a, t], rng)))
    vbr = _mp2('avi_vbr', 402, 40, bitrate_index=[8, 10, 12], mode=1, mode_ext=[0, 2], crc=[False, True])
    v = video_stream(rng, 40)
    a = mp2_stream(vbr, True)
    cases.append(AviCase('mp2_vbr_odml', [v, a], interleave([v, a], rng), segments=2, rec=3))
    # MP2 CBR starting mid-frame (bytes before the first header cost the first whole frame)
    mono = _mp2('avi_mid', 403, 30, bitrate_index=8, mode=3, crc=True)
    a = mp2_stream(mono, False, rng)
    a.chunks[0] = a.chunks[0][7:] if len(a.chunks[0]) > 7 else a.chunks[0]
    a.es = b''.join(a.chunks)
    v = video_stream(rng, 20)
    cases.append(AviCase('mp2_mid_frame', [v, a], interleave([v, a], rng), junk=3))
    return cases


def refused_cases():
    """[(case, stream index, refusal regex)]"""
    rng = np.random.default_rng([42])
    out = []

    def one(name, strf, codec, channels=2, bits=16):
        v = video_stream(rng, 4)
        a = Stream('auds', strf, [bytes(rng.integers(0, 256, 400, dtype=np.uint8))] * 4, codec=codec,
                   channels=channels, bits=bits)
        return AviCase(name, [v, a], interleave([v, a], rng))
    out.append((one('mp3', waveformat(0x55, 2, 48000, 0, block_align=1), 'mp3'), 1, 'is mp3'))
    out.append((one('ac3', waveformat(0x2000, 2, 48000, 0, block_align=1), 'ac3'), 1, 'is ac3'))
    out.append((one('aac', waveformat(0xFF, 2, 48000, 16, block_align=1), 'aac'), 1, 'is aac'))
    out.append((one('pcm8', waveformat(1, 2, 48000, 8), 'pcm_u8', bits=8), 1, 'is pcm_u8'))
    out.append((one('float', waveformat(3, 2, 48000, 32), 'pcm_f32le', bits=32), 1, 'is pcm_f32le'))
    out.append((one('flac', waveformat(0xF1AC, 2, 48000, 16, block_align=1), 'flac'), 1, 'is flac'))
    return out


def partial_frame_case():
    """(case, stream index, byte offset named): a 16-bit stereo PCM stream whose 3rd chunk is not whole frames"""
    rng = np.random.default_rng([43])
    v = video_stream(rng, 10)
    a = pcm_stream(rng, 2, 16, 48000, 480, chunk_frames=10)
    a.chunks[2] = a.chunks[2][:-2]
    a.es = b''.join(a.chunks)
    c = AviCase('partial_pcm_frames', [v, a], interleave([v, a], rng))
    return c, 1, a.offsets[2]


def damaged_cases():
    """(base case, [(name, file bytes, byte offset named, regex)]) from pcm16_every_frame"""
    base = good_cases()[0]
    data = base.data
    offs = base.streams[1].offsets
    out = []
    k = offs[5]
    broken = bytearray(data)
    broken[k:k + 4] = b'01w\x01'
    out.append(('broken_fourcc', bytes(broken), k, 'no chunk header'))
    k = offs[7]
    longer = bytearray(data)
    n = struct.unpack_from('<I', data, k + 4)[0]
    struct.pack_into('<I', longer, k + 4, n + 8)            # still whole frames
    out.append(('wrong_size', bytes(longer), k + 8 + n + 8, 'no chunk header'))
    k = offs[9]
    end = base.movi_extents()[0][1]
    past = bytearray(data)
    struct.pack_into('<I', past, k + 4, end - k)
    out.append(('size_past_movi', bytes(past), k, 'runs past its movi list'))
    k = offs[11]
    garbage = bytearray(data[:k] + b'\x11\x22\x33' + data[k:])
    movi = base.movi_extents()[0][0] - 12
    for at in (4, movi + 4):
        struct.pack_into('<I', garbage, at, struct.unpack_from('<I', garbage, at)[0] + 3)
    out.append(('garbage_between', bytes(garbage), k, 'no chunk header'))
    return base, out


def cut_case():
    """(case, file bytes cut inside an audio chunk's payload, the audio chunks wholly before the cut)"""
    base = good_cases()[0]
    offs = base.streams[1].offsets
    k = offs[-4]
    return base, base.data[:k + 8 + 1000], len(offs) - 4


def long_file(path, minutes=90.0, bits=24, distinct=7, seg_bytes=1 << 30):
    """Write a long OpenDML file to `path`: 1 s chunks of 48 kHz stereo PCM (`distinct` random ones, cycled) beside
    4 kB random-byte video chunks, `RIFF AVI ` up to seg_bytes and then `RIFF AVIX` lists.  Returns the int16 samples
    it loads as (frames x 2: the top 16 bits of each sample)."""
    rng = np.random.default_rng([44])
    rate, width, secs = 48000, bits // 8, int(round(minutes * 60))
    chunks = [rng.integers(0, 256, rate * 2 * width, dtype=np.uint8).tobytes() for _ in range(distinct)]
    video = rng.integers(0, 256, 4000, dtype=np.uint8).tobytes()
    v = video_stream(rng, 1)
    a = pcm_stream(rng, 2, bits, rate, rate, chunk_frames=1)
    head = AviCase('long', [v, a], [(0, 0), (1, 0)])._header(None)
    with open(path, 'wb') as f:
        k, seg = 0, 0
        while k < secs:
            start = f.tell()
            f.write(b'RIFF\0\0\0\0' + (b'AVI ' if seg == 0 else b'AVIX') + (head if seg == 0 else b''))
            movi = f.tell()
            f.write(b'LIST\0\0\0\0movi')
            while k < secs and f.tell() - start < seg_bytes:
                f.write(chunk(b'00dc', video) + chunk(b'01wb', chunks[k % distinct]))
                k += 1
            end = f.tell()
            f.seek(movi + 4)
            f.write(struct.pack('<I', end - movi - 8))
            f.seek(start + 4)
            f.write(struct.pack('<I', end - start - 8))
            f.seek(end)
            seg += 1
    top = [np.frombuffer(c, np.uint8).reshape(-1, width)[:, width - 2:].copy().view('<i2').reshape(-1, 2)
           for c in chunks]
    return np.concatenate([top[k % distinct] for k in range(secs)])
