"""Seeded NumPy writer of MPEG transport streams for the tests: BDAV (.m2ts, 192-byte packets) and plain 188-byte
streams, with the PCM each audio stream decodes to.

A case holds PAT and PMT sections with their CRC-32, repeated through the file (with or without an `HDMV`
registration descriptor), PCR-only packets, adaptation fields of every length from 0 to 183, null packets, and PES
packets of BD-LPCM audio (16, 20 and 24 bits, the 20-bit stream being one FFmpeg's decoder refuses; 1, 2, 3, 6 and 8 channels, the padding channel of an odd count holding
nonzero bytes; 48, 96 and 192 kHz; some PES with leftover bytes after their last whole sample frame), TrueHD (from
tests/truehd_cases.py, split into PES payloads regardless of its access units, with AC-3 sub-stream PES interleaved),
random-byte video and PGS.  `damaged_cases()` gives copies with one fault each and the byte offset that must be named;
`cut_cases()` gives copies cut short and the sample frames that survive.  `assert_coverage` checks that the cases
cover all of this."""
import os
import struct

import numpy as np

SEED = 20261016
PMT_PID, PCR_PID, VIDEO_PID, PGS_PID = 0x100, 0x1001, 0x1011, 0x1200
AUDIO_PID = 0x1100
NULL_PID = 0x1FFF
CH_CODE = {1: 1, 2: 3, 3: 4, 4: 6, 5: 8, 6: 9, 7: 10, 8: 11}
RATE_CODE = {48000: 1, 96000: 4, 192000: 5}
BITS_CODE = {16: 1, 20: 2, 24: 3}
HDMV_REG = b'\x05\x04HDMV'


def crc32_mpeg(data):
    crc = 0xFFFFFFFF
    for b in data:
        crc ^= b << 24
        for _ in range(8):
            crc = ((crc << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if crc & 0x80000000 else (crc << 1) & 0xFFFFFFFF
    return crc


def section(table_id, ext, body):
    n = 5 + len(body) + 4
    sec = bytes([table_id, 0xB0 | (n >> 8), n & 0xFF, ext >> 8, ext & 0xFF, 0xC1, 0, 0]) + body
    return sec + crc32_mpeg(sec).to_bytes(4, 'big')


def pts_bytes(pts, prefix=0x20):
    return bytes([prefix | ((pts >> 29) & 0x0E) | 1, (pts >> 22) & 0xFF, ((pts >> 14) & 0xFE) | 1, (pts >> 7) & 0xFF,
                  ((pts << 1) & 0xFE) | 1])


def pes(stream_id, payload, pts, ext_id=None, unbounded=False):
    """A PES packet: PTS, and PES extension 2 carrying stream_id_extension when ext_id is given."""
    opt = pts_bytes(pts)
    flags = 0x80
    if ext_id is not None:
        opt += bytes([0x01, 0x81, ext_id])          # extension flags: PES extension 2 only; marker + length 1; the id
        flags |= 0x01
    body = bytes([0x81, flags, len(opt)]) + opt + payload
    return b'\x00\x00\x01' + bytes([stream_id]) + struct.pack('>H', 0 if unbounded else len(body)) + body


class Stream(object):
    """One elementary stream of a case: `kind` ('lpcm', 'truehd', 'ac3', 'video', 'pgs'), its PES packets, and for
    audio the PCM it decodes to (int16, frames x channels) and each PES's frame count."""

    def __init__(self, pid, stream_type, kind):
        self.pid, self.stream_type, self.kind = pid, stream_type, kind
        self.pes, self.pes_frames = [], []
        self.pcm, self.rate, self.channels, self.bits = None, 0, 0, 0
        self.header_len = 14


def lpcm_stream(pid, channels, bits, rate, seconds, rng, max_frames=600, leftover=True, pcm=None):
    """BD-LPCM PES packets of `pcm` (frames x channels samples at `bits`; default: a seeded signal of `seconds`)."""
    s = Stream(pid, 0x80, 'lpcm')
    s.rate, s.channels, s.bits = rate, channels, bits
    full = (1 << (bits - 1)) - 1
    if pcm is None:
        frames = int(seconds * rate)
        t = np.arange(frames) / float(rate)
        pcm = np.zeros((frames, channels), np.int64)
        for c in range(channels):
            f = 180.0 + 70.0 * c + rng.random() * 40
            x = 0.7 * np.sin(2 * np.pi * f * t + c) + 0.25 * rng.standard_normal(frames)
            pcm[:, c] = np.clip(np.round(x * 0.45 * full), -full - 1, full)
        pcm[rng.integers(frames), 0] = full                   # full scale both ways
        pcm[rng.integers(frames), channels - 1] = -full - 1
    pcm = np.asarray(pcm, np.int64)
    frames = len(pcm)
    src = channels + (channels & 1)
    width = 2 if bits == 16 else 3
    coded = pcm << (24 - bits) if width == 3 else pcm
    raw = np.zeros((frames, src, width), np.uint8)
    u = coded.astype(np.int64) & ((1 << (8 * width)) - 1)
    for k in range(width):
        raw[:, :channels, k] = (u >> (8 * (width - 1 - k))) & 0xFF
    if channels & 1:
        raw[:, channels, :] = rng.integers(1, 256, (frames, width))       # the padding channel is not silent
    s.pcm = (coded >> 8 if width == 3 else pcm).astype(np.int16)
    s.raw = raw
    at, k = 0, 0
    hdr_tail = bytes([CH_CODE[channels] << 4 | RATE_CODE[rate], BITS_CODE[bits] << 6])
    while at < frames:
        n = int(min(frames - at, rng.integers(1, max_frames + 1) if k % 3 else max_frames // 3 + 1))
        audio = raw[at:at + n].tobytes()
        extra = rng.integers(0, 256, int(rng.integers(1, src * width))).astype(np.uint8).tobytes() \
            if leftover and k % 5 == 4 else b''
        s.pes.append(pes(0xBD, struct.pack('>H', len(audio)) + hdr_tail + audio + extra, 9000 + at))
        s.pes_frames.append(n)
        at += n
        k += 1
    return s


def truehd_stream(pid, case, rng, ac3=True):
    s = Stream(pid, 0x83, 'truehd')
    s.rate, s.channels, s.bits, s.pcm = case.rate, case.channels, 24, case.pcm16
    s.header_len = 17
    data, at = case.data, 0
    while at < len(data):
        n = int(rng.integers(200, 3000))
        s.pes.append(pes(0xFD, data[at:at + n], 9000 + at, ext_id=0x72))
        s.pes_frames.append(0)
        at += n
        if ac3 and rng.random() < 0.5:
            frame = b'\x0b\x77' + rng.integers(0, 256, int(rng.integers(100, 700))).astype(np.uint8).tobytes()
            s.pes.append(pes(0xFD, frame, 9000 + at, ext_id=0x76))
            s.pes_frames.append(None)                      # the AC-3 sub-stream
    return s


def blob_stream(pid, stream_type, kind, n, size, rng):
    s = Stream(pid, stream_type, kind)
    for k in range(n):
        body = rng.integers(1, 256, int(rng.integers(size // 4, size))).astype(np.uint8).tobytes()
        if kind == 'video':
            body = b'\x00\x00\x00\x01\x09\xf0' + body      # an access unit delimiter, then no start code
        s.pes.append(pes(0xE0 if kind == 'video' else 0xBD, body, 3000 * k, unbounded=kind == 'video'))
        s.pes_frames.append(None)
    return s


class TsCase(object):
    """A transport stream with what it decodes to.  `packets`: (file offset, PID, PES index or None, payload bytes,
    payload-unit start) per packet; `damage`: (regex, byte offset) for a damaged copy; `cut`: the file length of a cut
    copy."""

    def __init__(self, name, psize, hdmv, streams, rng, programs=1, af_sweep=True):
        self.name, self.psize, self.hdmv, self.streams = name, psize, hdmv, streams
        self.damage, self.cut, self.refused = None, None, None
        self.programs = programs
        self._build(rng, af_sweep)

    @property
    def ext(self):
        return '.m2ts' if self.psize == 192 else '.ts'

    def audio(self):
        return [s for s in self.streams if s.kind in ('lpcm', 'truehd')]

    def tables(self):
        body = b''.join(struct.pack('>HH', 1 + p, 0xE000 | (PMT_PID + p)) for p in range(self.programs))
        pat = section(0x00, 1, body)
        info = HDMV_REG if self.hdmv else b''
        es = b''.join(bytes([s.stream_type]) + struct.pack('>HH', 0xE000 | s.pid, 0xF000) for s in self.streams)
        pmt = section(0x02, 1, struct.pack('>HH', 0xE000 | PCR_PID, 0xF000 | len(info)) + info + es)
        return pat, pmt

    def _build(self, rng, af_sweep):
        pat, pmt = self.tables()
        cc = {}
        out = []                                            # (pid, 188 bytes, pes index or None, payload len, pusi)
        sweep = iter(range(0, 183)) if af_sweep else iter(())

        def packet(pid, payload=b'', pusi=False, af=None, tag=None):
            if af is None and len(payload) < 184:
                n = 183 - len(payload)
                af = b'' if n == 0 else b'\x00' + b'\xff' * (n - 1)
            afc = (2 if af is not None else 0) | (1 if payload else 0)
            c = cc.get(pid, 0)
            head = bytes([0x47, (0x40 if pusi else 0) | (pid >> 8), pid & 0xFF, (afc << 4) | c])
            if payload:
                cc[pid] = (c + 1) & 15
            pk = head + (bytes([len(af)]) + af if af is not None else b'') + payload
            assert len(pk) == 188, len(pk)
            out.append((pid, pk, tag, len(payload), pusi))

        def tables():
            for pid, sec in ((0, pat), (PMT_PID, pmt)):
                packet(pid, b'\x00' + sec + b'\xff' * (183 - len(sec)), pusi=True)

        def split(data):
            """payload sizes: mostly 184, some shorter (an adaptation field of every length)"""
            at = 0
            while at < len(data):
                n = next(sweep, None) if rng.random() < 0.3 else None
                n = 183 - n if n is not None else 184
                yield data[at:at + n], at == 0
                at += n

        queues = []
        for s in self.streams:
            q = []
            for k, p in enumerate(s.pes):
                for chunk, first in split(p):
                    q.append((s.pid, chunk, first, (s.pid, k)))
            queues.append(q)
        tables()
        heads = [0] * len(queues)
        remaining = sum(len(q) for q in queues)
        step = 0
        while remaining:
            weights = np.array([len(q) - h for q, h in zip(queues, heads)], np.float64)
            i = int(rng.choice(len(queues), p=weights / weights.sum()))
            pid, chunk, first, tag = queues[i][heads[i]]
            packet(pid, chunk, pusi=first, tag=tag)
            heads[i] += 1
            remaining -= 1
            step += 1
            if step % 97 == 0:
                tables()
            if rng.random() < 0.02:
                packet(NULL_PID, rng.integers(0, 256, 184).astype(np.uint8).tobytes())
            if rng.random() < 0.02:                     # PCR only: an adaptation field filling the packet
                pcr = int(step) * 300
                packet(PCR_PID, af=bytes([0x10]) + struct.pack('>IH', pcr >> 1, ((pcr & 1) << 15) | 0x7E00)
                       + b'\xff' * 176)
        chunks, self.packets = [], []
        at = 0
        for k, (pid, pk, tag, n, pusi) in enumerate(out):
            if self.psize == 192:
                pk = struct.pack('>I', (k * 1024) & 0x3FFFFFFF) + pk
            chunks.append(pk)
            self.packets.append((at, pid, tag, n, pusi))
            at += self.psize
        self.data = b''.join(chunks)

    def pes_offset(self, pid, k):
        """Byte offset of the packet that starts PES k of `pid`."""
        return next(at for at, p, tag, _, pusi in self.packets if tag == (pid, k) and pusi)

    def expected(self, s):
        """The PCM FFmpeg gives for stream s of this copy (cut copies keep the whole sample frames of a last PES
        whose whole packets survive the cut)."""
        if self.cut is None or s.kind != 'lpcm':
            return s.pcm
        kept = {}
        for at, pid, tag, n, _ in self.packets:
            if pid == s.pid and at + self.psize <= self.cut:
                kept[tag[1]] = kept.get(tag[1], 0) + n
        frames = 0
        width = 2 if s.bits == 16 else 3
        src = s.channels + (s.channels & 1)
        for k, nf in enumerate(s.pes_frames):
            got = kept.get(k, 0)
            if got == len(s.pes[k]):
                frames += nf
            elif got:
                frames += max(0, got - s.header_len - 4) // (src * width) if got >= s.header_len else 0
                break
            else:
                break
        return s.pcm[:frames]

    def write(self, directory, data=None):
        path = os.path.join(str(directory), self.name + self.ext)
        with open(path, 'wb') as f:
            f.write(self.data if data is None else data)
        return path

    def __repr__(self):
        return 'TsCase(%s)' % self.name


def write_wav(path, pcm16, rate):
    """The plain 16-bit PCM WAV of `pcm16` (frames x channels)."""
    body = np.ascontiguousarray(pcm16, '<i2').tobytes()
    ch = pcm16.shape[1]
    with open(str(path), 'wb') as f:
        f.write(b'RIFF' + struct.pack('<I', 36 + len(body)) + b'WAVEfmt ' +
                struct.pack('<IHHIIHH', 16, 1, ch, rate, rate * ch * 2, ch * 2, 16) + b'data' +
                struct.pack('<I', len(body)) + body)
    return str(path)


def long_m2ts(path, minutes=90.0, seed=60, bits=24, video_packets=0):
    """A BDAV stream of `minutes` of 48 kHz stereo LPCM at `bits`: one second of PES packets (240 frames each, 1600
    or 1200 TS packets per second) and `video_packets` (a multiple of 16) video filler packets spread between them,
    written over and over after one PAT and PMT (every continuity counter wraps evenly).  Returns (the second's int16
    PCM, repetitions)."""
    rng = _rng(seed)
    s = lpcm_stream(AUDIO_PID, 2, bits, 48000, 1.0, rng, leftover=False)
    filler = rng.integers(0, 256, 184).astype(np.uint8).tobytes()
    s.pes, s.pes_frames = [], []
    case = TsCase.__new__(TsCase)
    case.programs, case.hdmv, case.streams = 1, True, [s]
    pat, pmt = case.tables()
    head = b''.join(struct.pack('>I', 0) + bytes([0x47, 0x40 | (pid >> 8), pid & 0xFF, 0x10]) + b'\x00' + sec +
                    b'\xff' * (183 - len(sec)) for pid, sec in ((0, pat), (PMT_PID, pmt)))
    raw = s.raw
    out = bytearray()
    k = v = 0
    for at in range(0, 48000, 240):
        for _ in range(video_packets * (at // 240 + 1) // 200 - video_packets * (at // 240) // 200):
            out += struct.pack('>I', 0) + bytes([0x47, VIDEO_PID >> 8, VIDEO_PID & 0xFF, 0x10 | (v & 15)]) + filler
            v += 1
        audio = raw[at:at + 240].tobytes()
        data = pes(0xBD, struct.pack('>H', len(audio)) + bytes([0x31, BITS_CODE[bits] << 6]) + audio, 9000 + at)
        for j in range(0, len(data), 184):
            chunk = data[j:j + 184]
            af = b'' if len(chunk) == 184 else bytes([183 - len(chunk)]) + (b'\x00' + b'\xff' * (182 - len(chunk))
                                                                            if len(chunk) < 183 else b'')
            out += struct.pack('>I', k * 1024) + bytes([0x47, (0x40 if j == 0 else 0) | (AUDIO_PID >> 8),
                                                        AUDIO_PID & 0xFF, (0x30 if af else 0x10) | (k & 15)]) + af + chunk
            k += 1
    assert k % 16 == 0 and v % 16 == 0 and len(out) == (k + v) * 192
    reps = int(round(minutes * 60))
    seg = bytes(out)
    with open(str(path), 'wb') as f:
        f.write(head)
        for _ in range(reps):
            f.write(seg)
    return s.pcm, reps


def _rng(seed):
    return np.random.default_rng([SEED, seed])


def make_cases():
    from tests import truehd_cases as tc
    cases = []

    def add(name, psize, hdmv, build, seed, **kw):
        rng = _rng(seed)
        cases.append(TsCase(name, psize, hdmv, build(rng), rng, **kw))

    add('bd_stereo16_48k', 192, True, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 12, 30000, r),
        lpcm_stream(AUDIO_PID, 2, 16, 48000, 0.8, r),
        blob_stream(PGS_PID, 0x90, 'pgs', 4, 400, r)], 1)
    add('bd_mono16_96k', 192, True, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 4, 20000, r), lpcm_stream(AUDIO_PID, 1, 16, 96000, 0.4, r, max_frames=30)], 2)
    add('bd_stereo20_48k', 192, True, lambda r: [lpcm_stream(AUDIO_PID, 2, 20, 48000, 0.1, r)], 13)
    add('bd_3ch24_192k', 192, True, lambda r: [lpcm_stream(AUDIO_PID, 3, 24, 192000, 0.2, r, max_frames=900)], 3)
    add('bd_6ch16_48k', 192, True, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 4, 20000, r), lpcm_stream(AUDIO_PID, 6, 16, 48000, 0.4, r)], 4)
    add('bd_8ch24_48k', 192, True, lambda r: [lpcm_stream(AUDIO_PID, 8, 24, 48000, 0.3, r)], 5)
    add('ts_stereo24_48k', 188, True, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 6, 20000, r), lpcm_stream(AUDIO_PID, 2, 24, 48000, 0.6, r)], 6)
    add('bd_two_lpcm', 192, True, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 4, 20000, r), lpcm_stream(AUDIO_PID, 2, 16, 48000, 0.4, r),
        lpcm_stream(AUDIO_PID + 1, 2, 24, 48000, 0.4, r), blob_stream(PGS_PID, 0x90, 'pgs', 3, 300, r)], 7)
    thd = tc.make('ts_thd', 2, 24, 48000, n_au=160, seed=3, style=tc.FULL, restarts=(7, 16, 1, 30))
    add('bd_truehd', 192, True, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 4, 20000, r), truehd_stream(AUDIO_PID, thd, r)], 8)
    thd6 = tc.make('ts_thd6', 6, 24, 48000, n_au=80, n_sub=2, seed=8, style=tc.FULL, restarts=(13,))
    add('bd_truehd_6ch', 192, True, lambda r: [truehd_stream(AUDIO_PID, thd6, r),
                                               lpcm_stream(AUDIO_PID + 1, 2, 16, 48000, 0.1, r)], 9)
    add('ts_no_hdmv', 188, False, lambda r: [
        blob_stream(VIDEO_PID, 0x1B, 'video', 2, 5000, r), lpcm_stream(AUDIO_PID, 2, 16, 48000, 0.05, r),
        Stream(AUDIO_PID + 1, 0x83, 'private'), Stream(AUDIO_PID + 2, 0x81, 'private'),
        blob_stream(AUDIO_PID + 3, 0x0F, 'aac', 2, 300, r)], 10)
    add('bd_lossy', 192, True, lambda r: [
        blob_stream(AUDIO_PID, 0x81, 'ac3', 3, 500, r), blob_stream(AUDIO_PID + 1, 0x86, 'dts', 3, 500, r)], 11)
    add('bd_two_programs', 192, True, lambda r: [lpcm_stream(AUDIO_PID, 2, 16, 48000, 0.05, r)], 12, programs=2)
    cases[-1].refused = 'has 2 programs'
    return cases


_ALL = None


def all_cases():
    """Every undamaged case, built once."""
    global _ALL
    if _ALL is None:
        _ALL = make_cases()
        assert_coverage(_ALL)
    return _ALL


def case(name):
    return next(c for c in all_cases() if c.name == name)


def _copy(base, name, data, regex, offset):
    c = object.__new__(TsCase)
    c.__dict__.update(base.__dict__)
    c.name, c.data, c.damage = name, bytes(data), (regex, offset)
    return c


def damaged_cases():
    """Copies of bd_stereo16_48k (and ts_stereo24_48k) with one fault each, and the byte offset the refusal names."""
    out = []
    for base in (case('bd_stereo16_48k'), case('ts_stereo24_48k')):
        p, h = base.psize, base.psize - 188
        audio = [(at, tag, n, pusi) for at, pid, tag, n, pusi in base.packets if pid == AUDIO_PID]
        mid = audio[len(audio) // 2][0]
        short = base.name.split('_')[0]

        def with_byte(at, fn):
            d = bytearray(base.data)
            d[at] = fn(d[at])
            return d
        out.append(_copy(base, short + '_lost_sync', with_byte(mid + h, lambda b: 0x46), 'lost sync', mid))
        out.append(_copy(base, short + '_tei', with_byte(mid + h + 1, lambda b: b | 0x80), 'transport error', mid))
        out.append(_copy(base, short + '_scrambled', with_byte(mid + h + 3, lambda b: b | 0x80), 'scrambled', mid))
        out.append(_copy(base, short + '_cc_gap', with_byte(mid + h + 3, lambda b: (b & 0xF0) | ((b + 3) & 15)),
                         'continuity counter', mid))
        # a PES whose PES_packet_length is one too large, and one whose LPCM header gives another sample rate
        starts = [(at, tag) for at, tag, n, pusi in audio if pusi and n >= 20]
        at, tag = starts[len(starts) // 2]
        off = at + p - 188 + 4 + (1 + base.data[at + h + 4] if (base.data[at + h + 3] >> 4) & 2 else 0)
        d = bytearray(base.data)
        ln = struct.unpack('>H', d[off + 4:off + 6])[0]
        d[off + 4:off + 6] = struct.pack('>H', ln + 1)
        out.append(_copy(base, short + '_pes_length', d, 'PES_packet_length', at))
        at2, _ = starts[len(starts) // 2 + 1]
        off2 = at2 + p - 188 + 4 + (1 + base.data[at2 + h + 4] if (base.data[at2 + h + 3] >> 4) & 2 else 0)
        out.append(_copy(base, short + '_lpcm_change', with_byte(off2 + 14 + 2, lambda b: (b & 0xF0) | 4),
                         'BD-LPCM header changes', at2))
        # the CRC of the first PAT and of the first PMT
        first_pat = next(a for a, pid, _, _, _ in base.packets if pid == 0)
        first_pmt = next(a for a, pid, _, _, _ in base.packets if pid == PMT_PID)
        out.append(_copy(base, short + '_pat_crc', with_byte(first_pat + h + 5 + 9, lambda b: b ^ 1), 'PAT section',
                         first_pat))
        out.append(_copy(base, short + '_pmt_crc', with_byte(first_pmt + h + 5 + 12, lambda b: b ^ 1), 'PMT section',
                         first_pmt))
    return out


def cut_cases():
    """Copies cut short: inside a packet in the middle of a PES, and at a packet edge inside a PES."""
    out = []
    for base in (case('bd_stereo16_48k'), case('ts_stereo24_48k'), case('bd_6ch16_48k')):
        audio = [(at, tag, pusi) for at, pid, tag, n, pusi in base.packets if pid == AUDIO_PID]
        k = int(len(audio) * 0.6)
        while audio[k][2] or audio[k - 1][2] or audio[k - 2][2]:
            k += 1                                        # the third packet of a PES or later: whole frames remain
        for name, length in (('cut_in_packet', audio[k][0] + 100), ('cut_at_packet', audio[k][0])):
            c = _copy(base, base.name + '_' + name, base.data[:length], None, None)
            c.damage, c.cut = None, length
            out.append(c)
    return out


def assert_coverage(cases):
    lp = [s for c in cases for s in c.streams if s.kind == 'lpcm']
    assert {s.bits for s in lp} == {16, 20, 24}           # 20 bits: refused, as FFmpeg refuses it
    assert {1, 2, 3, 6, 8} <= {s.channels for s in lp}
    assert {s.rate for s in lp} == {48000, 96000, 192000}
    assert {c.psize for c in cases} == {188, 192} and {c.hdmv for c in cases} == {True, False}
    assert any(len(c.audio()) > 1 for c in cases) and any(s.kind == 'pgs' for c in cases for s in c.streams)
    assert any(s.kind == 'truehd' for c in cases for s in c.streams)
    # every adaptation field length, PCR-only packets, null packets, PES of one and of many packets
    afs, pcr, null = set(), False, False
    for c in cases:
        h = c.psize - 188
        for at, pid, _, n, _ in c.packets:
            pk = c.data[at + h:at + c.psize]
            if (pk[3] >> 4) & 2:
                afs.add(pk[4])
            pcr |= pid == PCR_PID and pk[4] == 183
            null |= pid == NULL_PID
    assert afs >= set(range(184)) and pcr and null, sorted(set(range(184)) - afs)
    spans = {}
    for c in cases:
        for _, pid, tag, _, _ in c.packets:
            if tag and pid == AUDIO_PID:
                spans[(c.name, tag)] = spans.get((c.name, tag), 0) + 1
    assert min(spans.values()) == 1 and max(spans.values()) > 10
    # some LPCM PES carry leftover bytes after their last whole frame
    assert any(len(p) - 18 > f * (s.channels + (s.channels & 1)) * (2 if s.bits == 16 else 3)
               for s in lp for p, f in zip(s.pes, s.pes_frames))
