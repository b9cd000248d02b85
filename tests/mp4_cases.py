"""A seeded MP4 / QuickTime writer for the tests: files whose streams, samples, chapters and PCM are known, refused and
damaged copies, cut copies and a sparse file whose `mdat` lies past 4 GiB.

`assert_coverage` checks that the files together use every box and sound-description form sushi_b200/mp4.py reads:
`moov` first and last, files without `ftyp`, `co64`, `stz2`, multi-run `stsc`, ISO / v0 / v1 / v2 / `wave` / `ipcm`
sound descriptions, `enda`, two audio tracks with different enabled flags beside random-byte video, `mov_text`, a
chapter text track and `chpl`, identity and refused edit lists."""
import os
import struct

import numpy as np

from tests import alac_cases as ac
from tests import mkv_cases as mc

SEED = 4711


def box(btype, *parts):
    body = b''.join(parts)
    return struct.pack('>I4s', 8 + len(body), btype) + body


def full(btype, version, flags, *parts):
    return box(btype, struct.pack('>I', (version << 24) | flags), *parts)


class Trak(object):
    """A track to write.  samples: its sample payloads (PCM: one payload per chunk, `frames` frames each);
    per_chunk: samples per chunk, cycled."""

    def __init__(self, handler, entry, samples, durations, timescale, enabled=True, per_chunk=(1,), pcm=None,
                 bits=16, codec=None, kind=None, chap=None, edits='identity', sizes='stsz',
                 offsets='stco', channels=0, rate=0, frames=None):
        self.handler, self.entry, self.samples, self.durations = handler, entry, samples, durations
        self.timescale, self.enabled, self.per_chunk, self.pcm, self.bits = timescale, enabled, per_chunk, pcm, bits
        self.codec, self.kind, self.chap, self.edits = codec, kind, chap, edits
        self.sizes, self.offsets, self.channels, self.rate = sizes, offsets, channels, rate
        self.frames = frames                     # PCM: frames per chunk payload
        self.stsz_size = 1                       # PCM: stsz's constant sample size (ISO ipcm: bytes per frame)


class Mp4Case(object):
    """`expect[stream id]` = (kind, codec, default); `chapters` the starts FFmpeg lists in seconds; `audio` the stream
    ids with PCM; `damage` / `refused`: regex of the refusal."""

    def __init__(self, name, data, traks, expect, chapters, used, refused=None, damage=None, cut=False, suffix='.mp4'):
        self.name, self.data, self.traks, self.expect, self.chapters = name, data, traks, expect, chapters
        self.used, self.refused, self.damage, self.cut, self.suffix = used, refused, damage, cut, suffix

    def write(self, directory):
        path = os.path.join(str(directory), self.name + self.suffix)
        with open(path, 'wb') as f:
            f.write(self.data)
        return path

    def audio_ids(self):
        return [i for i, t in enumerate(self.traks) if t.pcm is not None]

    def __repr__(self):
        return 'Mp4Case(%s)' % self.name


def sound_entry(fourcc, channels, bits, rate, version=0, kids=b'', v1=(1, 2, 4, 2), v2=None):
    head = bytes(6) + struct.pack('>H', 1)
    if version == 2:
        flags, bpf = v2
        body = struct.pack('>HHI', 2, 0, 0) + struct.pack('>HHHHI', 3, 16, 0xFFFE, 0, 65536)
        body += struct.pack('>IdIIIIII', 72, float(rate), channels, 0x7F000000, bits, flags, bpf, 1)
    else:
        body = struct.pack('>HHI', version, 0, 0) + struct.pack('>HHHHI', channels, bits, 0, 0, rate << 16)
        if version == 1:
            body += struct.pack('>IIII', *v1)
    return box(fourcc, head, body, kids)


def alac_entry(case, form='iso'):
    cookie = full(b'alac', 0, 0, case.cfg.cookie())
    if form == 'iso':
        return sound_entry(b'alac', case.channels, case.bits, case.rate, kids=cookie)
    wave = box(b'wave', box(b'frma', b'alac'), cookie, bytes(8))
    return sound_entry(b'alac', case.channels, case.bits, case.rate, version=1, kids=wave,
                       v1=(case.cfg.frame_length, 1, 2 * case.channels, 2))


def video_entry():
    return box(b'avc1', bytes(6) + struct.pack('>H', 1), bytes(16), struct.pack('>HH', 64, 36), bytes(50))


def text_entry(fourcc):
    return box(fourcc, bytes(6) + struct.pack('>H', 1), bytes(40))


def esds(oti):
    dec = bytes([4, 13, oti, 0x15]) + bytes(11)
    es = bytes([3, 3 + 2 + len(dec)]) + b'\x00\x01\x00' + dec
    return full(b'esds', 0, 0, es)


def _stbl(t, chunk_offsets):
    n = len(t.samples)
    ent = full(b'stsd', 0, 0, struct.pack('>I', 1), t.entry)
    if t.durations:
        runs = []
        for d in t.durations:
            if runs and runs[-1][1] == d:
                runs[-1][0] += 1
            else:
                runs.append([1, d])
        stts = full(b'stts', 0, 0, struct.pack('>I', len(runs)), b''.join(struct.pack('>II', *r) for r in runs))
    else:
        stts = full(b'stts', 0, 0, struct.pack('>I', 0))
    counts = t.frames if t.frames is not None else _chunk_counts(t)
    runs = []
    for k, c in enumerate(counts):
        if not runs or runs[-1][1] != c:
            runs.append((k + 1, c))
    stsc = full(b'stsc', 0, 0, struct.pack('>I', len(runs)), b''.join(struct.pack('>III', a, c, 1) for a, c in runs))
    if t.frames is not None:                               # PCM: a sample is one frame
        total = sum(t.frames)
        stsz = full(b'stsz', 0, 0, struct.pack('>II', t.stsz_size, total))
    elif t.sizes == 'stz2':
        stsz = full(b'stz2', 0, 0, bytes([0, 0, 0, 16]), struct.pack('>I', n), struct.pack('>%dH' % n, *[len(s) for s in t.samples]))
    else:
        stsz = full(b'stsz', 0, 0, struct.pack('>II', 0, n), struct.pack('>%dI' % n, *[len(s) for s in t.samples]))
    if t.offsets == 'co64':
        co = full(b'co64', 0, 0, struct.pack('>I', len(chunk_offsets)), struct.pack('>%dQ' % len(chunk_offsets),
                                                                                   *chunk_offsets))
    else:
        co = full(b'stco', 0, 0, struct.pack('>I', len(chunk_offsets)), struct.pack('>%dI' % len(chunk_offsets),
                                                                                   *chunk_offsets))
    return box(b'stbl', ent, stts, stsc, stsz, co)


def _chunk_counts(t):
    counts, k, i = [], 0, 0
    while i < len(t.samples):
        c = min(t.per_chunk[k % len(t.per_chunk)], len(t.samples) - i)
        counts.append(c)
        i += c
        k += 1
    return counts


def _trak(t, track_id, chunk_offsets, movie_ts):
    dur = sum(t.durations)
    tkhd = full(b'tkhd', 0, 1 if t.enabled else 0, struct.pack('>IIII', 0, 0, track_id, 0),
                struct.pack('>I', dur * movie_ts // t.timescale), bytes(60))
    mdhd = full(b'mdhd', 0, 0, struct.pack('>IIII', 0, 0, t.timescale, dur), struct.pack('>HH', 0x55C4, 0))
    hdlr = full(b'hdlr', 0, 0, b'mhlr' if t.handler != b'soun' else bytes(4), t.handler, bytes(12), b'x\0')
    dref = full(b'dref', 0, 0, struct.pack('>I', 1), full(b'url ', 0, 1 if t.edits != 'external' else 0))
    minf = box(b'minf', full(b'smhd', 0, 0, bytes(4)), box(b'dinf', dref), _stbl(t, chunk_offsets))
    kids = [tkhd]
    if t.chap:
        kids.append(box(b'tref', box(b'chap', struct.pack('>I', t.chap))))
    movie_dur = -(-dur * movie_ts // t.timescale)                 # an identity edit covers the whole track
    if t.edits == 'identity':
        kids.append(box(b'edts', full(b'elst', 0, 0, struct.pack('>I', 1), struct.pack('>Iii', movie_dur, 0, 0x10000))))
    elif t.edits == 'shift':
        kids.append(box(b'edts', full(b'elst', 0, 0, struct.pack('>I', 1), struct.pack('>Iii', movie_dur // 2, 1024,
                                                                                         0x10000))))
    elif t.edits == 'rate':
        kids.append(box(b'edts', full(b'elst', 0, 0, struct.pack('>I', 1), struct.pack('>Iii', movie_dur * 2, 0,
                                                                                         0x8000))))
    elif t.edits == 'two':
        kids.append(box(b'edts', full(b'elst', 0, 0, struct.pack('>I', 2), struct.pack('>Iii', 100, -1, 0x10000),
                                      struct.pack('>Iii', movie_dur, 0, 0x10000))))
    kids.append(box(b'mdia', mdhd, hdlr, minf))
    return box(b'trak', *kids)


def build(name, traks, moov_first=True, ftyp=b'isom', chpl=None, extra_moov=b'', mdat_gap=0, lead=b'',
          suffix='.mp4'):
    """The file's bytes: [lead] [ftyp] moov mdat (or mdat moov); chunks of the tracks interleaved round-robin."""
    movie_ts = 1000
    # the chunks in file order: round-robin over the tracks
    per = []
    for t in traks:
        counts = _chunk_counts(t)
        chunks, i = [], 0
        for c in counts:
            chunks.append(b''.join(t.samples[i:i + c]))
            i += c
        per.append(chunks)
    order = []
    k = 0
    while any(k < len(c) for c in per):
        for ti, c in enumerate(per):
            if k < len(c):
                order.append((ti, k))
        k += 1
    head = lead + (box(b'ftyp', ftyp, struct.pack('>I', 0), ftyp, b'mp41') if ftyp else b'')

    def moov_bytes(offsets):
        kids = [full(b'mvhd', 0, 0, struct.pack('>IIII', 0, 0, movie_ts, 0), bytes(80))]
        kids += [_trak(t, i + 1, offsets[i], movie_ts) for i, t in enumerate(traks)]
        if chpl is not None:
            kids.append(box(b'udta', full(b'chpl', 1, 0, bytes(4), bytes([len(chpl)]),
                                          b''.join(struct.pack('>QB', s, 3) + b'ch%d' % (k % 10) for k, s in
                                                   enumerate(chpl)))))
        return box(b'moov', *kids, extra_moov)

    offsets = [[0] * len(c) for c in per]
    moov_len = len(moov_bytes(offsets))
    payload = b''.join(per[ti][k] for ti, k in order)
    mdat_hdr = struct.pack('>I4s', 8 + len(payload), b'mdat') if 8 + len(payload) < 2 ** 32 else \
        struct.pack('>I4sQ', 1, b'mdat', 16 + len(payload))
    base = len(head) + (moov_len if moov_first else 0) + mdat_gap + len(mdat_hdr)
    at = base
    for ti, k in order:
        offsets[ti][k] = at
        at += len(per[ti][k])
    moov = moov_bytes(offsets)
    assert len(moov) == moov_len
    mdat = mdat_hdr + payload
    return head + (moov + mdat if moov_first else mdat + moov) if not mdat_gap else (head, moov, mdat)


# ---- tracks -----------------------------------------------------------------------------------------------------------
def alac_trak(case, form='iso', enabled=True, per_chunk=(3, 3, 2), **kw):
    durs = [ac.frame_samples(case.cfg, f) for f in case.frames]
    return Trak(b'soun', alac_entry(case, form), list(case.frames), durs, case.rate, enabled=enabled,
                per_chunk=per_chunk, pcm=case.pcm, bits=case.bits, codec='alac', kind='audio', channels=case.channels,
                rate=case.rate, **kw)


def pcm_trak(fourcc, channels, bits, rate, n_frames, seed, big, version=0, enda=None, enabled=True, per_chunk=800,
             v2flags=None, ipcm=False, **kw):
    rng = np.random.default_rng([SEED, seed])
    top = (1 << (bits - 1)) - 1
    t = np.arange(n_frames)
    pcm = np.stack([np.clip(np.round(top * 0.4 * np.sin(2 * np.pi * (0.003 + 0.002 * c) * t) +
                                     rng.normal(0, top * 0.01, n_frames)), -top - 1, top).astype(np.int64)
                    for c in range(channels)], 1)
    width = bits // 8
    raw = pcm.astype('<i4').view(np.uint8).reshape(n_frames, channels, 4)[:, :, :width]
    if big:
        raw = raw[:, :, ::-1]
    data = np.ascontiguousarray(raw).reshape(n_frames, -1)
    chunks, frames = [], []
    for a in range(0, n_frames, per_chunk):
        chunks.append(data[a:a + per_chunk].tobytes())
        frames.append(min(per_chunk, n_frames - a))
    kids = b''
    if enda is not None:
        kids = box(b'wave', box(b'frma', fourcc), box(b'enda', struct.pack('>H', enda)), bytes(8))
    if ipcm:
        kids = full(b'pcmC', 0, 0, bytes([0 if big else 1, bits]))
    fb = channels * width
    entry = sound_entry(fourcc, channels, bits, rate, version=version, kids=kids, v1=(1, width, fb, width),
                        v2=(v2flags, fb) if version == 2 else None)
    codec = 'pcm_s%d%s' % (bits, 'be' if big else 'le')
    t = Trak(b'soun', entry, chunks, [1] * n_frames, rate, enabled=enabled, per_chunk=(1,), pcm=pcm, bits=bits,
                codec=codec, kind='audio', frames=frames, channels=channels, rate=rate, **kw)
    if ipcm:
        t.stsz_size = fb
    return t


def video_trak(count, seed, chap=None):
    rng = np.random.default_rng([SEED, seed])
    samples = [rng.integers(0, 256, int(rng.integers(300, 900)), dtype=np.uint8).tobytes() for _ in range(count)]
    return Trak(b'vide', video_entry(), samples, [1001] * count, 24000, per_chunk=(4,), codec='h264', kind='video',
                chap=chap, edits=None)


def text_trak(handler, fourcc, texts, durations, timescale=1000, enabled=False):
    samples = [struct.pack('>H', len(s)) + s for s in texts]
    return Trak(handler, text_entry(fourcc), samples, durations, timescale, enabled=enabled, per_chunk=(1,),
                codec='mov_text', kind='subtitles', edits=None)


def as_chapter_track(t):
    """FFmpeg lists a track `tref/chap` names, unless it is video, as a data stream"""
    t.kind, t.codec = 'data', 'bin_data'
    return t


def aac_trak(seed, enabled=True):
    rng = np.random.default_rng([SEED, seed])
    samples = [rng.integers(0, 256, 200, dtype=np.uint8).tobytes() for _ in range(10)]
    entry = sound_entry(b'mp4a', 2, 16, 48000, kids=esds(0x40))
    return Trak(b'soun', entry, samples, [1024] * 10, 48000, enabled=enabled, per_chunk=(5,), codec='aac',
                kind='audio', edits=None)


def flac_trak(seed):
    spec = mc.flac_track(9000, 2, 16, 44100, 1152, seed)
    info = spec.private[4:]
    streaminfo = bytes([0x80]) + info[1:38]
    entry = sound_entry(b'fLaC', 2, 16, 44100, kids=full(b'dfLa', 0, 0, streaminfo))
    return Trak(b'soun', entry, [f for f, _, _ in spec.frames], [d for _, _, d in spec.frames], 44100, per_chunk=(2, 3),
                pcm=spec.pcm, bits=16, codec='flac', kind='audio', channels=2, rate=44100)


# ---- the cases ----------------------------------------------------------------------------------------------------------
def _case(name, traks, chapters=(), used=(), **kw):
    opts = {k: kw.pop(k) for k in ('moov_first', 'ftyp', 'chpl', 'extra_moov', 'lead') if k in kw}
    suffix = kw.pop('suffix', '.mp4')
    data = build(name, traks, **opts)
    expect = [(t.kind, t.codec, t.enabled) for t in traks]
    return Mp4Case(name, data, traks, expect, list(chapters), set(used), suffix=suffix, **kw)


def _alac(name):
    return [c for c in ac.all_cases() if c.name == name][0]


def good_cases():
    out = []
    out.append(_case('m4a_alac', [alac_trak(_alac('stereo16'))], used={'moov_first', 'ftyp', 'iso', 'multi_stsc',
                                                                        'stco', 'identity_edit'},
                     ftyp=b'M4A ', suffix='.m4a'))
    out.append(_case('mov_alac_last', [alac_trak(_alac('layout8'), form='wave', sizes='stz2', offsets='co64',
                                                 per_chunk=(2,), edits=None)],
                     used={'moov_last', 'no_ftyp', 'v1', 'wave', 'stz2', 'co64'}, moov_first=False, ftyp=None,
                     lead=box(b'wide', b''), suffix='.mov'))
    out.append(_case('mov_alac24', [alac_trak(_alac('d24'), per_chunk=(1, 4)), alac_trak(_alac('d20'), enabled=False)],
                     used={'two_alac'}, suffix='.mov'))
    # a QuickTime master: video with a chapter track, two audio tracks with different enabled flags, PCM of three
    # layouts, a mov_text subtitle, chpl
    chap_texts = [b'Intro', b'Part A', b'Part B']
    traks = [video_trak(40, 1, chap=7),
             pcm_trak(b'twos', 2, 16, 48000, 5000, 2, True, enabled=False),
             pcm_trak(b'sowt', 2, 16, 48000, 4100, 3, False, per_chunk=1000),
             pcm_trak(b'in24', 2, 24, 48000, 3000, 4, True, version=1, enda=0, enabled=False),
             pcm_trak(b'in24', 1, 24, 44100, 3000, 5, False, version=1, enda=1, enabled=False),
             text_trak(b'sbtl', b'tx3g', [b'hello', b'', b'world'], [500, 700, 900], enabled=False),
             as_chapter_track(text_trak(b'text', b'text', chap_texts, [1500, 2500, 4000]))]
    out.append(_case('mov_master', traks, chapters=[0.0, 1.5, 4.0], chpl=[0, 20000000, 30000000, 90000000],
                     used={'chpl', 'chap_track', 'video', 'mov_text', 'enda', 'v0', 'two_audio_enabled'},
                     ftyp=b'qt  ', suffix='.mov'))
    # sowt / twos by bits per sample; a plain `text` subtitle track; a tx3g track named as the chapter track
    traks = [pcm_trak(b'sowt', 2, 24, 48000, 3000, 12, False, chap=4),
             pcm_trak(b'twos', 2, 24, 44100, 2500, 13, True, enabled=False),
             text_trak(b'text', b'text', [b'one', b'two'], [400, 600], enabled=False),
             as_chapter_track(text_trak(b'sbtl', b'tx3g', [b'A', b'B', b'C'], [250, 750, 1000]))]
    out.append(_case('mov_widths', traks, chapters=[0.0, 0.25, 1.0], used={'sowt24', 'twos24', 'text_subtitle',
                                                                          'tx3g_chapter'}, ftyp=b'qt  ',
                     suffix='.mov'))
    out.append(_case('mov_lpcm', [pcm_trak(b'lpcm', 2, 24, 48000, 4000, 6, True, version=2, v2flags=0xE),
                                  pcm_trak(b'lpcm', 3, 16, 48000, 2500, 7, False, version=2, v2flags=0xC)],
                     used={'v2'}, ftyp=b'qt  ', suffix='.mov'))
    out.append(_case('mp4_ipcm', [pcm_trak(b'ipcm', 2, 16, 48000, 3000, 8, True, ipcm=True),
                                  pcm_trak(b'ipcm', 2, 24, 48000, 2000, 9, False, ipcm=True, enabled=False)],
                     used={'ipcm'}, chpl=[0, 5000000]))
    out.append(_case('mp4_flac', [flac_trak(10)], used={'flac'}))
    out.append(_case('mp4_aac', [aac_trak(11), alac_trak(_alac('mono16'), enabled=False)], used={'aac'},
                     suffix='.m4a'))
    for c in out:
        if c.name == 'mov_master':
            c.chapters = [0.0, 1.5, 4.0, 9.0]
        elif c.name == 'mp4_ipcm':
            c.chapters = [0.0, 0.5]
    return out


def refused_cases():
    """(case, regex): files opened, whose audio track is refused; files refused when opened."""
    a = _alac('mono16')
    out = []
    out.append((_case('edit_shift', [alac_trak(a, edits='shift')]), r'track 0 has an edit list'))
    out.append((_case('edit_two', [alac_trak(a, edits='two')]), r'track 0 has an edit list'))
    out.append((_case('aac_only', [aac_trak(12)]), r'Audio track 0 is aac'))
    out.append((_case('external', [alac_trak(a, edits='external')]), r'media in another file'))
    two = alac_trak(a)
    two.entry = two.entry + two.entry
    out.append((_case('two_entries', [two]), r'2 sample descriptions|sample descriptions'))
    out.append((_case('fragmented', [alac_trak(a)], extra_moov=box(b'mvex', full(b'trex', 0, 0, bytes(20)))),
                r'fragmented'))
    out.append((_case('edit_rate', [alac_trak(a, edits='rate')]), r'track 0 has an edit list'))
    for fourcc, bits, codec in ((b'sowt', 32, 'pcm_s32le'), (b'twos', 32, 'pcm_s32be'), (b'twos', 8, 'pcm_s8')):
        pcm = pcm_trak(fourcc, 2, bits, 48000, 1000, 14, fourcc == b'twos')
        pcm.pcm, pcm.codec = None, codec
        out.append((_case('%s%d' % (fourcc.decode(), bits), [pcm], suffix='.mov'), r'Audio track 0 is %s' % codec))
    out.append((_case('cmov', [alac_trak(a)], extra_moov=box(b'cmov', bytes(8))), r'compressed movie header'))
    return out


def damaged_cases():
    """(case, regex naming the box and byte offset)"""
    base = _case('dmg', [alac_trak(_alac('mono16'), per_chunk=(2,))])
    data = base.data
    out = []

    def at(tag):
        return data.index(tag) - 4

    def patched(name, pos, value, regex):
        d = bytearray(data)
        d[pos:pos + len(value)] = value
        out.append((Mp4Case(name, bytes(d), base.traks, base.expect, [], set()), regex))

    trak = at(b'trak')
    patched('trak_past_parent', trak, struct.pack('>I', len(data)), r"box 'trak' at byte offset %d runs past its parent"
            % trak)
    stco = at(b'stco')
    patched('stco_count', stco + 12, struct.pack('>I', 1000), r'stco box at byte offset %d: 1000 entries' % stco)
    stsc = at(b'stsc')
    patched('stsc_past_stco', stsc + 16, struct.pack('>I', 9), r'stsc box at byte offset %d names chunks past' % stsc)
    stsz = at(b'stsz')
    patched('stsz_count', stsz + 16, struct.pack('>I', 5), r'stsz box at byte offset %d lists 5 samples' % stsz)
    d = bytearray(data)
    co = stco + 16
    struct.pack_into('>I', d, co + 4, len(data) + 100)
    out.append((Mp4Case('sample_past_end', bytes(d), base.traks, base.expect, [], set()),
                r'sample 2 at byte offset %d lies past the end' % (len(data) + 100)))
    return out


def cut_cases():
    """(case, cut length): copies cut inside mdat after a whole moov (moov first)"""
    out = []
    for c in good_cases():
        if c.name == 'm4a_alac':
            out.append((c, len(c.data) - len(c.traks[0].samples[-1]) // 2))
        if c.name == 'mov_master':
            out.append((c, len(c.data) - 1234))
        if c.name == 'mp4_flac':
            out.append((c, len(c.data) - 700))
    return out


def sparse_file(path, case=None):
    """An ALAC .m4a whose mdat lies past 4 GiB behind a sparse `free` box (offsets need co64); returns the case."""
    case = case or _alac('d24')
    t = alac_trak(case, offsets='co64', edits=None)
    gap = (1 << 32) + 4096
    head, moov, mdat = build('sparse', [t], ftyp=b'M4A ', mdat_gap=gap)
    with open(path, 'wb') as f:
        f.write(head + moov)
        f.write(struct.pack('>I4sQ', 1, b'free', gap))
        f.seek(gap - 16, os.SEEK_CUR)
        f.write(mdat)
    return case


def assert_coverage(cases):
    used = set().union(*[c.used for c in cases])
    need = {'moov_first', 'moov_last', 'no_ftyp', 'iso', 'v0', 'v1', 'v2', 'wave', 'ipcm', 'enda', 'stz2', 'co64',
            'multi_stsc', 'stco', 'chpl', 'chap_track', 'video', 'mov_text', 'two_audio_enabled', 'identity_edit',
            'flac', 'aac', 'sowt24', 'twos24', 'text_subtitle', 'tx3g_chapter'}
    assert not need - used, sorted(need - used)
