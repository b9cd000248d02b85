"""A seeded NumPy Matroska writer and the Matroska files the tests read.

Each case is a file as bytes, written element by element, plus what it holds: per track the frames (after content
encodings) with their timestamps and the file offset of the block holding each, the chapter starts FFmpeg keeps, and
for audio tracks the PCM.  FLAC frames and PCM come from tests/flac_cases.py's encoder.  Shared by the CPU tests
(tests/test_mkv_cases.py against the libavformat demuxer of tests/ref_mkv.py, tests/test_kernel_emulation_mkv_flac.py,
tests/test_matroska_cli.py) and the GPU test of the loader (tests/test_gpu_matroska.py).

The set spans (assert_coverage checks it): no lacing, Xiph, EBML (negative deltas) and fixed lacing; SimpleBlock and
BlockGroup; negative relative timestamps; a non-default TimestampScale; known- and unknown-size Segment and Cluster;
Void and CRC-32 elements; SeekHead, Cues, Tags and Attachments; two and three audio tracks with FlagDefault absent, 0
and 1; header stripping and zlib; FLAC at 16 and 24 bits, 1, 2 and 6 channels, fixed and variable blocking; a cut FLAC
track; A_PCM/INT/LIT at 16 and 24 bits; ASS, SSA and UTF-8 subtitles with events out of time order; two chapter
editions with nested, hidden, UID-0 and backward atoms; a video track with B-frame timestamps; refused tracks (AAC,
big-endian PCM, encryption, bzlib) and damaged files (a lace table past its block, an element past its parent, a
file cut inside a block, FLAC frames with a bad CRC-8 and a bad CRC-16)."""
import functools
import os
import struct
import zlib

import numpy as np

from sushi_b200.wavstream import FlacFile
from tests import flac_cases as fc

SEED = 20261017
NS = 1000000000


# ---- EBML -----------------------------------------------------------------------------------------------------------
class Blob(object):
    """Bytes with named marks at offsets into them (where a block starts, for the expected tables)."""

    def __init__(self, data=b'', marks=()):
        self.data, self.marks = bytes(data), list(marks)


def cat(parts):
    data, marks, at = [], [], 0
    for p in parts:
        if isinstance(p, (bytes, bytearray)):
            p = Blob(p)
        data.append(p.data)
        marks += [(k, at + o) for k, o in p.marks]
        at += len(p.data)
    return Blob(b''.join(data), marks)


def id_bytes(i):
    return i.to_bytes((i.bit_length() + 7) // 8, 'big')


def size_bytes(n, length=None):
    length = length or next(k for k in range(1, 9) if n < (1 << (7 * k)) - 1)
    return ((1 << (7 * length)) | n).to_bytes(length, 'big')


UNKNOWN = b'\x01\xff\xff\xff\xff\xff\xff\xff'


def el(i, *kids, unknown=False, mark=None, size=None):
    body = cat(kids)
    head = id_bytes(i) + (UNKNOWN if unknown else size_bytes(len(body.data) if size is None else size))
    marks = [(k, len(head) + o) for k, o in body.marks] + ([(mark, 0)] if mark is not None else [])
    return Blob(head + body.data, marks)


def uint(i, v):
    return el(i, int(v).to_bytes(max(1, (int(v).bit_length() + 7) // 8), 'big'))


def text(i, s):
    return el(i, s.encode('utf-8'))


def flt(i, v):
    return el(i, struct.pack('>d', v))


def void(n):
    return el(0xEC, b'\0' * n)


def with_crc(i, *kids, **kw):
    """A master element whose first child is a CRC-32 of the rest (little-endian, as the specification has it)."""
    body = cat(kids)
    return el(i, el(0xBF, struct.pack('<I', zlib.crc32(body.data) & 0xFFFFFFFF)), body, **kw)


def signed_vint(d):
    for k in range(1, 9):
        bias = (1 << (7 * k - 1)) - 1
        if -bias <= d <= bias:
            return size_bytes(d + bias, k)
    raise ValueError(d)


def block_body(number, rel, frames, lacing, keyframe=True, simple=True):
    flags = (0x80 if keyframe and simple else 0) | {'none': 0, 'xiph': 2, 'fixed': 4, 'ebml': 6}[lacing]
    out = size_bytes(number) + struct.pack('>hB', rel, flags)
    if lacing == 'none':
        assert len(frames) == 1
        return out + frames[0]
    out += bytes([len(frames) - 1])
    if lacing == 'xiph':
        for f in frames[:-1]:
            out += b'\xff' * (len(f) // 255) + bytes([len(f) % 255])
    elif lacing == 'ebml':
        out += size_bytes(len(frames[0]))
        for a, b in zip(frames[:-2], frames[1:-1]):
            out += signed_vint(len(b) - len(a))
    else:
        assert len({len(f) for f in frames}) == 1
    return out + b''.join(frames)


# ---- tracks and files -----------------------------------------------------------------------------------------------
class TrackSpec(object):
    """A track to write: `frames` are (bytes as the track holds them, time in ticks, duration in ticks or None)."""

    def __init__(self, kind, codec, private=b'', default=None, name='', language=None, default_duration=0, rate=None,
                 channels=None, bits=None, encodings=(), pcm=None, pcm_bits=16):
        self.kind, self.codec, self.private, self.default = kind, codec, private, default
        self.name, self.language, self.default_duration = name, language, default_duration
        self.rate, self.channels, self.bits = rate, channels, bits
        self.encodings = list(encodings)      # ('strip', settings) | ('zlib',) | ('bzlib',) | ('encrypt',)
        self.frames = []
        self.pcm, self.pcm_bits = pcm, pcm_bits

    def stored(self, frame):
        for e in self.encodings:
            if e[0] == 'strip':
                assert frame.startswith(e[1])
                frame = frame[len(e[1]):]
            elif e[0] in ('zlib', 'bzlib', 'encrypt'):
                frame = zlib.compress(frame)
        return frame

    def entry(self, number):
        kids = [uint(0xD7, number), uint(0x73C5, number * 1000 + 7),
                uint(0x83, {'video': 1, 'audio': 2, 'subtitles': 17, 'buttons': 18}[self.kind])]
        if self.codec:
            kids.append(text(0x86, self.codec))
        if self.default is not None:
            kids.append(uint(0x88, 1 if self.default else 0))
        if self.name:
            kids.append(text(0x536E, self.name))
        if self.language:
            kids.append(text(0x22B59C, self.language))
        if self.default_duration:
            kids.append(uint(0x23E383, self.default_duration))
        private = self.private
        encs = []
        for order, e in enumerate(reversed(self.encodings)):
            if e[0] == 'strip':
                comp = el(0x5034, uint(0x4254, 3), el(0x4255, e[1]))
                encs.append(el(0x6240, uint(0x5031, order), uint(0x5032, 1), uint(0x5033, 0), comp))
            elif e[0] in ('zlib', 'bzlib'):
                scope = 3 if private and e[0] == 'zlib' else 1
                if scope & 2:
                    private = zlib.compress(private)
                encs.append(el(0x6240, uint(0x5031, order), uint(0x5032, scope), uint(0x5033, 0),
                               el(0x5034, uint(0x4254, 0 if e[0] == 'zlib' else 1))))
            else:
                encs.append(el(0x6240, uint(0x5031, order), uint(0x5032, 1), uint(0x5033, 1),
                               el(0x5035, uint(0x47E1, 5))))
        if encs:
            kids.append(el(0x6D80, *encs))
        if private:
            kids.append(el(0x63A2, private))
        if self.kind == 'audio':
            a = [flt(0xB5, float(self.rate)), uint(0x9F, self.channels)]
            if self.bits:
                a.append(uint(0x6264, self.bits))
            kids.append(el(0xE1, *a))
        if self.kind == 'video':
            kids.append(el(0xE0, uint(0xB0, 64), uint(0xBA, 36)))
        return el(0xAE, *kids)


class MkvCase(object):
    """A Matroska file (bytes) and what it holds.  `expect[stream id]` = list of (frame bytes, time in ns, file offset
    of its block); `chapters` = the chapter starts in ns FFmpeg keeps; `damage` = None or (kind, byte offset, regex)."""

    def __init__(self, name, data, specs, expect, chapters, scale, damage=None, refused=None, script=None):
        self.name, self.data, self.specs, self.expect = name, data, specs, expect
        self.chapters, self.scale, self.damage, self.refused, self.script = chapters, scale, damage, refused, script

    def write(self, directory, suffix='.mkv'):
        path = os.path.join(str(directory), self.name + suffix)
        with open(path, 'wb') as f:
            f.write(self.data)
        return path

    def audio_ids(self):
        return [i for i, s in enumerate(self.specs) if s.kind == 'audio' and s.pcm is not None]

    def wav(self, sid):
        """The plain PCM WAV of audio track `sid`'s samples."""
        s = self.specs[sid]
        case = fc.FlacCase('x', b'', s.pcm, s.rate, s.pcm_bits, [], [], 12000, 'uint8')
        return case.wav()

    def write_wav(self, directory, sid):
        path = os.path.join(str(directory), '%s_%d.wav' % (self.name, sid))
        with open(path, 'wb') as f:
            f.write(self.wav(sid))
        return path

    def __repr__(self):
        return 'MkvCase(%s)' % self.name


def atom(uid, start, hidden=False, nested=()):
    kids = ([uint(0x73C4, uid)] if uid is not None else []) + [uint(0x91, start)]
    if hidden:
        kids.append(uint(0x98, 1))
    kids.append(el(0x80, text(0x85, 'chapter %d' % start)))
    return el(0xB6, *(kids + list(nested)))


def chapters_element(editions):
    """editions: list of lists of (uid, start ns, hidden, nested atoms)."""
    return el(0x1043A770, *[el(0x45B9, uint(0x45BC, k + 1), *[atom(*a) for a in ed]) for k, ed in enumerate(editions)])


def ffmpeg_chapters(editions):
    out, max_start = [], 0
    for ed in editions:
        for a in ed:
            uid, start = a[0], a[1]
            if uid and (max_start == 0 or start > max_start):
                out.append(start)
                max_start = start
    return out


def build(name, specs, blocks, clusters, scale=1000000, editions=(), segment_unknown=False, cluster_unknown=(),
          extras=True, crc=False, damage=None, refused=None, script=None):
    """blocks: per cluster a list of dict(track (0-based spec index), rel, frames (indices into the spec's frames),
    lacing, group, duration).  clusters: the clusters' timestamps in ticks."""
    header = el(0x1A45DFA3, uint(0x4286, 1), uint(0x42F7, 1), uint(0x42F2, 4), uint(0x42F3, 8),
                text(0x4282, 'matroska'), uint(0x4287, 4), uint(0x4285, 2))
    info = [uint(0x2AD7B1, scale), text(0x4D80, 'mkv_cases'), text(0x5741, 'mkv_cases'), flt(0x4489, 1000.0)]
    info = with_crc(0x1549A966, *info) if crc else el(0x1549A966, *info)
    tracks = el(0x1654AE6B, *[s.entry(k + 1) for k, s in enumerate(specs)])
    top = []
    if extras:
        top.append(el(0x114D9B74, el(0x4DBB, el(0x53AB, id_bytes(0x1549A966)), uint(0x53AC, 1234))))
        top.append(void(37))
    top += [info, tracks]
    if editions:
        top.append(chapters_element(editions))
    if extras:
        font = np.random.default_rng([SEED, 5]).integers(0, 256, 3000, dtype=np.uint8).tobytes()
        top.append(el(0x1941A469, el(0x61A7, text(0x466E, 'font.ttf'), text(0x4660, 'font/ttf'),
                                      el(0x465C, font), uint(0x46AE, 99))))
        top.append(el(0x1254C367, el(0x7373, el(0x63C0, uint(0x68CA, 50)), el(0x67C8, text(0x45A3, 'TITLE'),
                                                                             text(0x4487, 'mkv_cases')))))
    expect = {k: [] for k in range(len(specs))}
    for c, (ts, cblocks) in enumerate(zip(clusters, blocks)):
        kids = [uint(0xE7, ts)]
        if extras and c == 0:
            kids.append(void(5))
        for j, b in enumerate(cblocks):
            spec = specs[b['track']]
            frames = [spec.frames[i][0] for i in b['frames']]
            body = block_body(b['track'] + 1, b['rel'], [spec.stored(f) for f in frames], b['lacing'],
                              simple=not b.get('group'))
            key = (c, j)
            if b.get('group'):
                g = [el(0xA1, body, mark=key)]
                if b.get('duration') is not None:
                    g.append(uint(0x9B, b['duration']))
                kids.append(el(0xA0, *g))
            else:
                kids.append(el(0xA3, body, mark=key))
            laces = len(b['frames'])
            block_dur = b['duration'] if b.get('group') and b.get('duration') is not None else \
                spec.default_duration * laces // scale
            for k, i in enumerate(b['frames']):
                expect[b['track']].append((spec.frames[i][0], key, (ts + b['rel'] + k * (block_dur // laces)) * scale))
        if crc:
            top.append(with_crc(0x1F43B675, *kids, unknown=c in cluster_unknown, mark=('cluster', c)))
        else:
            top.append(el(0x1F43B675, *kids, unknown=c in cluster_unknown, mark=('cluster', c)))
    if extras:
        top.append(el(0x1C53BB6B, el(0xBB, uint(0xB3, 0), el(0xB7, uint(0xF7, 1), uint(0xF1, 100)))))
    segment = el(0x18538067, *top, unknown=segment_unknown)
    data = cat([header, segment])
    where = dict(data.marks)
    # FFmpeg's streams: TrackEntries of a type it handles with a CodecID, in order; the case lists those only
    streams = [k for k, s in enumerate(specs) if s.kind in ('video', 'audio', 'subtitles') and s.codec]
    exp = {sid: [(f, t, where[key]) for f, key, t in expect[k]] for sid, k in enumerate(streams)}
    case = MkvCase(name, data.data, [specs[k] for k in streams], exp, ffmpeg_chapters(editions), scale, damage,
                   refused, script)
    case.clusters = [where[('cluster', c)] for c in range(len(clusters))]
    return case


# ---- track contents -------------------------------------------------------------------------------------------------
def flac_track(frames_count, channels, bits, rate, block, seed, variable=False, cut=0, default=None, name='',
               language='jpn', encodings=(), lpc=True, kinds=('lpc', 'fixed'), assignments=(10, 0, 8, 9)):
    """A FLAC track: fc.encode's frames (CodecPrivate = its marker and metadata).  cut > 0 drops the first `cut`
    frames, leaving STREAMINFO's total as it was (stale) and frame numbers starting at `cut`.  DefaultDuration is the
    block's duration to the millisecond."""
    rng = np.random.default_rng([SEED, seed])
    pcm = fc.make_pcm('programme', frames_count, channels, bits, rate, rng)
    if variable:
        sizes = [int(v) for v in rng.integers(block // 2, block * 2, frames_count // block + 2)]
        blocks, left = [], frames_count
        for s in sizes:
            if left <= 0:
                break
            blocks.append(min(s, left))
            left -= blocks[-1]
        if left:
            blocks.append(left)
    else:
        blocks = fc.fixed_blocks(frames_count, block)
    plan = fc.uniform_plan(channels, kind='auto', order=8) if lpc else fc.uniform_plan(channels, kind='fixed', order=2)
    if channels == 2:
        plan = fc.stereo_plan(list(kinds), assignments=assignments, order=8, porder=3)
    data, _, offsets = fc.encode(pcm, rate, bits, blocks, plan, rng, variable=variable)
    offsets = [int(o) for o in offsets]
    spec = TrackSpec('audio', 'A_FLAC', data[:offsets[0]], default, name, language,
                     int(round(block * 1000.0 / rate)) * 1000000, rate, channels, bits, encodings,
                     pcm=pcm[sum(blocks[:cut]):], pcm_bits=bits)
    t = sum(blocks[:cut])
    for k in range(cut, len(blocks)):
        spec.frames.append((data[offsets[k]:offsets[k + 1]], None, None))
        spec.frames[-1] = (spec.frames[-1][0], t, blocks[k])
        t += blocks[k]
    return spec


def pcm_track(frames_count, channels, bits, rate, per_frame, seed, default=None, name='', codec='A_PCM/INT/LIT'):
    rng = np.random.default_rng([SEED, seed])
    pcm = fc.make_pcm('programme', frames_count, channels, bits, rate, rng)
    case = fc.FlacCase('x', b'', pcm, rate, bits, [], [], 12000, 'uint8')
    payload = case.wav()[44:]
    assert per_frame * NS % rate == 0
    spec = TrackSpec('audio', codec, b'', default, name, 'eng', per_frame * NS // rate, rate, channels, bits, pcm=pcm,
                     pcm_bits=bits)
    step = per_frame * channels * bits // 8
    for k, a in enumerate(range(0, len(payload), step)):
        spec.frames.append((payload[a:a + step], k * per_frame, per_frame))
    return spec


def ass_script(seed, n=12, ssa=False):
    """(header lines, [(read order, start cs, end cs, block payload)]) of an ASS / SSA script: the header lines are
    the CodecPrivate, the payloads are what the blocks hold (ReadOrder, Layer, Style, ..., Text)."""
    rng = np.random.default_rng([SEED, seed])
    head = ['[Script Info]', 'Title: mkv_cases', 'ScriptType: %s' % ('v4.00' if ssa else 'v4.00+'), '',
            '[V4+ Styles]' if not ssa else '[V4 Styles]',
            'Format: Name, Fontname, Fontsize, PrimaryColour, SecondaryColour, OutlineColour, BackColour, Bold, Italic, '
            'Underline, StrikeOut, ScaleX, ScaleY, Spacing, Angle, BorderStyle, Outline, Shadow, Alignment, MarginL, '
            'MarginR, MarginV, Encoding',
            'Style: Default,Arial,20,&H00FFFFFF,&H000000FF,&H00000000,&H00000000,0,0,0,0,100,100,0,0,1,2,2,2,10,10,10,1',
            '', '[Events]', 'Format: Layer, Start, End, Style, Name, MarginL, MarginR, MarginV, Effect, Text']
    events = []
    for k in range(n):
        start = int(rng.integers(100, 6000))
        end = start + int(rng.integers(50, 400))
        txt = 'line %d, with a comma{\\i1}and tags{\\i0}' % k
        events.append((k, start, end, '%d,%d,Default,spk%d,0,0,%d,,%s' % (k, k % 3, k, k % 2 * 5, txt)))
    return head, events


# ---- the cases ------------------------------------------------------------------------------------------------------
def video_track(count, seed, size=20000, scale=1000000):
    """B-frame pattern in decode order (I P B B ...), 23.976 fps, random payloads of `size` bytes."""
    rng = np.random.default_rng([SEED, seed])
    spec = TrackSpec('video', 'V_VP9', default=True, language='und')
    order = []
    for g in range(0, count, 3):
        order += [g, g + 2, g + 1] if g + 2 < count else list(range(g, count))
    for n in order:
        t = int(round(n * 1001 / 24000 * NS / scale))
        spec.frames.append((rng.integers(0, 256, size, dtype=np.uint8).tobytes(), t, None))
    return spec


def sub_track(codec, events, private=b'', encodings=(('zlib',),), default=None, name=''):
    spec = TrackSpec('subtitles', codec, private, default, name, 'eng', encodings=encodings)
    for e in events:
        spec.frames.append(e)
    return spec


def _blocks_for(spec_index, spec, layout):
    """Frames of one track into per-cluster block lists.  layout(k) -> (lacing, frames per block, group, duration)."""
    out = []
    k = 0
    j = 0
    while k < len(spec.frames):
        lacing, per, group, dur = layout(j)
        idx = list(range(k, min(k + per, len(spec.frames))))
        if lacing == 'none' or len(idx) == 1:
            lacing, idx = 'none', idx[:1]
        if lacing == 'fixed' and len({len(spec.frames[i][0]) for i in idx}) != 1:
            lacing, idx = 'none', idx[:1]
        out.append(dict(track=spec_index, frames=idx, lacing=lacing, group=group, duration=dur,
                        time=spec.frames[idx[0]][1]))
        k = idx[-1] + 1
        j += 1
    return out


def arrange(specs, per_cluster_ticks, track_blocks, negative=0):
    """Sort every block into clusters of `per_cluster_ticks` by its time (decode order kept per track).  With
    negative > 0, each cluster's timestamp is pushed `negative` ticks past its first block, so early blocks carry
    negative relative timestamps."""
    allb = [b for blist in track_blocks for b in blist]
    last = max(b['time'] for b in allb)
    n = int(last // per_cluster_ticks) + 1
    clusters = [[] for _ in range(n)]
    for b in allb:
        clusters[int(max(b['time'], 0) // per_cluster_ticks)].append(b)
    ts = []
    for c, blist in enumerate(clusters):
        base = c * per_cluster_ticks + (negative if blist and negative else 0)
        ts.append(base)
        for b in blist:
            b['rel'] = b['time'] - base
            assert -32768 <= b['rel'] < 32768
    keep = [(t, bl) for t, bl in zip(ts, clusters) if bl]
    return [t for t, _ in keep], [bl for _, bl in keep]


def _timed(spec, ticks_per_sample):
    """Set each FLAC / PCM frame's time (in samples) to ticks."""
    spec.frames = [(f, int(round(t * ticks_per_sample)), d) for f, t, d in spec.frames]
    return spec


def case_main():
    """Stereo 16-bit FLAC with every lacing, SimpleBlock and BlockGroup, negative relative timestamps; B-frame
    video; an ASS track (zlib, events out of time order); two chapter editions; every top-level extra; CRC-32."""
    scale = 1000000
    a = _timed(flac_track(4096 * 24 + 700, 2, 16, 48000, 1024, 1, default=True, name='main'), 1000.0 / 48000)
    head, events = ass_script(2)
    s = sub_track('S_TEXT/ASS', [(e[3].encode(), e[1] * 10, (e[2] - e[1]) * 10) for e in events],
                  ('\n'.join(head) + '\n').encode())
    v = video_track(60, 3)
    specs = [v, a, s]
    lac = ['none', 'xiph', 'ebml', 'none', 'xiph', 'ebml']
    ab = _blocks_for(1, a, lambda j: (lac[j % 6], 1 + j % 4, j % 5 == 3, None))
    vb = _blocks_for(0, v, lambda j: ('none', 1, False, None))
    sb = _blocks_for(2, s, lambda j: ('none', 1, True, s.frames[j][2]))
    ts, clusters = arrange(specs, 1000, [vb, ab, sb], negative=300)
    editions = [[(11, 0, False, ()), (12, 5 * NS, True, (atom(99, 6 * NS),)), (0, 7 * NS, False, ()),
                 (13, 3 * NS, False, ()), (14, 9 * NS + 123456789, False, ())],
                [(21, 2 * NS, False, ()), (22, 10 * NS + 500, False, ())]]
    return build('main', specs, clusters, ts, scale, editions, crc=True, script=(head, events))


def case_unknown_sizes():
    """24-bit 6-channel FLAC, variable blocking, header stripping; SSA track; unknown-size segment and clusters; a
    TimestampScale of 100 us."""
    scale = 100000
    a = _timed(flac_track(2048 * 14 + 33, 6, 24, 44100, 2048, 4, variable=True, encodings=[('strip', b'\xff\xf9')]),
               10000.0 / 44100)
    head, events = ass_script(5, ssa=True)
    s = sub_track('S_TEXT/SSA', [(e[3].encode(), e[1] * 100, (e[2] - e[1]) * 100) for e in events],
                  ('\n'.join(head) + '\n').encode(), encodings=())
    specs = [a, s]
    ab = _blocks_for(0, a, lambda j: (('ebml', 'none', 'xiph')[j % 3], 2 + j % 2, j % 4 == 1, None))
    sb = _blocks_for(1, s, lambda j: ('none', 1, True, s.frames[j][2]))
    ts, clusters = arrange(specs, 20000, [ab, sb])
    return build('unknown_sizes', specs, clusters, ts, scale, segment_unknown=True,
                 cluster_unknown=set(range(0, len(ts), 2)), script=(head, events))


def case_cut():
    """A mono 16-bit FLAC track cut from a longer stream: frame numbers start at 5, the STREAMINFO total is stale."""
    a = _timed(flac_track(1152 * 20 + 99, 1, 16, 48000, 1152, 6, cut=5, lpc=False), 1000.0 / 48000)
    a.frames = [(f, t - a.frames[0][1], d) for f, t, d in a.frames]
    ab = _blocks_for(0, a, lambda j: ('xiph', 3, False, None))
    ts, clusters = arrange([a], 5000, [ab])
    return build('cut', [a], clusters, ts, extras=False)


def case_multi():
    """Three audio tracks: FLAC with FlagDefault absent, PCM 16-bit with 0 (fixed lacing), PCM 24-bit with 1; a UTF-8
    track (zlib)."""
    a = _timed(flac_track(4096 * 6 + 5, 2, 16, 48000, 4096, 7, name='flac', language='jpn'), 1000.0 / 48000)
    p16 = _timed(pcm_track(48000 * 2 + 17, 2, 16, 48000, 1440, 8, default=False, name='pcm16'), 1000.0 / 48000)
    p24 = _timed(pcm_track(44100 * 2 + 3, 1, 24, 44100, 1323, 9, default=True, name='pcm24'), 1000.0 / 44100)
    srt = [('line %d\nsecond row, %d' % (k, k)).encode() for k in range(8)]
    rng = np.random.default_rng([SEED, 10])
    times = sorted(int(t) for t in rng.integers(0, 2500, 8))
    s = sub_track('S_TEXT/UTF8', [(b, t, 300 + 7 * k) for k, (b, t) in enumerate(zip(srt, times))])
    specs = [a, p16, p24, s]
    ab = _blocks_for(0, a, lambda j: ('none', 1, False, None))
    pb = _blocks_for(1, p16, lambda j: ('fixed', 3, False, None))
    qb = _blocks_for(2, p24, lambda j: ('fixed', 2, j % 2 == 1, None))
    sb = _blocks_for(3, s, lambda j: ('none', 1, True, s.frames[j][2]))
    ts, clusters = arrange(specs, 700, [ab, pb, qb, sb])
    return build('multi', specs, clusters, ts, script=srt)


def case_two_no_default():
    a = _timed(pcm_track(8000, 1, 16, 8000, 800, 11, default=False), 1000.0 / 8000)
    b = _timed(pcm_track(8000, 1, 16, 8000, 800, 12, default=False), 1000.0 / 8000)
    ts, clusters = arrange([a, b], 10000, [_blocks_for(0, a, lambda j: ('none', 1, False, None)),
                                           _blocks_for(1, b, lambda j: ('none', 1, False, None))])
    return build('two_no_default', [a, b], clusters, ts, extras=False)


def case_skipped_tracks():
    """A buttons track (TrackType 18) and an audio TrackEntry without a CodecID, each with blocks, before a PCM track:
    FFmpeg gives neither a stream, so the PCM track is stream 0."""
    b = TrackSpec('buttons', 'B_VOBBTN')
    b.frames = [(bytes(range(40)), 0, None), (bytes(range(50)), 500, None)]
    n = _timed(pcm_track(4000, 1, 16, 8000, 800, 15), 1000.0 / 8000)
    n.codec = ''
    a = _timed(pcm_track(8000, 2, 16, 8000, 800, 16, default=True), 1000.0 / 8000)
    specs = [b, n, a]
    ts, clusters = arrange(specs, 10000, [_blocks_for(k, s, lambda j: ('none', 1, False, None))
                                          for k, s in enumerate(specs)])
    return build('skipped_tracks', specs, clusters, ts, extras=False)


def refused_cases():
    """Files whose audio track cannot be decoded: (case, regex of the refusal)."""
    out = []
    base = lambda: _timed(pcm_track(8000, 1, 16, 8000, 800, 13, default=True), 1000.0 / 8000)
    for name, change, regex in (
            ('aac', lambda t: setattr(t, 'codec', 'A_AAC'), r'Audio track 0 is A_AAC'),
            ('pcm_big', lambda t: setattr(t, 'codec', 'A_PCM/INT/BIG'), r'Audio track 0 is A_PCM/INT/BIG at 16 bits'),
            ('encrypted', lambda t: t.encodings.append(('encrypt',)), r'track 0 is encrypted'),
            ('bzlib', lambda t: t.encodings.append(('bzlib',)), r'track 0 is compressed with bzlib')):
        t = base()
        change(t)
        ts, clusters = arrange([t], 10000, [_blocks_for(0, t, lambda j: ('none', 1, False, None))])
        out.append(build('refused_' + name, [t], clusters, ts, extras=False, refused=regex))
    return out


def damaged_cases():
    """(the undamaged base, [damaged copies]): files the reader or the decoder must refuse, each with the byte offset
    of the block the message names."""
    out = []
    a = _timed(flac_track(1024 * 24, 2, 16, 48000, 1024, 14, kinds=('verbatim', 'fixed'), assignments=(0,)),
               1000.0 / 48000)
    ts, clusters = arrange([a], 100, [_blocks_for(0, a, lambda j: ('xiph', 2, False, None))])
    good = build('damage_base', [a], clusters, ts, extras=False)
    data = good.data
    offs = sorted({e[2] for e in good.expect[0]})

    def block_at(k):
        """(element offset, header length, body length) of the k-th block."""
        pos = offs[k]
        hl = 1 + (9 - data[pos + 1].bit_length())
        return pos, hl, int.from_bytes(data[pos + 1:pos + hl], 'big') & ((1 << (7 * (hl - 1))) - 1)

    def copy(kind, d, pos, regex, expect=None):
        out.append(MkvCase('damage_' + kind, bytes(d), good.specs, expect or good.expect, [], good.scale,
                           damage=(kind, pos, regex)))

    # block 3's Xiph lace size never ends: 255s up to the end of the block
    pos, hl, n = block_at(3)
    lace = pos + hl + 4 + 1                           # track, timestamp, flags, lace count
    d = bytearray(data)
    d[lace:pos + hl + n] = b'\xff' * (pos + hl + n - lace)
    copy('lace', d, pos, r'lace table of the block at byte %d runs past its block' % pos)
    # the last block of the first cluster runs one byte past its cluster (not past the file)
    second = good.clusters[1]
    k = max(i for i, o in enumerate(offs) if o < second)
    pos, hl, n = block_at(k)
    assert pos + hl + n == second and hl == 3
    d = bytearray(data)
    d[pos + 1:pos + 3] = size_bytes(n + 1, 2)
    copy('parent', d, pos, r'element at byte %d runs past its parent' % pos)
    # the file cut inside block 7: blocks 0 to 6 load
    pos, hl, n = block_at(7)
    copy('truncated', data[:pos + hl + n // 2], pos, None, {0: [e for e in good.expect[0] if e[2] < pos]})
    # the first frame of block 4 with a bad CRC-8 (its header's last byte), of block 6 with a bad CRC-16 (a bit of
    # its VERBATIM samples)
    for kind, blk, regex in (('crc8', 4, 'frame header CRC-8 mismatch'), ('crc16', 6, 'frame CRC-16 mismatch')):
        pos, hl, n = block_at(blk)
        idx = [i for i, e in enumerate(good.expect[0]) if e[2] == pos]
        first = good.expect[0][idx[0]][0]
        at = pos + hl + n - sum(len(good.expect[0][i][0]) for i in idx)
        assert data[at:at + len(first)] == first
        d = bytearray(data)
        d[at + (_flac_header_len(first) - 1 if kind == 'crc8' else 100)] ^= 0x10
        copy(kind, d, pos, r'FLAC frame %d at byte offset %d: %s' % (idx[0], pos, regex))
    # an unknown-size Segment (as a muxer writing to a pipe leaves it), cut inside a block of a known-size Cluster,
    # inside a block of an unknown-size Cluster, and inside the Cues after the last Cluster
    u = build('damage_base_unknown', [a], clusters, ts, segment_unknown=True, cluster_unknown={1, 3})
    uoffs = sorted({e[2] for e in u.expect[0]})
    for kind, cluster in (('truncated_unknown_segment', 2), ('truncated_unknown_cluster', 3)):
        assert cluster + 1 < len(u.clusters)
        pos = [o for o in uoffs if u.clusters[cluster] < o < u.clusters[cluster + 1]][1]
        out.append(MkvCase('damage_' + kind, u.data[:pos + 20], u.specs, {0: [e for e in u.expect[0] if e[2] < pos]},
                           [], u.scale, damage=(kind, pos, None)))
    # an empty FLAC frame: the second Xiph lace of a block has size 0
    e = _timed(flac_track(1024 * 8, 2, 16, 48000, 1024, 17), 1000.0 / 48000)
    e.frames.insert(3, (b'', e.frames[3][1], 0))
    ts, clusters = arrange([e], 100, [_blocks_for(0, e, lambda j: ('xiph', 2, False, None))])
    ec = build('damage_empty', [e], clusters, ts, extras=False)
    pos = ec.expect[0][3][2]
    assert ec.expect[0][3][0] == b'' and ec.expect[0][2][2] == pos
    ec.damage = ('empty', pos, r'FLAC frame 3 at byte offset %d: empty frame' % pos)
    out.append(ec)
    cues = u.data.rindex(id_bytes(0x1C53BB6B))
    out.append(MkvCase('damage_truncated_cues', u.data[:cues + 6], u.specs, u.expect, [], u.scale,
                       damage=('truncated_cues', cues, None)))
    return good, out


def _flac_header_len(frame):
    """Bytes of a FLAC frame header, its CRC-8 included (fixed block and rate codes, as flac_cases writes them)."""
    at = 4
    b = frame[at]
    extra = 0 if b < 0x80 else 1 if b < 0xE0 else 2 if b < 0xF0 else 3 if b < 0xF8 else 4
    at += 1 + extra
    bcode, rcode = frame[2] >> 4, frame[2] & 15
    at += 1 if bcode == 6 else 2 if bcode == 7 else 0
    at += 1 if rcode == 12 else 2 if rcode in (13, 14) else 0
    return at + 1


@functools.lru_cache(maxsize=None)
def audio_cases():
    cases = [case_main(), case_unknown_sizes(), case_cut(), case_multi(), case_two_no_default(), case_skipped_tracks()]
    return cases


@functools.lru_cache(maxsize=None)
def all_cases():
    """Every readable case (damaged and refused ones included, since their containers parse)."""
    good, damaged = damaged_cases()
    cases = list(audio_cases()) + refused_cases() + [good] + damaged
    assert len({c.name for c in cases}) == len(cases)
    assert_coverage(cases)
    return cases


def assert_coverage(cases):
    data = b''.join(c.data for c in cases)
    specs = [s for c in cases for s in c.specs]
    audio = [s for s in specs if s.kind == 'audio']
    assert {s.codec for s in audio} >= {'A_FLAC', 'A_PCM/INT/LIT', 'A_PCM/INT/BIG', 'A_AAC'}
    flac = [s for s in audio if s.codec == 'A_FLAC']
    assert {s.bits for s in flac} == {16, 24} and {s.channels for s in flac} >= {1, 2, 6}
    assert {s.bits for s in audio if s.codec == 'A_PCM/INT/LIT'} == {16, 24}
    assert {s.codec for s in specs if s.kind == 'subtitles'} == {'S_TEXT/ASS', 'S_TEXT/SSA', 'S_TEXT/UTF8'}
    encs = {e[0] for s in specs for e in s.encodings}
    assert encs >= {'strip', 'zlib', 'bzlib', 'encrypt'}
    multi = [c for c in cases if len([s for s in c.specs if s.kind == 'audio']) >= 3][0]
    assert {s.default for s in multi.specs if s.kind == 'audio'} == {None, False, True}
    assert b'\x1f\x43\xb6\x75' + UNKNOWN in data and b'\x18\x53\x80\x67' + UNKNOWN in data
    for i in (0x114D9B74, 0x1C53BB6B, 0x1254C367, 0x1941A469, 0xEC, 0xBF):
        assert id_bytes(i) in data
    assert {c.damage[0] for c in cases if c.damage} == {'lace', 'parent', 'truncated', 'truncated_unknown_segment',
                                                         'truncated_unknown_cluster', 'truncated_cues', 'crc8', 'crc16',
                                                         'empty'}
    assert any(c.scale != 1000000 for c in cases)


# ---- long files, written as a stream ------------------------------------------------------------------------------
def write_av(path, codec_private, frames, samples, rate, channels, bits, video_count, video_size, seed,
             cluster_ms=5000):
    """A remux-shaped file at `path`, written cluster by cluster: a FLAC track (frames[i] holds samples[i] samples per
    channel) and a video track of `video_count` frames at 23.976 fps, each `video_size` random bytes (from a pool of
    16).  TimestampScale 1 ms, unknown-size Segment, known-size Clusters of `cluster_ms`, SimpleBlocks without lacing.
    Returns (bytes written, video payload bytes)."""
    rng = np.random.default_rng([SEED, seed])
    pool = [rng.integers(0, 256, video_size, dtype=np.uint8).tobytes() for _ in range(16)]
    audio = TrackSpec('audio', 'A_FLAC', codec_private, True, '', 'jpn', 0, rate, channels, bits)
    video = TrackSpec('video', 'V_VP9', default=True, language='und')
    head = el(0x1A45DFA3, text(0x4282, 'matroska'), uint(0x4287, 4), uint(0x4285, 2)).data
    head += id_bytes(0x18538067) + UNKNOWN
    head += el(0x1549A966, uint(0x2AD7B1, 1000000)).data + el(0x1654AE6B, video.entry(1), audio.entry(2)).data
    a_ms = (np.concatenate([[0], np.cumsum(samples)[:-1]]) * 1000 // rate).astype(np.int64)
    v_ms = (np.arange(video_count, dtype=np.int64) * 1001) // 24
    last = max(int(a_ms[-1]) if len(a_ms) else 0, int(v_ms[-1]) if len(v_ms) else 0)
    ai = vi = 0
    total, vbytes = 0, 0
    with open(path, 'wb') as f:
        f.write(head)
        total += len(head)
        for c in range(last // cluster_ms + 1):
            end = (c + 1) * cluster_ms
            parts = [id_bytes(0xE7) + size_bytes(4) + (c * cluster_ms).to_bytes(4, 'big')]
            while (ai < len(a_ms) and a_ms[ai] < end) or (vi < len(v_ms) and v_ms[vi] < end):
                if vi >= len(v_ms) or (ai < len(a_ms) and a_ms[ai] <= v_ms[vi]):
                    number, rel, payload = 2, int(a_ms[ai]) - c * cluster_ms, frames[ai]
                    ai += 1
                else:
                    number, rel, payload = 1, int(v_ms[vi]) - c * cluster_ms, pool[vi % 16]
                    vbytes += len(payload)
                    vi += 1
                body_head = size_bytes(number) + struct.pack('>hB', rel, 0x80)
                parts += [id_bytes(0xA3) + size_bytes(len(body_head) + len(payload)) + body_head, payload]
            size = sum(len(p) for p in parts)
            f.write(id_bytes(0x1F43B675) + size_bytes(size, 8))
            for p in parts:
                f.write(p)
            total += 12 + size
    return total, vbytes


def flac_frames_of(data, first, block, rate, channels, bits, n_frames):
    """Frame slices of a VERBATIM-coded fc.periodic_file: every frame but the last is its header, one subframe header
    byte and `block` samples per channel, and the CRC-16; the last ends the file."""
    view = memoryview(data)
    frames, at = [], first
    body = channels * (1 + block * bits // 8) + 2
    for i in range(n_frames):
        n = len(fc.frame_header(i, block, rate, channels, 1, bits, {})[0]) + body
        frames.append(view[at:at + n])
        at += n
    frames.append(view[at:])
    return frames


def baseline_mkv(path, seed=8, video_count=129600, video_size=64):
    """The BASELINE-size file: 90 minutes of 48 kHz stereo 16-bit FLAC (63 281 VERBATIM frames of 4096 samples and a
    last one of 1024, about 1 GB) muxed with a 23.976 fps video track of `video_count` frames.
    Returns the PCM ((frames, 2) int16)."""
    rate, block, n_frames = 48000, 4096, 63281
    tail = 90 * 60 * rate - n_frames * block
    data, pcm = fc.periodic_file(n_frames, tail, 16, lambda j: None, seed, rate, block, period=256)
    first = FlacFile.from_bytes(data[:65536], path).frame_offset
    frames = flac_frames_of(data, first, block, rate, 2, 16, n_frames)
    write_av(path, data[:first], frames, [block] * n_frames + [tail], rate, 2, 16, video_count, video_size, seed)
    return pcm.astype(np.int16)


def pair_mkv(path, flac_case, script_head, events, chapters_ns, video_count, seed):
    """A small source or destination file for the command line: the FLAC of `flac_case` (one block per frame), an ASS
    track of `events` ((read order, start cs, end cs, block payload)) under `script_head`, the chapters (one edition)
    and a 23.976 fps video track.  Returns the case."""
    offs = [int(o) for o in flac_case.offsets]
    a = TrackSpec('audio', 'A_FLAC', flac_case.flac[:offs[0]], True, '', 'jpn', 0, flac_case.rate, flac_case.channels,
                  flac_case.bits)
    t = 0
    for k in range(len(offs) - 1):
        a.frames.append((flac_case.flac[offs[k]:offs[k + 1]], t * 1000 // flac_case.rate, None))
        t += flac_case.frames[k]['block_size']
    s = sub_track('S_TEXT/ASS', [(e[3].encode(), e[1] * 10, (e[2] - e[1]) * 10) for e in events],
                  ('\n'.join(script_head) + '\n').encode())
    v = video_track(video_count, seed, size=200)
    specs = [v, a, s]
    blocks = [_blocks_for(i, sp, lambda j: ('none', 1, sp.kind == 'subtitles', sp.frames[j][2])) for i, sp in
              enumerate(specs)]
    ts, clusters = arrange(specs, 10000, blocks)
    case = build(os.path.basename(path), specs, clusters, ts, editions=[[(k + 1, c, False, ()) for k, c in
                                                                         enumerate(chapters_ns)]])
    with open(path, 'wb') as f:
        f.write(case.data)
    return case
