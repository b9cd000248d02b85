"""Seeded WAV files at the edges where the loader can go wrong, with the oracle restatement of the reference loader as
their truth.

Pure NumPy, shared by the CPU test of the host mirror (tests/test_loader_cases.py) and the GPU test of the loader
kernels (tests/test_gpu_loader_cases.py).  A case is a RIFF file as bytes, written with `struct` so that header and
payload can disagree, plus the output sample rate and sample type to load it with.  The set is a fixed list of named
corners plus a seeded sample, and it spans:

* frame rates 8000, 11025, 22050, 12000 (no resample), 32000, 44100, 48000, 96000 and the odd 7919 and 12001, loaded at
  12000, 8000 and 24000 Hz;
* 1, 2, 3, 5, 6, 8 and 64 channels (64 is the GPU loader's limit: a 2048-wide fine histogram);
* 16-bit samples and 24-bit samples with random low bytes, which the decoder ignores;
* frame counts 0, 1, fr - 1, fr, fr + 1, fr + 2 at 48 kHz (Python 2's round half away: 0.5 -> 1), a last chunk that
  resamples to zero samples, last chunks that leave the one-sample gap where ceil(total * rate) exceeds the samples
  written, and lengths whose padded size covers every residue mod 8 (the tails of the vectorised kernels);
* value families aimed at the median selector (see FAMILIES);
* container shapes: a chunk after `data` (the reference's last one-second read runs into it), a `data` chunk cut short
  by the end of the file, the same with a partial frame at the end, an odd-sized chunk before `data`, and a 40-byte
  WAVE_FORMAT_EXTENSIBLE fmt chunk.

Two inputs make the reference raise: a last chunk too short for one output sample (cv2.resize to width 0) and a file
that ends inside a 16-bit sample or inside the first two bytes of a 24-bit one (np.frombuffer / a broadcast).  The
product's loaders take no sample from such a chunk and drop a partial frame; `oracle_load(case, documented=True)` is
the oracle with exactly those two rules applied to what it reads (DESIGN.md section 2), and `case.quirk` says which
rule a case needs.

`branches` reports which paths of the GPU median selection (sushi_b200/csrc/sb_loader.cu, medians_from_histograms) a
padded array takes; `assert_coverage` checks that the set as a whole takes every one of them."""
import math
import os
import struct

import numpy as np

from oracle import ref_loader
from sushi_b200 import synth

SEED = 20261015
N_SEEDED = 110
RATES = (8000, 11025, 22050, 12000, 32000, 44100, 48000, 96000, 7919, 12001)
OUT_RATES = (12000, 8000, 24000)
CHANNELS = (1, 2, 3, 5, 6, 8, 64)
MAX_CHANNELS = 64
FAMILIES = (
    'programme',      # synth.programme_audio, channels offset from one another
    'silence',
    'dc_pos',         # every sample > 0: the subset {x <= 0} is empty, padding included
    'dc_neg',         # every sample < 0: {x >= 0} is empty
    'half_zeros',     # half zeros, half the smallest positive value: one middle rank is 0, the other just above it
    'two_valued',     # -5000, -40, 40, 5000 in quarters: the middle ranks of each subset fall in different coarse bins
    'bin_edges',      # acc = 32 * ch * k and 32 * ch * k +- 1 (acc = -1 included): values on coarse-bin edges
    'full_scale',     # -32768 and 32767 (24-bit: -0x800000 and 0x7FFFFF): medians in the first and the last bin
    'exact_quant',    # medians +-85 and every integer in [-255, 255]: x * 255 + 0.5 lands on integers
)
CONTAINERS = ('plain', 'after', 'truncated', 'ragged', 'odd_before', 'extensible')
BRANCHES = ('zero', 'bin1024', 'bin0', 'split', 'four_bins', 'empty')
KSDATAFORMAT_SUBTYPE_PCM = bytes.fromhex('0100000000001000800000aa00389b71')
COARSE_WIDTH, COARSE_ZERO, COARSE_BINS = 32, 1024, 2048


class LoaderCase(object):
    def __init__(self, name, wav, sample_rate, sample_type, framerate, channels, width, header_frames, container,
                 family, quirk):
        self.name, self.wav, self.sample_rate, self.sample_type = name, wav, sample_rate, sample_type
        self.framerate, self.channels, self.width = framerate, channels, width
        self.header_frames, self.container, self.family, self.quirk = header_frames, container, family, quirk

    @property
    def sample_count(self):                       # wav.py:113-116
        return math.ceil(self.header_frames / float(self.framerate) * self.sample_rate)

    @property
    def padded_length(self):                      # wav.py:119
        return int(10 * 2 * self.framerate + self.sample_count)

    def write(self, directory):
        path = os.path.join(str(directory), self.name + '.wav')
        with open(path, 'wb') as f:
            f.write(self.wav)
        return path

    def __repr__(self):
        return 'LoaderCase(%s)' % self.name


# ---- the file ----------------------------------------------------------------------------------------------------
def riff(channels, framerate, width, payload, data_size, before=b'', after=b'', extensible=False):
    if extensible:
        fmt = struct.pack('<HHLLHHHHL', 0xFFFE, channels, framerate, framerate * channels * width, channels * width,
                          8 * width, 22, 8 * width, 0) + KSDATAFORMAT_SUBTYPE_PCM
    else:
        fmt = struct.pack('<HHLLHH', 1, channels, framerate, framerate * channels * width, channels * width, 8 * width)
    body = b'WAVE' + b'fmt ' + struct.pack('<L', len(fmt)) + fmt + before + b'data' + struct.pack('<L', data_size)
    body += payload + after
    return b'RIFF' + struct.pack('<L', len(body)) + body


def encode(pcm, width, rng, low_bytes=None):
    """(frames, channels) int16 -> interleaved little-endian bytes; 24-bit gets random low bytes unless given."""
    pcm = np.ascontiguousarray(pcm, np.int16).reshape(-1)
    if width == 2:
        return pcm.astype('<i2').tobytes()
    out = np.empty((pcm.size, 3), np.uint8)
    out[:, 0] = rng.integers(0, 256, pcm.size, dtype=np.uint8) if low_bytes is None else low_bytes.reshape(-1)
    u = pcm.view(np.uint16)
    out[:, 1] = u & 0xFF
    out[:, 2] = u >> 8
    return out.tobytes()


# ---- the values ----------------------------------------------------------------------------------------------------
def spread(acc, channels, rng):
    """Per-frame channel sums -> (frames, channels) int16 whose rows add up to acc exactly, not all channels equal."""
    acc = np.asarray(acc, np.int64)
    q = np.floor_divide(acc, channels)
    r = acc - q * channels
    pcm = q[:, None] + (np.arange(channels)[None, :] < r[:, None])
    if channels > 1:
        d = rng.integers(-300, 301, len(acc))
        a, b = pcm[:, 0] + d, pcm[:, 1] - d
        ok = (a >= -32768) & (a <= 32767) & (b >= -32768) & (b <= 32767)
        pcm[ok, 0], pcm[ok, 1] = a[ok], b[ok]
    assert pcm.min(initial=0) >= -32768 and pcm.max(initial=0) <= 32767
    return pcm.astype(np.int16)


def family_pcm(family, frames, channels, rng, framerate, exact=None):
    """(frames, channels) int16 of a value family, plus 24-bit low bytes where the family fixes them.
    exact: (count of the two outer values, count of the two inner ones) for the quarters of 'two_valued', or the
    number of zero frames for 'half_zeros'; otherwise the layout is proportional."""
    lo_bytes = None
    ch = channels
    if family == 'programme':
        base = synth.programme_audio(max(frames, 1), int(rng.integers(1 << 30)), rate=framerate)[:frames].astype(np.int64)
        pcm = np.stack([np.roll(base, 7 * c) // (1 + c % 3) for c in range(ch)], 1).astype(np.int16)
    elif family == 'silence':
        pcm = np.zeros((frames, ch), np.int16)
    elif family in ('dc_pos', 'dc_neg'):
        mag = rng.integers(1, 3000, frames) * ch + rng.integers(0, ch, frames)
        pcm = spread(mag if family == 'dc_pos' else -mag, ch, rng)
        pcm = np.abs(pcm) if family == 'dc_pos' else -np.abs(pcm)
        pcm[pcm == 0] = 1 if family == 'dc_pos' else -1
    elif family == 'half_zeros':
        nz = frames // 2 if exact is None else exact
        acc = np.concatenate([np.zeros(nz, np.int64), np.ones(frames - nz, np.int64)])
        pcm = np.zeros((frames, ch), np.int16)
        pcm[:, 0] = acc
    elif family == 'two_valued':
        outer, inner = (frames // 4, frames // 4) if exact is None else exact
        counts = [outer, inner, inner, frames - outer - 2 * inner]
        acc = np.repeat(np.array([-5000, -40, 40, 5000], np.int64) * ch, counts)
        pcm = spread(acc, ch, rng)
    elif family == 'bin_edges':
        w = COARSE_WIDTH * ch
        edges = np.array([w * k + d for k in (-3, -1, 0, 1, 3) for d in (-1, 0, 1)] + [-1], np.int64)
        acc = np.where(rng.random(frames) < 0.7, rng.choice(edges, frames),
                       w * rng.integers(-1024, 1024, frames) + rng.integers(-1, 2, frames))
        acc = np.clip(acc, -32768 * ch, 32767 * ch)
        pcm = spread(acc, ch, rng)
    elif family == 'full_scale':
        pcm = np.where(rng.random((frames, ch)) < 0.5, -32768, 32767).astype(np.int16)
        pcm[rng.random((frames, ch)) < 0.05] = 0
        lo_bytes = np.where(pcm == 32767, 0xFF, 0x00).astype(np.uint8)
    elif family == 'exact_quant':
        u = rng.random(frames)
        v = np.where(u < 0.3, 85, np.where(u < 0.6, -85, rng.integers(-255, 256, frames)))
        pcm = spread(v.astype(np.int64) * ch, ch, rng)
    else:
        raise ValueError(family)
    return pcm, lo_bytes


# ---- one case ------------------------------------------------------------------------------------------------------
def predict_quirk(framerate, sample_rate, header_frames, width, channels, file_bytes_after_data):
    """Which documented rule the case needs, from the reads of the reference's chunk loop: 'ragged' when the bytes it
    reads end inside a sample the way np.frombuffer / the 24-bit unpack reject, 'zero_chunk' when a read yields frames
    that resample to no sample; None when the reference loads the file."""
    fs = channels * width
    reads = math.ceil(header_frames / float(framerate))
    got = min(reads * framerate * fs, file_bytes_after_data)
    extra = got % fs
    if (width == 2 and extra % 2) or (width == 3 and extra % 3 == 2):
        return 'ragged'
    rate = sample_rate / float(framerate)
    for i in range(reads):                        # a read past the end of a truncated file is empty
        frames = min(max(got - i * framerate * fs, 0), framerate * fs) // fs
        if rate != 1 and math.floor(frames * rate + 0.5) == 0:
            return 'zero_chunk'
    return None


def make_case(name, framerate, channels, width, frames, family, container='plain', sample_rate=12000,
              sample_type='uint8', seed=0, exact=None, cut=None, after_frames=None):
    """frames: the header's frame count.  cut: for 'truncated' / 'ragged', the bytes of PCM the file holds.
    after_frames: for 'after', the size of the chunk after the PCM in frames (header included)."""
    rng = np.random.default_rng([SEED, seed])
    fs = channels * width
    pcm, lo_bytes = family_pcm(family, frames, channels, rng, framerate, exact)
    payload = encode(pcm, width, rng, lo_bytes)
    data_size = len(payload)
    before = after = b''
    if container == 'after':
        k = after_frames or int(rng.integers(4, 40))
        k = max(k, -(-8 // fs))
        body = rng.integers(0, 256, fs * k - 8, dtype=np.uint8).tobytes()
        after = b'LIST' + struct.pack('<L', len(body)) + body
    elif container in ('truncated', 'ragged'):
        payload = payload[:cut]
    elif container == 'odd_before':
        before = b'junk' + struct.pack('<L', 5) + b'odd!!' + b'\x00'
    wav = riff(channels, framerate, width, payload, data_size, before, after, container == 'extensible')
    quirk = predict_quirk(framerate, sample_rate, frames, width, channels, len(payload) + len(after))
    return LoaderCase(name, wav, sample_rate, sample_type, framerate, channels, width, frames, container, family, quirk)


def zero_tail(framerate, sample_rate):
    """Frames of a last chunk that resamples to zero samples (largest such count), or None."""
    rate = sample_rate / float(framerate)
    z = [k for k in range(1, 8) if math.floor(k * rate + 0.5) == 0]
    return z[-1] if z else None


def gap_tail(framerate, sample_rate):
    """Frames of a last chunk whose resampled length rounds down while ceil(total * rate) rounds up: a one-sample gap
    before the tail padding."""
    for k in range(1, framerate):
        if math.ceil((framerate + k) / float(framerate) * sample_rate) > sample_rate + math.floor(
                k * (sample_rate / float(framerate)) + 0.5) and math.floor(k * sample_rate / float(framerate) + 0.5) > 0:
            return k
    return None


# ---- the set -------------------------------------------------------------------------------------------------------
def named_cases():
    cases = []
    stypes = ('uint8', 'float32')

    def add(name, *a, **kw):
        kw.setdefault('seed', len(cases))
        cases.append(make_case(name, *a, **kw))

    small_ch = (1, 2, 3, 5, 6, 8)
    # every frame rate at every frame-count corner
    for i, fr in enumerate(RATES):
        counts = [('empty', 0), ('one', 1), ('fr_m1', fr - 1), ('fr', fr), ('fr_p1', fr + 1)]
        zt, gt = zero_tail(fr, 12000), gap_tail(fr, 12000)
        if zt:
            counts.append(('zero_tail', 2 * fr + zt))
        if gt:
            counts.append(('gap_tail', fr + gt))
        for j, (what, frames) in enumerate(counts):
            ch = small_ch[(i + j) % len(small_ch)]
            width = 2 + (i + j) % 2
            fam = 'programme' if j % 3 else ('bin_edges' if j % 2 else 'exact_quant')
            add('rate%d_%s_ch%d_w%d' % (fr, what, ch, width), fr, ch, width, frames, fam,
                sample_type=stypes[(i + j) % 2])
    # Python 2 rounding of a half sample at 48 kHz, with both widths
    for width in (2, 3):
        add('rate48000_fr_p2_w%d' % width, 48000, 2, width, 48002, 'programme', sample_type=stypes[width - 2])
    # the other output rates
    for i, (fr, sr) in enumerate([(44100, 8000), (48000, 8000), (7919, 8000), (12001, 8000), (8000, 8000),
                                  (44100, 24000), (48000, 24000), (96000, 24000), (12001, 24000), (22050, 24000)]):
        zt = zero_tail(fr, sr)
        frames = 2 * fr + zt if zt and i % 2 == 0 else fr + 1 + 317 * i
        add('rate%d_to%d' % (fr, sr), fr, small_ch[i % 6], 2 + i % 2, frames, 'programme', sample_rate=sr,
            sample_type=stypes[i % 2])
    # every channel count, 64 included, with both widths
    for i, ch in enumerate(CHANNELS):
        for width in (2, 3):
            fr = 48000 if ch == 64 else (11025, 44100)[width - 2]
            add('ch%d_w%d' % (ch, width), fr, ch, width, fr + 1000 + 13 * i, ('programme', 'bin_edges')[width - 2],
                sample_type=stypes[(i + width) % 2])
    # every value family at 12 kHz (the identity map) and 44.1 kHz, both sample types
    for i, fam in enumerate(FAMILIES):
        for fr in (12000, 44100):
            for st in stypes:
                ch = small_ch[(i + len(st)) % 6]
                add('fam_%s_rate%d_ch%d_%s' % (fam, fr, ch, st), fr, ch, 2 + i % 2, fr + 5 + 3 * i, fam, sample_type=st)
    # exact layouts at 12 kHz, where padded = P x first + content + P x last with P = 120000:
    # half zeros -> ranks P + m - 1 and P + m of {x >= 0} are 0 and the smallest positive value;
    # quarters (m, m + P, m + P, m) -> every subset has two middle ranks in different coarse bins: four fine bins
    for st in stypes:
        add('exact_half_zeros_%s' % st, 12000, 1, 2, 12000, 'half_zeros', sample_type=st, exact=6000)
        add('exact_four_bins_%s' % st, 12000, 2, 3, 252000, 'two_valued', sample_type=st, exact=(3000, 123000))
    # container shapes, at a resampled rate and at 12 kHz
    for fr in (48000, 12000):
        for fam, ch, width in (('programme', 2, 2), ('dc_neg', 1, 3)):
            fs = ch * width
            add('after_%d_%s' % (fr, fam), fr, ch, width, int(1.7 * fr) + 3, fam, container='after', after_frames=fr // 3)
            add('truncated_%d_%s' % (fr, fam), fr, ch, width, 5 * fr, fam, container='truncated',
                cut=(2 * fr + fr // 3) * fs, sample_type='float32')
        add('ragged_%d_stereo' % fr, fr, 2, 2, 3 * fr, 'programme', container='ragged', cut=(fr + 901) * 4 + 2)
        add('ragged_%d_odd_byte' % fr, fr, 1, 2, 3 * fr, 'programme', container='ragged', cut=(fr + 901) * 2 + 1)
        add('ragged_%d_w3_one_byte' % fr, fr, 1, 3, 3 * fr, 'dc_pos', container='ragged', cut=(fr + 55) * 3 + 1)
        add('ragged_%d_w3_two_bytes' % fr, fr, 1, 3, 3 * fr, 'dc_pos', container='ragged', cut=(fr + 55) * 3 + 2)
        add('odd_before_%d' % fr, fr, 3, 2, fr + 77, 'programme', container='odd_before')
        add('extensible_%d' % fr, fr, 6, 3, fr + 99, 'full_scale', container='extensible', sample_type='float32')
    return cases


def seeded_cases(n=N_SEEDED, seed=SEED):
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(n):
        fr = int(rng.choice(RATES))
        sr = int(rng.choice(OUT_RATES, p=[0.6, 0.2, 0.2]))
        ch = int(rng.choice(CHANNELS, p=[0.25, 0.25, 0.12, 0.12, 0.1, 0.1, 0.06]))
        if ch == 64:
            fr = min(fr, 48000)
        width = int(rng.integers(2, 4))
        fam = str(rng.choice(FAMILIES))
        container = str(rng.choice(CONTAINERS, p=[0.6, 0.1, 0.1, 0.05, 0.1, 0.05]))
        kind = int(rng.integers(0, 4))
        if kind == 0:
            frames = int(rng.integers(1, 3 * fr))
        elif kind == 1:
            frames = fr * int(rng.integers(1, 3)) + int(rng.integers(-8, 9))
        elif kind == 2:
            frames = int(rng.integers(1, 64))
        else:
            frames = fr + (zero_tail(fr, sr) or gap_tail(fr, sr) or 1)
        if ch == 64:
            frames = min(frames, fr + 4099)
        frames = max(frames, 1)
        cut = None
        if container in ('truncated', 'ragged'):
            cut = int(rng.integers(0, frames)) * ch * width
            if container == 'ragged':
                cut += int(rng.integers(1, ch * width)) if ch * width > 1 else 0
        cases.append(make_case('seeded%03d_rate%d_to%d_ch%d_w%d_%s_%s' % (i, fr, sr, ch, width, fam, container),
                               fr, ch, width, frames, fam, container, sr, str(rng.choice(['uint8', 'float32'])),
                               seed=10000 + i, cut=cut))
    return cases


def all_cases():
    cases = named_cases() + seeded_cases()
    names = [c.name for c in cases]
    assert len(set(names)) == len(names)
    # coverage of the geometry (the value branches need the oracle: assert_coverage)
    assert {c.framerate for c in cases} == set(RATES)
    assert {c.sample_rate for c in cases} == set(OUT_RATES)
    assert {c.channels for c in cases} == set(CHANNELS)
    assert {c.width for c in cases} == {2, 3}
    assert {c.family for c in cases} == set(FAMILIES)
    assert {c.container for c in cases} == set(CONTAINERS)
    assert {c.padded_length % 8 for c in cases} == set(range(8))
    assert {c.quirk for c in cases} == {None, 'zero_chunk', 'ragged'}
    assert any(c.header_frames == 0 for c in cases)
    for fr in RATES:
        have = {c.header_frames for c in cases if c.framerate == fr}
        assert {1, fr - 1, fr, fr + 1} <= have, fr
    assert 48002 in {c.header_frames for c in cases if c.framerate == 48000}
    for fr in (48000, 12000):
        got = {c.container for c in cases if c.framerate == fr}
        assert {'after', 'truncated'} <= got, fr
    return cases


# ---- the truth -----------------------------------------------------------------------------------------------------
def oracle_padded(case, path, documented=False):
    """The oracle's padded float32 array before normalisation, (data, sample_count, padding_size).  documented=True
    applies the product's two rules to what the reference reads: a partial frame at the end is dropped, and a read
    whose frames resample to no sample contributes none."""
    with open(path, 'rb') as f:
        info = ref_loader.parse_header(f, path)
        fs, fr = info['frame_size'], info['framerate']
        rate = case.sample_rate / float(fr)

        def read_raw(n):
            b = f.read(n * fs)
            return b[:len(b) // fs * fs] if documented else b
        return ref_loader.pad_stream(read_raw, info['frames_count'], fr, info['sample_width'], info['channels'],
                                     case.sample_rate, skip_empty=documented)


def oracle_load(case, path, documented=False):
    """-> (padded float32, data, sample_count, padding_size, min_value, max_value) of the oracle."""
    padded, count, pad = oracle_padded(case, path, documented)
    data, lo, hi = ref_loader.normalise(padded.copy(), case.sample_type)
    return padded, data, count, pad, np.float32(lo), np.float32(hi)


def coarse_bin(v):
    return int(min(max(math.floor(float(v) / COARSE_WIDTH) + COARSE_ZERO, 0), COARSE_BINS - 1))


def branches(padded):
    """The paths the GPU median selection takes on this padded array: a middle rank that is exactly zero ('zero'),
    a non-zero one in the coarse bin just above zero ('bin1024'), one in bin 0 ('bin0'), two middle ranks of one subset
    in different coarse bins ('split'), four fine bins at once ('four_bins'), an empty subset ('empty')."""
    flat = padded.reshape(-1)
    out, bins = set(), set()
    for sub in (flat[flat >= 0], flat[flat <= 0]):
        if sub.size == 0:
            out.add('empty')
            continue
        k = (sub.size - 1) // 2
        ranks = [k] if sub.size % 2 else [k, k + 1]
        vals = np.partition(sub, ranks)[ranks]
        got = []
        for v in vals:
            if v == 0:
                out.add('zero')
                continue
            b = coarse_bin(v)
            out.add('bin1024') if b == COARSE_ZERO else None
            out.add('bin0') if b == 0 else None
            got.append(b)
            bins.add(b)
        if len(got) == 2 and got[0] != got[1]:
            out.add('split')
    if len(bins) == 4:
        out.add('four_bins')
    return out


def exact_quant_hits(padded, lo, hi):
    """Samples whose normalised value x 255 + 0.5 is exactly an integer in float32 (where truncation is sharpest)."""
    with np.errstate(invalid='ignore', divide='ignore'):
        x = np.clip(padded, lo, hi)
        x = (x - lo) / (hi - lo)
        x = x * np.float32(255.0) + np.float32(0.5)
    return int(np.count_nonzero(np.isfinite(x) & (x == np.floor(x))))


def assert_coverage(seen):
    """seen: {case name: (branch set, exact-quantisation hits)} over the whole set."""
    hit = set().union(*[b for b, _ in seen.values()])
    assert hit >= set(BRANCHES), sorted(set(BRANCHES) - hit)
    assert any(q > 0 for _, q in seen.values())
