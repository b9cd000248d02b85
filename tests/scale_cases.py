"""Seeded inputs at the size the benchmark runs (BASELINE config 3: 10 000 events on a pair of 90-minute streams,
+-120 s), with the fp64 closed form as their truth and a model of how run_batch cuts such a batch into launches.

Pure NumPy, shared by tests/test_scale_cases.py (CPU) and tests/test_gpu_scale_closed_form.py.  At this size a batch
goes through launch-level cuts that the small cases of tests/closed_form_cases.py never reach:

* record chunks -- with records (body 3, uint8, find), launch_packed_typed / launch_pair_typed cut a launch into chunks
  of RUN_CHUNK CTAs, each with its own k_finish_runs; a query whose lag blocks straddle a cut has its key merged by
  atomicMin across two finish launches;
* super-chunks -- run_batch groups whole queries until their partitions reach max_parts;
* product-buffer chunks of the blocked class (PREMAC_CHUNK lag blocks);
* stream positions past 2^24 and 2^25, where float32 running values lose integer resolution.

`BatchModel` restates plan_batch / run_batch (sb_matcher.cu) and the chunk loops of sb_fused2.cu for the packed engines
at B = 16384, hop B.  The builder inserts near-tie ladders (the constructions of closed_form_cases.py) at the batch
positions the model picks, so that the two copies of a ladder lie on the two sides of a cut."""
import functools

import numpy as np

from oracle.ref_matcher import sqdiff_normed_fp64
from sushi_b200 import synth
from sushi_b200.wavstream import StreamGeometry
from tests import closed_form_cases as cf

B = cf.B
RATE = 12000
PAD = 10 * RATE                         # the padding of a loaded stream (WavStream.PADDING_SECONDS)
DUR = 5400.0
COUNT = int(DUR * RATE)                 # 64 800 000 samples of content
TOTAL = COUNT + 2 * PAD
SHIFT = 18000                           # the template stream is the image moved left by 1.5 s, plus noise
NOISE = 4
EVENTS = 10000
WINDOW = 120.0
RUN_CHUNK = 1 << 19                     # kRunChunk, sb_fused2.cu
MAX_PARTS = 16384                       # Ctx::max_parts
PREMAC_CHUNK = 4096                     # lag blocks per product buffer, run_batch
BLOCKED_FROM = 12                       # kBlockedFromPartitions
LADDER_N = 5000                         # template length of a ladder (one partition)
LADDER_NK = 180                         # lag blocks of a ladder's window: more than any config-3 query has (177)
                                        # (the long-template batch, 441 at most, takes 460)


# ---------------------------------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------------------------------
def programme_long(n, seed, chunk=1 << 22):
    """closed_form_cases.programme for streams of tens of millions of samples, generated in chunks: smoothed noise
    under an envelope that changes every 2400 samples."""
    rng = np.random.default_rng(seed)
    env = rng.uniform(0.2, 1.0, n // 2400 + 1)
    w = np.hanning(9)
    out = np.empty(n, np.uint8)
    tail = rng.standard_normal(8)
    for a in range(0, n, chunk):
        b = min(a + chunk, n)
        x = np.concatenate([tail, rng.standard_normal(b - a)])
        tail = x[-8:]
        y = np.convolve(x, w, 'valid') * env[np.arange(a, b) // 2400]
        out[a:b] = np.clip(np.rint(128 + 70 * y), 0, 255)
    return out


def shifted_noisy_copy(img, shift, amp, seed, chunk=1 << 22):
    """closed_form_cases.noisy_copy in chunks: img moved left by `shift` samples (wrapping) with +-amp integer noise."""
    rng = np.random.default_rng(seed)
    src = np.concatenate([img[shift:], img[:shift]])
    for a in range(0, src.size, chunk):
        b = min(a + chunk, src.size)
        src[a:b] = np.clip(src[a:b].astype(np.int16) + rng.integers(-amp, amp + 1, b - a, dtype=np.int16), 0, 255)
    return src


def to_float32(arr, levels=None, shift=0):
    """arr / 255 as float32; with levels = (lo, hi), 0.2 * (arr / 255 - 0.5) around lo in the first half of the
    image and around hi in the second (the template stream passes shift = SHIFT so that its copies keep their level)."""
    x = arr.astype(np.float32) / np.float32(255.0)
    if levels is None:
        return x
    x = (x - np.float32(0.5)) * np.float32(0.2)
    cut = TOTAL // 2 - shift
    x[:cut] += np.float32(levels[0])
    x[cut:] += np.float32(levels[1])
    return x


# ---------------------------------------------------------------------------------------------------------------------
# the model of run_batch
# ---------------------------------------------------------------------------------------------------------------------
class BatchModel(object):
    """run_batch's plan of one find batch for engine 2 (per-batch choice), 4 (pairs) or 5 (single lag blocks).

    Processing order: the direct class (P < BLOCKED_FROM partitions) in caller order, then the blocked class.  Every
    position p of that order has k0, nk, P and the item / partition / group bases of plan_batch.  Super-chunks are
    (qb, qe) ranges of positions per class; the units of a direct super-chunk (lag blocks, or pairs of them) are cut
    into record chunks of RUN_CHUNK: `cuts` lists the first unit of every chunk but the first of its super-chunk."""

    def __init__(self, tlen, lag0, nlags, engine=2, max_parts=MAX_PARTS):
        tlen, lag0, nlags = [np.asarray(a, np.int64) for a in (tlen, lag0, nlags)]
        P = (tlen + B - 1) // B
        blocked = P >= BLOCKED_FROM
        self.order = np.concatenate([np.nonzero(~blocked)[0], np.nonzero(blocked)[0]])
        self.n_direct = int((~blocked).sum())
        self.count = tlen.size
        self.P = P[self.order]
        self.k0 = (lag0 // B)[self.order]
        self.nk = ((lag0 + nlags - 1) // B)[self.order] - self.k0 + 1
        self.blocked = blocked[self.order]
        groups = np.where(self.blocked, (self.nk + 7) // 8, (self.nk + 1) // 2)
        excl = lambda a: np.concatenate([[0], np.cumsum(a)])
        self.item_base, self.part_base, self.group_base = excl(self.nk), excl(self.P), excl(groups)
        self.pos_of = np.empty(self.count, np.int64)
        self.pos_of[self.order] = np.arange(self.count)
        d = slice(0, self.n_direct)
        self.use_pairs = engine == 4 or (engine == 2 and self.n_direct > 0 and
                                         float((self.nk[d] * self.P[d]).sum()) >= 4.0 * float(self.nk[d].sum()))
        cap = max(min(int(self.part_base[-1]), max_parts), int(self.P.max()))
        self.superchunks = []                   # (class, qb, qe)
        for cls, (lo, hi) in enumerate(((0, self.n_direct), (self.n_direct, self.count))):
            qb = lo
            while qb < hi:
                qe = int(np.searchsorted(self.part_base, self.part_base[qb] + cap, 'right')) - 1
                qe = min(max(qe, qb + 1), hi)
                self.superchunks.append((cls, qb, qe))
                qb = qe
        self.units = self.group_base if self.use_pairs else self.item_base
        self.cuts, self.finish_launches = [], 0
        for cls, qb, qe in self.superchunks:
            if cls == 0:
                u0, u1 = int(self.units[qb]), int(self.units[qe])
                self.finish_launches += (u1 - u0 + RUN_CHUNK - 1) // RUN_CHUNK
                self.cuts += list(range(u0 + RUN_CHUNK, u1, RUN_CHUNK))
        # the blocked class: product-buffer chunks of whole queries, at most PREMAC_CHUNK lag blocks unless one query
        # alone has more
        self.premac_chunks = []
        for cls, qb, qe in self.superchunks:
            qa = qb
            while cls == 1 and qa < qe:
                qz, ni = qa, 0
                while qz < qe and (qz == qa or ni + self.nk[qz] <= PREMAC_CHUNK):
                    ni += int(self.nk[qz])
                    qz += 1
                self.premac_chunks.append((qa, qz))
                qa = qz

    def owner(self, unit):
        """Position (processing order) of the query that owns a unit."""
        return int(np.searchsorted(self.units, unit, 'right')) - 1

    def unit_of_lag(self, pos, j):
        """The unit (lag block or pair) of position `pos` that evaluates absolute lag j."""
        blk = j // B - int(self.k0[pos])
        assert 0 <= blk < int(self.nk[pos])
        return int(self.units[pos]) + (blk // 2 if self.use_pairs else blk)

    def chunk_of(self, unit):
        """(super-chunk index, record chunk inside it) of a unit of the direct class."""
        for s, (cls, qb, qe) in enumerate(self.superchunks):
            if cls == 0 and self.units[qb] <= unit < self.units[qe]:
                return s, (unit - int(self.units[qb])) // RUN_CHUNK
        raise AssertionError(unit)

    def straddles(self, pos):
        """The cuts that fall inside the units of position pos."""
        return [c for c in self.cuts if self.units[pos] < c < self.units[pos + 1]]


# ---------------------------------------------------------------------------------------------------------------------
# the batch
# ---------------------------------------------------------------------------------------------------------------------
class ScaleBatch(object):
    """Queries (toff, tlen, lag0, nlags) in caller order over one image / template pair, with what is known of them:
    `event` (index into the event list, or -1 for a ladder), `expect` (query -> first index of the minimum, relative
    to lag0), `gap` (query -> exact fp64 gap of the swapped copy; 0 for a mirror), `ladders` (query -> its record)."""

    def __init__(self, rows, event):
        self.rows = [list(r) for r in rows]
        self.event = list(event)
        self.expect, self.gap, self.ladders = {}, {}, {}

    def cols(self):
        return [np.array([r[k] for r in self.rows], np.int64) for k in range(4)]

    @property
    def queries(self):
        return [tuple(r) for r in self.rows]

    def model(self, engine=2, max_parts=MAX_PARTS):
        return BatchModel(*self.cols()[1:], engine=engine, max_parts=max_parts)

    def insert(self, pos, row, ladder):
        self.rows.insert(pos, list(row))
        self.event.insert(pos, -1)
        self.ladders = {(q + 1 if q >= pos else q): v for q, v in self.ladders.items()}
        self.ladders[pos] = ladder


class Ladder(object):
    """One planted near-tie: the query's template lies in the template stream's padding (no event reads it).  A gap
    ladder gets an exact copy at p1 and a swapped copy at p0 < p1 whose fp64 value exceeds the exact copy's by `gap`;
    'rgap' the other way round (the exact copy at p0 first, the swapped one at p1); a mirror gets two exact copies and
    the first must win.  `cut`: (engine, unit) the copies straddle."""

    def __init__(self, kind, g, toff, p0, p1, lag0, nlags, cut=None):
        self.kind, self.g, self.toff, self.p0, self.p1 = kind, g, toff, p0, p1
        self.lag0, self.nlags, self.cut = lag0, nlags, cut
        self.gap = None

    def row(self):
        return (self.toff, LADDER_N, self.lag0, self.nlags)

    @property
    def expect(self):
        return (self.p1 if self.kind == 'gap' else self.p0) - self.lag0

    @property
    def swapped(self):
        """Where the swapped copy sits (None for a mirror)."""
        return {'gap': self.p0, 'rgap': self.p1}.get(self.kind)


def _representable(t):
    """closed_form_cases' mirror rule: nudge samples until sum T^2 is a multiple of the float32 spacing at its size."""
    k = 0
    while True:
        tsq = int(np.dot(t.astype(np.int64), t.astype(np.int64)))
        ulp = 2 ** (int(np.floor(np.log2(tsq))) - 23)
        if tsq % ulp == 0:
            return t
        i = 17 * k % t.size
        t[i] = t[i] + 1 if t[i] < 255 else t[i] - 1
        k += 1


def _window_around(kc, m_second, nk):
    """A ladder window of nk lag blocks whose local lag block m_second is the image's block kc."""
    k0 = kc - m_second
    lag0 = k0 * B + 100
    last = (k0 + nk - 1) * B + 50
    assert k0 >= 0 and last + LADDER_N <= TOTAL
    return lag0, last - lag0 + 1


def _place_cut_ladders(batch, engines, kinds, blocks, next_toff, nk=LADDER_NK):
    """Insert a ladder at the query that owns the last unit before every cut of the models of `engines`, earliest
    first, until every cut is straddled by a ladder: its lag block m (last of chunk c) holds p0 and m + 1 (first of
    chunk c + 1) holds p1; around a pair cut, m is the second half of the last pair of chunk c."""
    kinds, blocks = list(kinds), list(blocks)
    for _ in range(len(kinds) + 1):
        todo = []
        for engine in engines:
            m = batch.model(engine)
            for c in m.cuts:
                pos = m.owner(c - 1)
                q = int(m.order[pos])
                lad = batch.ladders.get(q)
                if lad is None or lad.cut != (engine, c):
                    todo.append((pos, engine, c, m))
        if not todo:
            return
        assert kinds, 'more cuts than ladders'
        pos, engine, c, m = min(todo, key=lambda t: t[0])
        q = int(m.order[pos])                       # insert before it: the ladder takes its bases
        assert not m.blocked[pos] and q not in batch.ladders
        u = c - 1 - int(m.units[pos])                # the ladder's local unit of the last unit of chunk c
        m_second = 2 * u + 2 if m.use_pairs else u + 1
        assert m_second < nk
        kind, g = kinds.pop(0)
        kc = blocks.pop(0)
        lag0, nlags = _window_around(kc, m_second, nk)
        p0 = kc * B - 900 - 8 * len(blocks)
        p1 = p0 + LADDER_N + 333
        assert p0 // B == kc - 1 and p1 // B == kc
        lad = Ladder(kind, g, next_toff(), p0, p1, lag0, nlags, (engine, c))
        batch.insert(q, lad.row(), lad)
    raise AssertionError('the cuts did not settle')


def _fixed_ladders(next_toff):
    """Ladders whose copies straddle 2^24 and 2^25 and one whose exact copy sits on the stream's last lag."""
    out = []
    for kind, g, p in (('gap', 1e-5, 1 << 24), ('mirror', 0.0, 1 << 25)):
        p0 = p - 2600
        out.append(Ladder(kind, g, next_toff(), p0, p0 + LADDER_N + 100, p - 1000000, 2880001))
    p1 = TOTAL - LADDER_N
    out.append(Ladder('gap', 4e-6, next_toff(), p1 - LADDER_N - 77, p1, p1 - 2880000, 2880001))
    return out


def _plant(img, tmpl, ladders, seed):
    """Write every ladder's template into the template stream and its copies into the image."""
    rng = np.random.default_rng(seed)
    regions = []
    for i, lad in enumerate(ladders):
        t = cf.programme(LADDER_N, seed + 1 + i)
        if lad.kind == 'mirror':
            # a quiet template (a tenth of the programme's swing around 128): the fp32 FFT rounding of sum(I*T), which
            # grows with the centred template's norm, stays well below half the float32 spacing of sum T^2, so the
            # two exact copies round to the same value (at full swing it reaches that spacing at this size)
            t = _representable(np.clip(np.rint(128 + 0.1 * (t.astype(np.float64) - 128)), 0, 255).astype(np.uint8))
        tmpl[lad.toff:lad.toff + LADDER_N] = t
        if lad.kind == 'mirror':
            img[lad.p0:lad.p0 + LADDER_N] = t
            img[lad.p1:lad.p1 + LADDER_N] = t
            lad.gap = 0.0
        elif lad.kind == 'gap':
            lad.gap = cf._plant_generic(img, t, lad.p0, lad.p1, rng, lad.g)
        else:
            tsq = int(np.dot(t.astype(np.int64), t.astype(np.int64)))
            pert = t.copy()
            for a, b in cf._swap_pairs(t, lad.g * tsq / 2.0, rng):
                pert[a], pert[b] = t[b], t[a]
            img[lad.p0:lad.p0 + LADDER_N] = t
            img[lad.p1:lad.p1 + LADDER_N] = pert
            lad.gap = float(np.sum((pert.astype(np.int64) - t.astype(np.int64)) ** 2)) / tsq
        regions += [(lad.p0, lad.p0 + LADDER_N), (lad.p1, lad.p1 + LADDER_N)]
    regions.sort()
    assert all(a[1] <= b[0] for a, b in zip(regions, regions[1:])), 'planted copies overlap'
    return regions


def _known_lags(batch, regions):
    """expect for every event whose copy (the image at toff + SHIFT) lies in its window and outside every planted
    region, and for every ladder."""
    lo = np.array([r[0] for r in regions])
    hi = np.array([r[1] for r in regions])
    for q, (toff, n, lag0, nlags) in enumerate(batch.rows):
        if batch.event[q] < 0:
            lad = batch.ladders[q]
            batch.expect[q], batch.gap[q] = lad.expect, lad.gap
            continue
        a = toff + SHIFT
        if lag0 <= a < lag0 + nlags and not ((lo < a + n) & (hi > a)).any():
            batch.expect[q] = a - lag0


class Scale(object):
    """Everything the scale tests use: the uint8 pair, the config-3 batch with its ladders, the long-template batch."""


@functools.lru_cache(maxsize=None)
def build(seed=9001):
    s = Scale()
    s.image = programme_long(TOTAL, seed)
    s.template = shifted_noisy_copy(s.image, SHIFT, NOISE, seed + 1)
    geom = StreamGeometry(RATE, PAD, COUNT, TOTAL)
    toffs = iter(range(1000, PAD - LADDER_N, LADDER_N + 7))     # ladder templates: the template stream's padding
    next_toff = lambda: next(toffs)

    # config 3: 10 000 events at +-120 s, ladders at every record cut of engines 2 and 4 and at the fixed positions
    s.starts, s.ends = synth.make_events(EVENTS, DUR, 2, 1.0, 4.0)
    toff, tlen, lag0, nlags, s.t0 = geom.plan_queries(geom, s.starts, s.ends, s.starts, np.full(EVENTS, WINDOW))
    batch = ScaleBatch(zip(toff, tlen, lag0, nlags), range(EVENTS))
    for lad in _fixed_ladders(next_toff):
        batch.insert(len(batch.rows), lad.row(), lad)
    kinds = [('gap', 1e-5), ('rgap', 1e-5), ('rgap', 4e-6), ('mirror', 0.0), ('gap', 1e-5), ('mirror', 0.0)]
    blocks = [700, 1500, 2300, 3100, 1900, 2700, 3500, 500]     # lag blocks of the exact copies, spread over the stream
    _place_cut_ladders(batch, (2, 4), kinds, blocks, next_toff)
    s.config3 = batch

    # long templates: 5.5-6 s at +-300 s (P = 5: engine 2 picks pairs) and 12 x 30 s at +-600 s (22 partitions)
    ls, le = synth.make_events(2650, DUR, 11, 5.5, 6.0)
    bs = np.linspace(700.0, 4600.0, 12) + 0.37
    s.long_starts = np.concatenate([ls, bs])
    s.long_ends = np.concatenate([le, bs + 30.0])
    win = np.concatenate([np.full(ls.size, 300.0), np.full(12, 600.0)])
    toff, tlen, lag0, nlags, s.long_t0 = geom.plan_queries(geom, s.long_starts, s.long_ends, s.long_starts, win)
    lb = ScaleBatch(zip(toff, tlen, lag0, nlags), range(len(toff)))
    _place_cut_ladders(lb, (2,), [('gap', 1e-5), ('mirror', 0.0)], [1200, 2600], next_toff, nk=460)
    s.long = lb

    ladders = list(batch.ladders.values()) + list(lb.ladders.values())
    s.regions = _plant(s.image, s.template, ladders, seed + 100)
    _known_lags(batch, s.regions)
    _known_lags(lb, s.regions)
    return s


# ---------------------------------------------------------------------------------------------------------------------
# truth
# ---------------------------------------------------------------------------------------------------------------------
def closed_form(image, template, row):
    toff, n, lag0, nlags = row
    return sqdiff_normed_fp64(image[lag0:lag0 + nlags + n - 1], template[toff:toff + n])


def value_at(image, template, row, idx):
    """fp64 TM_SQDIFF_NORMED of one query at one index (relative to lag0): exact integer sums for uint8."""
    toff, n, lag0, _ = row
    t, w = template[toff:toff + n], image[lag0 + idx:lag0 + idx + n]
    if image.dtype == np.uint8:
        t, w = t.astype(np.int64), w.astype(np.int64)
        tsq, wnd, sit = int(np.dot(t, t)), int(np.dot(w, w)), int(np.dot(w, t))
        num = float(max(wnd - 2 * sit + tsq, 0))
    else:
        t, w = t.astype(np.float64), w.astype(np.float64)
        tsq, wnd, sit = float(np.dot(t, t)), float(np.dot(w, w)), float(np.dot(w, t))
        num = max(wnd - 2.0 * sit + tsq, 0.0)
    den = np.sqrt(float(wnd)) * np.sqrt(float(tsq))
    return num / den if num < den else 1.0
