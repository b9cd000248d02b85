"""Seeded inputs at the edges where the match kernels can go wrong, with the fp64 closed form as their truth.

Pure NumPy, shared by the GPU test (tests/test_gpu_closed_form.py) and the CPU emulator of the packed kernels
(tests/test_kernel_emulation_closed_form.py).  A case is one image stream, one template stream and a list of queries
(toff, n, lag0, nlags) of one sample type; its truth is oracle.ref_matcher.sqdiff_normed_fp64 on the exact slices
(fp64, exact integer window sums for uint8).  Families:

* edge grid -- template lengths, lag counts, lag0 residues (mod 8 = a run, 32 = a thread, 1024 = a warp, B = a lag
  block) and image lengths around the block size, sampled from a seed plus a fixed list of named corners;
* near-tie ladder -- an exact copy of the template and an EARLIER copy whose value exceeds the exact copy's by a known
  gap g, placed in one run of 8 lags, one warp, two warps of one lag block, the two halves of one pair of lag blocks and
  two CTAs; plus the mirror: two exact copies, where the first must win;
* flat curves -- noise against noise (and against templates of 1 and 2 samples: thousands of exact ties), a periodic
  stream with more minima per lag block than a CTA has record slots, silence inside programme audio, a zero template;
* float32 streams -- data in [0, 1], values around 1000 +- 5 (a hard case for the centring), exact-zero stretches.

Every planted copy is recorded with the case (`expect`: query -> index of the first minimum relative to lag0, and
`gap`: query -> the exact gap of the perturbed copy), and tests/test_closed_form_cases.py checks both against the
truth on the CPU."""
import numpy as np

from oracle.ref_matcher import sqdiff_normed_fp64

B = 16384
GAPS = (1e-4, 1e-5, 4e-6)


class ClosedFormCase(object):
    def __init__(self, name, family, image, template, queries, dtype, expect=None, gap=None):
        self.name, self.family, self.dtype = name, family, np.dtype(dtype).type
        self.image = np.ascontiguousarray(image, dtype)
        self.template = np.ascontiguousarray(template, dtype)
        self.queries = [tuple(int(v) for v in q) for q in queries]
        self.expect = dict(expect or {})        # query -> first index of the minimum, relative to lag0
        self.gap = dict(gap or {})              # query -> fp64 value of the perturbed copy minus the exact copy's
        for (toff, n, lag0, nlags) in self.queries:
            assert n >= 1 and nlags >= 1 and 0 <= toff and toff + n <= self.template.size, (name, toff, n)
            assert 0 <= lag0 and lag0 + nlags - 1 + n <= self.image.size, (name, lag0, nlags, n)
        self._truth = None

    def truth(self):
        """fp64 curve of every query (computed once)."""
        if self._truth is None:
            self._truth = [sqdiff_normed_fp64(self.image[lag0:lag0 + nlags + n - 1], self.template[toff:toff + n])
                           for (toff, n, lag0, nlags) in self.queries]
        return self._truth

    @property
    def lags(self):
        return sum(q[3] for q in self.queries)

    def __repr__(self):
        return 'ClosedFormCase(%s)' % self.name


def programme(n, seed):
    """uint8 stand-in for normalised programme audio: smoothed noise under a slowly varying envelope."""
    rng = np.random.default_rng(seed)
    x = np.convolve(rng.standard_normal(n + 8), np.hanning(9), 'valid') * np.repeat(rng.uniform(0.2, 1.0, n // 2400 + 1), 2400)[:n]
    return np.clip(np.rint(128 + 70 * x), 0, 255).astype(np.uint8)


def noisy_copy(img, shift, amp, seed):
    """The image moved left by `shift` samples with +-amp uniform integer noise: templates that have a dip somewhere."""
    rng = np.random.default_rng(seed)
    return np.clip(np.roll(img, -shift).astype(np.int32) + rng.integers(-amp, amp + 1, img.size), 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# edge grid
# ---------------------------------------------------------------------------------------------------------------------
TEMPLATE_LENGTHS = (1, 2, 7, 8, 9, 255, 256, 257, B - 1, B, B + 1, 2 * B - 1, 2 * B + 1, 4 * B + 3, 11 * B + 1, 12 * B + 1,
                    21 * B + 5)                                 # the last: 22 partitions; 11B + 1 = P 12, the blocked route
LAG_COUNTS = (1, 7, 8, 9, 1023, 1024, 1025, B - 1, B, B + 1, 2 * B, 2 * B + 1, 3 * B + 17)
RESIDUE_MODULI = (8, 32, 1024, B)
IMAGE_LENGTHS = (B - 1, B, B + 1, 2 * B, 5 * B + 777)
LONG_IMAGE = 25 * B + 777                                       # holds 22-partition templates with 3B + 17 lags
MAX_LAGS_PER_CASE = 600000


def _lag0(rng, span_hi):
    """A start lag in [0, span_hi] with a chosen residue modulo a run / thread / warp / lag block (or the last lag)."""
    if span_hi <= 0:
        return 0
    if rng.random() < 0.25:
        return span_hi                                          # the range ends on the stream's last possible lag
    m = int(rng.choice(RESIDUE_MODULI))
    r = int(rng.choice([0, 1, m - 1, int(rng.integers(m))]))
    v = int(rng.integers(0, span_hi // m + 1)) * m + r
    while v > span_hi and v >= m:
        v -= m
    return v if v <= span_hi else span_hi


def edge_grid_cases(seed=20261015, per_image=6):
    out = []
    for li, L in enumerate(IMAGE_LENGTHS + (LONG_IMAGE,)):
        img = programme(L, 1000 + li)
        tmpl = noisy_copy(img, 700 if L > 2000 else 3, 4, 2000 + li)
        rng = np.random.default_rng(seed + li)
        queries = []
        # named corners: one-sample template over the whole stream, the whole stream as the template (one lag),
        # the last lag alone, a template of B + 1 up to the last lag
        queries += [(0, 1, 0, min(L, 3 * B + 17)), (0, L, 0, 1), (3, 1, L - 1, 1)]
        if L > B + 1:
            queries.append((1, B + 1, L - (B + 1) - 1000 + 1, 1000))
        if L == LONG_IMAGE:
            queries = [(0, 11 * B + 1, 5 * B - 3, 2 * B + 1), (100, 12 * B + 1, 0, 3 * B + 17), (7, 21 * B + 5, L - (21 * B + 5) - 1024 + 1, 1024),
                       (B, 4 * B + 3, 1024 * 9 + 31, 2 * B)]
        lags = sum(q[3] for q in queries)
        tries = 0
        while len(queries) < per_image + 4 and tries < 200:
            tries += 1
            n = int(rng.choice([v for v in TEMPLATE_LENGTHS if v <= L]))
            nl = int(rng.choice([v for v in LAG_COUNTS if v <= L - n + 1] or [L - n + 1]))
            if lags + nl > MAX_LAGS_PER_CASE:
                continue
            lag0 = _lag0(rng, L - n - nl + 1)
            toff = int(rng.integers(0, tmpl.size - n + 1))
            queries.append((toff, n, lag0, nl))
            lags += nl
        out.append(ClosedFormCase('edge_L%d' % L, 'edge', img, tmpl, queries, np.uint8))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# near-tie ladder
# ---------------------------------------------------------------------------------------------------------------------
def _swap_pairs(t, r_target, rng, exact=False):
    """Pairs (i, j) of template positions whose values differ by chosen amounts d_k with sum d_k^2 >= r_target (and
    as close to it as the data allows; == with exact, r_target an integer).  Swapping the two values of a pair keeps the
    sum of squares of the copy equal to the template's, so the fp64 value of the swapped copy is exactly
    sum (2 d_k^2) / sum T^2."""
    t = t.astype(np.int64)
    used = np.zeros(t.size, bool)
    pairs, rem = [], int(np.ceil(r_target))
    order = rng.permutation(t.size)
    while rem > 0:
        d = int(np.floor(np.sqrt(rem)))
        if d * d < rem and d < 40 and not exact:
            d = d + 1 if (d + 1) ** 2 - rem < rem - d * d else d
        d = max(d, 1)
        found = None
        for i in order:
            if used[i]:
                continue
            js = np.nonzero((t == t[i] + d) & ~used)[0]
            js = js[js != i]
            if js.size:
                found = (int(i), int(js[0]))
                break
        assert found is not None, 'no pair with difference %d' % d
        used[list(found)] = True
        pairs.append(found)
        rem -= d * d
    return pairs


def _plant_generic(img, tmpl, p0, p1, rng, g):
    """Exact copy of tmpl at p1, swapped copy at p0 (p1 - p0 >= n).  Returns the exact gap."""
    n = tmpl.size
    assert p1 - p0 >= n
    tsq = int(np.dot(tmpl.astype(np.int64), tmpl.astype(np.int64)))
    pert = tmpl.copy()
    for i, j in _swap_pairs(tmpl, g * tsq / 2.0, rng):
        pert[i], pert[j] = tmpl[j], tmpl[i]
    img[p1:p1 + n] = tmpl
    img[p0:p0 + n] = pert
    return float(np.sum((pert.astype(np.int64) - tmpl.astype(np.int64)) ** 2)) / tsq


def _periodic_template(s, d, g, n_max):
    """A template of period s (values 90..170 and one pair d apart) whose length makes 2 d^2 / sum T^2 >= g as tightly
    as possible: the copy s samples before the exact one differs from it in that pair only."""
    period = np.array([110, 110 + d] + [90, 165, 140, 125, 150][:s - 2], np.int64)
    sq = np.cumsum(np.tile(period * period, n_max // s + 1))[:n_max]
    n = int(np.nonzero(sq <= 2 * d * d / g)[0][-1]) + 1
    return np.tile(period, n // s + 1)[:n].astype(np.uint8)


def _plant_periodic(img, p0, s, d, g):
    """Copies s < n apart: the region [p0, p0 + s + n) repeats a period of s, so the window at p0 equals the one at
    p0 + s; swapping the first two samples (d apart) of the region perturbs the window at p0 only."""
    t = _periodic_template(s, d, g, 40000)
    n = t.size
    img[p0:p0 + s + n] = np.tile(t[:s], (s + n) // s + 1)[:s + n]
    img[p0], img[p0 + 1] = img[p0 + 1], img[p0]
    tsq = int(np.dot(t.astype(np.int64), t.astype(np.int64)))
    return t, 2.0 * d * d / tsq


# (name, p0, p1 or None for the periodic construction, lag0, nlags) in a stream of 6 lag blocks; the pair and CTA
# placements start their query on lag block 3, so pairs of lag blocks are (3, 4) and (5, 6)
PLACEMENTS = (('run', 8 * 300 + 1, None, 0, 6000),                                # lags 2401 / 2406: one run of 8
              ('warp', B + 3 * 1024 + 40, B + 3 * 1024 + 900, B, B),              # one warp (1024 lags) of one lag block
              ('warps', 2 * B + 1024 + 7, 2 * B + 9 * 1024 + 300, 2 * B, B),       # warps 1 and 9 of lag block 2
              ('pair', 3 * B + 13000, 4 * B + 500, 3 * B, B + 4000),               # lag blocks 3 and 4: one pair
              ('ctas', 4 * B + 9000, 5 * B + 4000, 3 * B, 2 * B + 8000))           # lag blocks 4 and 5: two pairs
LADDER_LENGTH = 6 * B - 300


def near_tie_cases(seed=4242):
    out = []
    for gi, g in enumerate(GAPS):
        rng = np.random.default_rng(seed + gi)
        img = programme(LADDER_LENGTH, seed + 10 + gi)
        tmpl_parts, queries, expect, gap = [], [], {}, {}
        toff = 0
        for q, (name, p0, p1, lag0, nlags) in enumerate(PLACEMENTS):
            if p1 is None:
                d = int(round(np.sqrt(4500 * g * 16000 / 2)))          # about 4500 samples at a mean square of 16000
                t, gq = _plant_periodic(img, p0, 5, d, g)
                p1 = p0 + 5
            else:
                n = min(p1 - p0, 800 if name == 'warp' else 6000)
                t = programme(n, seed + 100 * gi + q)
                gq = _plant_generic(img, t, p0, p1, rng, g)
            assert gq >= g and lag0 <= p0 and p1 < lag0 + nlags
            assert lag0 + nlags - 1 + t.size <= img.size
            queries.append((toff, t.size, lag0, nlags))
            expect[q], gap[q] = p1 - lag0, gq
            tmpl_parts.append(t)
            toff += t.size
        out.append(ClosedFormCase('ladder_g%g' % g, 'ladder', img, np.concatenate(tmpl_parts), queries, np.uint8, expect, gap))
    # the mirror: two exact copies, the first wins.  sum T^2 is made a multiple of the float32 spacing at its magnitude,
    # so that OpenCV's float32 rounding of sum(I*T) starts from a representable value at both copies: the two values are
    # equal unless the FFT rounding at the two positions differs by about half that spacing.
    img = programme(4 * B - 100, seed + 50)
    tmpl_parts, queries, expect = [], [], {}
    toff = 0
    for q, (p0, p1, lag0, nlags, n) in enumerate(((B + 2 * 1024 + 5, B + 11 * 1024 + 77, B, B, 5000),
                                                  (2 * B + 6000, 3 * B + 2000, 2 * B, B + 5000, 6000))):
        t = programme(n, seed + 60 + q)
        tsq = int(np.dot(t.astype(np.int64), t.astype(np.int64)))
        ulp = 2 ** (int(np.floor(np.log2(tsq))) - 23)
        k = 0
        while tsq % ulp:                                         # nudge samples by one until sum T^2 is representable
            i = 17 * k % n
            v = int(t[i])
            t[i] = v + 1 if v < 255 else v - 1
            tsq = int(np.dot(t.astype(np.int64), t.astype(np.int64)))
            k += 1
        img[p0:p0 + n] = t
        img[p1:p1 + n] = t
        queries.append((toff, n, lag0, nlags))
        expect[q] = p0 - lag0
        tmpl_parts.append(t)
        toff += n
    out.append(ClosedFormCase('ladder_mirror', 'mirror', img, np.concatenate(tmpl_parts), queries, np.uint8, expect, {0: 0.0, 1: 0.0}))
    out.append(_sub_resolution_case(seed + 70))
    return out


# sum d^2 of each copy above the base: 2 / sum T^2 ~ 1e-8 per unit, far below the fp32 screening's resolution
FINE_STEPS = (3, 1, 2, 0, 1, 0, 2, 3, 0, 1, 2, 0, 1, 3)


def _sub_resolution_case(seed):
    """The bottom rung: no exact copy, fourteen swapped copies at 1e-5 whose exact values differ by 0 to 6e-8 -- less
    than the fp32 screening values resolve, so which copy wins is decided by the fp64 evaluation of every candidate the
    screening keeps.  Copies in one warp, in neighbouring warps, across lag blocks and pairs."""
    rng = np.random.default_rng(seed)
    img = programme(LADDER_LENGTH, seed)
    n = 3000
    t = programme(n, seed + 1)
    tsq = int(np.dot(t.astype(np.int64), t.astype(np.int64)))
    r0 = int(round(1e-5 * tsq / 2))
    starts = [100 + 6900 * k for k in range(len(FINE_STEPS))]
    starts[1] = starts[0] + n                                # right behind the first copy
    for p, k in zip(starts, FINE_STEPS):
        pert = t.copy()
        for i, j in _swap_pairs(t, r0 + k, rng, exact=True):
            pert[i], pert[j] = t[j], t[i]
        img[p:p + n] = pert
    queries = [(0, n, 0, img.size - n + 1), (0, n, 2 * B + 5, 2 * B)]
    return ClosedFormCase('ladder_sub_resolution', 'fine', img, t, queries, np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# flat curves and degenerate blocks
# ---------------------------------------------------------------------------------------------------------------------
def flat_cases(seed=777):
    out = []
    rng = np.random.default_rng(seed)
    noise = rng.integers(0, 256, 4 * B, dtype=np.uint8)
    other = rng.integers(0, 256, 2 * B, dtype=np.uint8)
    out.append(ClosedFormCase('flat_noise', 'flat', noise, other,
                              [(100, 3000, 0, 3 * B), (5, 1, 3, 2 * B + 1), (9, 2, B - 5, B + 17), (0, 2 * B, 0, 2 * B + 1)],
                              np.uint8))
    # period 1000, exact copies: sixteen minima per lag block, more than a CTA's eight record slots
    period = programme(1000, seed + 1)
    img = np.tile(period, 3 * B // 1000 + 2)[:3 * B]
    out.append(ClosedFormCase('flat_periodic', 'periodic', img, img.copy(), [(2000, 3000, 500, 2 * B + 300), (2345, 700, 0, B)],
                              np.uint8))
    # silence inside programme audio; a zero template (every value 1: index 0); an exact copy next to the silence
    img = programme(3 * B, seed + 2)
    img[9000:31000] = 0
    src = img.copy()
    src[40000:41000] = 0
    out.append(ClosedFormCase('flat_silence', 'silence', img, src,
                              [(12000, 6000, 0, 34001), (100, 5000, 8000, 20000), (33000, 5000, 0, 2 * B + 1000), (40000, 1000, 100, 1000)],
                              np.uint8, expect={0: 0, 2: 33000, 3: 0}))
    return out


def float32_cases(seed=31):
    out = []
    rng = np.random.default_rng(seed)
    img = (programme(4 * B - 3000, seed).astype(np.float32) / np.float32(255.0)).astype(np.float32)
    src = (np.roll(img, -300) + rng.normal(0, 0.01, img.size)).astype(np.float32)
    out.append(ClosedFormCase('f32_unit', 'float32', img, src,
                              [(20000, 18000, 5, 2 * B + 5000), (100, 1, 0, B + 1), (7, B + 1, B - 3, B + 17)], np.float32))
    img = (1000.0 + 5.0 * rng.standard_normal(4 * B)).astype(np.float32)
    out.append(ClosedFormCase('f32_offset', 'float32', img, img.copy(),
                              [(20000, 5000, 2000, 30000), (30000, 2 * B + 1, 0, B + 1), (3, 9, 4 * B - 9 - 1023, 1024)],
                              np.float32, expect={0: 18000}))
    img = (programme(3 * B, seed + 1).astype(np.float32) / np.float32(255.0)).astype(np.float32)
    img[5000:24000] = 0.0
    src = img.copy()
    src[30000:31000] = 0.0
    out.append(ClosedFormCase('f32_zeros', 'float32', img, src,
                              [(6000, 4000, 0, 30001), (30000, 1000, 100, 5000), (35000, 5000, 0, 2 * B + 3000)],
                              np.float32, expect={0: 0, 1: 0, 2: 35000}))
    return out


def all_cases():
    return edge_grid_cases() + near_tie_cases() + flat_cases() + float32_cases()
