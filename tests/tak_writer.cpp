// A seeded TAK encoder mirror for the tests (tests/tak_cases.py compiles it with g++): each stage of FFmpeg's `tak`
// decoder run in reverse.  Given a frame's target samples, it picks the sample shifts, the channel lpc modes, the
// decorrelation (stereo dmode or multichannel pair list), the subframe layout, the filters (orders, shifts,
// quantisation, predictors) and the residual coding at random, then computes the residuals that reproduce the target
// exactly.  It does not try to compress well.  Written from the bitstream as FFmpeg's decoder reads it, independently
// of sushi_b200/csrc/sb_tak.cuh.  Test infrastructure only.
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>

namespace {

struct Rng {
    uint64_t s;
    uint64_t next() {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    int below(int n) { return n <= 0 ? 0 : (int)(next() % (uint64_t)n); }
    int range(int lo, int hi) { return lo + below(hi - lo + 1); }     // [lo, hi]
    bool chance(int percent) { return below(100) < percent; }
};

struct BitWriter {
    std::vector<uint8_t> out;
    int64_t pos = 0;
    void put(uint64_t v, int n) {                   // n bits, lowest first (FFmpeg's little-endian reader)
        for (int k = 0; k < n; ++k, ++pos) {
            if ((pos >> 3) >= (int64_t)out.size()) out.push_back(0);
            if ((v >> k) & 1) out[(size_t)(pos >> 3)] |= (uint8_t)(1u << (pos & 7));
        }
    }
    void sput(int64_t v, int n) { put((uint64_t)v & ((n >= 64) ? ~0ull : ((1ull << n) - 1)), n); }
    void esc4(int v) { if (v) { put(1, 1); put((uint64_t)(v - 1), 4); } else put(0, 1); }
};

// FFmpeg's xcodes rows: init, escape, scale, aescape, bias
struct Code { uint64_t init, escape, scale, aescape, bias; };
const uint32_t kCodes[50][5] = {
    {0x1, 0x1, 0x1, 0x3, 0x8}, {0x2, 0x3, 0x1, 0x7, 0x6}, {0x3, 0x5, 0x2, 0xE, 0xD}, {0x3, 0x3, 0x3, 0xD, 0x18},
    {0x4, 0xB, 0x4, 0x1C, 0x19}, {0x4, 0x6, 0x6, 0x1A, 0x30}, {0x5, 0x16, 0x8, 0x38, 0x32}, {0x5, 0xC, 0xC, 0x34, 0x60},
    {0x6, 0x2C, 0x10, 0x70, 0x64}, {0x6, 0x18, 0x18, 0x68, 0xC0}, {0x7, 0x58, 0x20, 0xE0, 0xC8},
    {0x7, 0x30, 0x30, 0xD0, 0x180}, {0x8, 0xB0, 0x40, 0x1C0, 0x190}, {0x8, 0x60, 0x60, 0x1A0, 0x300},
    {0x9, 0x160, 0x80, 0x380, 0x320}, {0x9, 0xC0, 0xC0, 0x340, 0x600}, {0xA, 0x2C0, 0x100, 0x700, 0x640},
    {0xA, 0x180, 0x180, 0x680, 0xC00}, {0xB, 0x580, 0x200, 0xE00, 0xC80}, {0xB, 0x300, 0x300, 0xD00, 0x1800},
    {0xC, 0xB00, 0x400, 0x1C00, 0x1900}, {0xC, 0x600, 0x600, 0x1A00, 0x3000}, {0xD, 0x1600, 0x800, 0x3800, 0x3200},
    {0xD, 0xC00, 0xC00, 0x3400, 0x6000}, {0xE, 0x2C00, 0x1000, 0x7000, 0x6400}, {0xE, 0x1800, 0x1800, 0x6800, 0xC000},
    {0xF, 0x5800, 0x2000, 0xE000, 0xC800}, {0xF, 0x3000, 0x3000, 0xD000, 0x18000},
    {0x10, 0xB000, 0x4000, 0x1C000, 0x19000}, {0x10, 0x6000, 0x6000, 0x1A000, 0x30000},
    {0x11, 0x16000, 0x8000, 0x38000, 0x32000}, {0x11, 0xC000, 0xC000, 0x34000, 0x60000},
    {0x12, 0x2C000, 0x10000, 0x70000, 0x64000}, {0x12, 0x18000, 0x18000, 0x68000, 0xC0000},
    {0x13, 0x58000, 0x20000, 0xE0000, 0xC8000}, {0x13, 0x30000, 0x30000, 0xD0000, 0x180000},
    {0x14, 0xB0000, 0x40000, 0x1C0000, 0x190000}, {0x14, 0x60000, 0x60000, 0x1A0000, 0x300000},
    {0x15, 0x160000, 0x80000, 0x380000, 0x320000}, {0x15, 0xC0000, 0xC0000, 0x340000, 0x600000},
    {0x16, 0x2C0000, 0x100000, 0x700000, 0x640000}, {0x16, 0x180000, 0x180000, 0x680000, 0xC00000},
    {0x17, 0x580000, 0x200000, 0xE00000, 0xC80000}, {0x17, 0x300000, 0x300000, 0xD00000, 0x1800000},
    {0x18, 0xB00000, 0x400000, 0x1C00000, 0x1900000}, {0x18, 0x600000, 0x600000, 0x1A00000, 0x3000000},
    {0x19, 0x1600000, 0x800000, 0x3800000, 0x3200000}, {0x19, 0xC00000, 0xC00000, 0x3400000, 0x6000000},
    {0x1A, 0x2C00000, 0x1000000, 0x7000000, 0x6400000}, {0x1A, 0x1800000, 0x1800000, 0x6800000, 0xC000000},
};
Code code_of(int mode) {
    const uint32_t* r = kCodes[mode - 1];
    return Code{r[0], r[1], r[2], r[3], r[4]};
}
const int kOrders[15] = {4, 8, 12, 16, 24, 32, 48, 64, 80, 96, 128, 160, 192, 224, 256};

// stats slots (tests/tak_cases.py names them)
enum {
    S_ORDERS, S_SUB_LPC, S_CH_LPC, S_NSUB, S_CONT, S_PATHS, S_PARTITIONED, S_DELTAS, S_DMODES, S_MC_INDEX, S_CHAINED,
    S_SHIFTS, S_CLIPS, S_WRAPS, S_ZERO_SEGMENTS, S_FRESH, S_DVALS, S_FIR_ORDERS, S_COUNT
};

// option slots
enum {
    O_DMODE, O_CH_LPC, O_MAX_SHIFT, O_ORDER, O_NSUB, O_ESCAPE_EVERY, O_MC, O_FILTERED, O_CONT, O_PARTITION, O_PRED,
    O_DSHIFT, O_COUNT
};

struct Enc {
    Rng rng;
    BitWriter w;
    int64_t* st;
    const int32_t* opt;
    int bits, channels, nb, uval, scale;
    int64_t values = 0;

    uint32_t zig(int32_t v) { return ((uint32_t)v << 1) ^ (uint32_t)(v >> 31); }

    // the bits of u in mode c, or -1 when it cannot be coded there; writes when `write`
    int value(uint64_t u, const Code& c, bool force_escape, bool write) {
        const uint64_t top = 1ull << c.init, top2 = top << 1;
        if (!force_escape) {
            if (u < top) {
                if (write) {
                    w.put(u, (int)c.init);
                    if (u >= c.escape) w.put(0, 1);
                    st[S_PATHS] |= u >= c.escape ? 2 : 1;
                }
                return (int)c.init + (u >= c.escape);
            }
            if (u + c.escape < c.aescape) {                         // x = u + escape in [2^init + escape, aescape)
                if (write) { w.put(u + c.escape - top, (int)c.init); w.put(1, 1); st[S_PATHS] |= 4; }
                return (int)c.init + 1;
            }
            const uint64_t base = u + c.escape;
            const uint64_t k = base >= top2 ? (base - (top2 - 1) + c.scale - 1) / c.scale : 0;
            if (k <= 8 && base - k * c.scale >= c.aescape && base - k * c.scale < top2) {
                if (write) {
                    w.put(base - k * c.scale - top, (int)c.init);
                    w.put(1, 1);
                    w.put(0, (int)k);
                    w.put(1, 1);
                    st[S_PATHS] |= 8;
                }
                return (int)(c.init + 2 + k);
            }
        }
        // escape: x in [aescape, 2^(init + 1)), then u = x + bias, or x + bias + scale * (S + 1)
        if (u < c.bias + c.aescape) return -1;
        const uint64_t r = u - c.bias;
        if (r < top2 && !(force_escape && (u & 1))) {
            if (write) {
                w.put(r - top, (int)c.init); w.put(1, 1); w.put(0, 9); w.put(0, 3);
                st[S_PATHS] |= 16;
            }
            return (int)c.init + 13;
        }
        if (r < c.aescape + c.scale) return -1;
        const uint64_t x = c.aescape + (r - c.aescape) % c.scale;
        if (x >= top2) return -1;
        const uint64_t s = (r - x) / c.scale - 1;
        int sb = 1;
        while (sb < 64 && (s >> sb)) ++sb;
        if (sb > 29) return -1;
        if (write) {
            w.put(x - top, (int)c.init); w.put(1, 1); w.put(0, 9);
            if (sb < 7) w.put((uint64_t)sb, 3);
            else { w.put(7, 3); w.put((uint64_t)(sb - 7), 5); }
            w.put(s, sb);
            st[S_PATHS] |= sb < 7 ? 32 : 64;
        }
        return (int)c.init + 13 + sb + (sb >= 7 ? 5 : 0);
    }

    // the cheapest coding mode of vals[0, n) (0 when all are zero), near the one their mean suggests
    int best_mode(const int32_t* v, int n) {
        uint64_t sum = 0;
        bool zero = true;
        for (int i = 0; i < n; ++i) { sum += zig(v[i]); zero &= v[i] == 0; }
        if (zero && n > 0 && rng.chance(70)) return 0;
        const uint64_t mean = n ? sum / (uint64_t)n : 0;
        int t = 1;
        while (t < 26 && (1ull << t) <= mean) ++t;
        int best = -1;
        int64_t best_cost = INT64_MAX;
        for (int mode = std::max(1, 2 * t - 4); mode <= std::min(50, 2 * t + 1) || best < 0; ++mode) {
            if (mode > 50) break;
            const Code c = code_of(mode);
            int64_t cost = 0;
            for (int i = 0; i < n && cost >= 0; ++i) {
                const int b = value(zig(v[i]), c, false, false);
                cost = b < 0 ? -1 : cost + b;
            }
            if (cost >= 0 && cost < best_cost) { best = mode; best_cost = cost; }
        }
        return best;
    }

    void segment(const int32_t* v, int n, int mode) {
        if (mode == 0) { st[S_ZERO_SEGMENTS]++; return; }
        const Code c = code_of(mode);
        const int every = opt[O_ESCAPE_EVERY];
        for (int i = 0; i < n; ++i) {
            const uint64_t u = zig(v[i]);
            ++values;
            const bool force = every > 0 && values % every == 0 && value(u, c, true, false) >= 0;
            value(u, c, force, true);
        }
    }

    // FFmpeg's decode_residues in reverse
    void residues(const int32_t* v, int length) {
        int wlength = uval ? length / uval : 0;
        int rval = length - wlength * uval;
        if (rval < uval / 2) rval += uval;
        else ++wlength;
        const bool can = wlength > 1 && wlength <= 128;
        const bool part = can && (opt[O_PARTITION] < 0 ? rng.chance(50) : opt[O_PARTITION] > 0);
        if (!part) {
            w.put(0, 1);
            const int mode = best_mode(v, length);
            w.put((uint64_t)mode, 6);
            segment(v, length, mode);
            return;
        }
        st[S_PARTITIONED]++;
        w.put(1, 1);
        std::vector<int> modes((size_t)wlength), lens((size_t)wlength);
        for (int i = 0, at = 0; i < wlength; ++i) {
            lens[(size_t)i] = i == wlength - 1 ? rval : uval;
            modes[(size_t)i] = best_mode(v + at, lens[(size_t)i]);
            if (i && rng.chance(30)) modes[(size_t)i] = modes[(size_t)i - 1];      // runs of one mode
            // a mode that cannot code the window is raised until it can
            for (;;) {
                const int m = modes[(size_t)i];
                bool ok = true;
                if (m == 0) { for (int k = 0; k < lens[(size_t)i]; ++k) ok &= v[at + k] == 0; }
                else for (int k = 0; k < lens[(size_t)i] && ok; ++k) ok = value(zig(v[at + k]), code_of(m), false, false) >= 0;
                if (ok) break;
                modes[(size_t)i] = m + 1;
            }
            at += lens[(size_t)i];
        }
        w.put((uint64_t)modes[0], 6);
        for (int i = 1; i < wlength; ++i) {
            const int d = modes[(size_t)i] - modes[(size_t)i - 1];
            int c;
            if (d == 0) c = 0;
            else if (d == -1) c = 1;
            else if (d == 1) c = 2;
            else if (d >= -4 && d <= 4 && !rng.chance(15)) c = (d < 0 ? -d : d) + 1;
            else c = 6;
            st[S_DELTAS] |= 1 << c;
            w.put(0, c);
            if (c < 6) w.put(1, 1);
            if (c >= 3 && c <= 5) w.put(d < 0 ? 1 : 0, 1);
            if (c == 6) w.put((uint64_t)modes[(size_t)i], 6);
        }
        for (int i = 0, at = 0; i < wlength; ++i) {
            segment(v + at, lens[(size_t)i], modes[(size_t)i]);
            at += lens[(size_t)i];
        }
    }

    // the differences that mode (1 to 3) nested prefix sums from element mode - l (level l) turn back into d
    static void unscan(int32_t* d, int mode, int n) {
        for (int l = mode; l >= 1; --l)
            for (int i = n - 1; i > mode - l; --i) d[i] = (int32_t)((uint32_t)d[i] - (uint32_t)d[i - 1]);
    }

    int32_t clip13(int32_t v) {
        if (v < -8192 || v > 8191) { st[S_CLIPS]++; return v < -8192 ? -8192 : 8191; }
        return v;
    }

    // one filtered subframe: history d[hist, hist + order), outputs d[hist + order, + count), coded after the layout
    void filtered(const int32_t* d, int hist, int order, int count) {
        const int dshift = rng.range(0, std::min(16, opt[O_DSHIFT]));
        const int size = rng.range(6, 7);
        const int qbits = rng.chance(50) ? -1 : rng.range(0, 6);
        const int quant = qbits < 0 ? 10 : 10 - (qbits + 1);
        w.esc4(dshift);
        w.put((uint64_t)(size - 6), 1);
        if (qbits < 0) w.put(0, 1);
        else { w.put(1, 1); w.put((uint64_t)qbits, 3); }
        std::vector<int16_t> pred((size_t)std::max(order, 4), 0);
        const int how = opt[O_PRED];
        auto pick = [&](int width) -> int {
            const int lim = 1 << (width - 1);
            if (how == 0) return 0;
            if (how == 1) return rng.range(-std::min(lim, 4), std::min(lim - 1, 4));
            return rng.range(-lim, lim - 1);
        };
        for (int i = 0; i < 2; ++i) { const int v = pick(10); w.sput(v, 10); pred[(size_t)i] = (int16_t)v; }
        for (int i = 2; i < 4; ++i) { const int v = pick(size); w.sput(v, size); pred[(size_t)i] = (int16_t)(v * (1 << (10 - size))); }
        if (order > 4) {
            const int drop = rng.range(0, 1);
            w.put((uint64_t)drop, 1);
            const int tmp = size - drop;
            int x = 0;
            for (int i = 4; i < order; ++i) {
                if (!(i & 3)) { const int g = rng.range(0, 3); w.put((uint64_t)g, 2); x = tmp - g; }
                const int v = pick(x);
                w.sput(v, x);
                pred[(size_t)i] = (int16_t)(v * (1 << (10 - size)));
            }
        }
        // the predictors' filter, by FFmpeg's recurrence
        std::vector<int32_t> t((size_t)std::max(order, 1), 0);
        std::vector<int16_t> filter((size_t)std::max(order, 1), 0);
        if (order) t[0] = pred[0] * 64;
        for (int i = 1; i < order; ++i) {
            for (int j = 0; j < (i + 1) / 2; ++j) {
                const uint32_t a = (uint32_t)t[(size_t)j], z = (uint32_t)t[(size_t)(i - 1 - j)];
                const int32_t p = pred[(size_t)i];
                const int32_t x = (int32_t)(a + (uint32_t)((int32_t)((uint32_t)p * z + 256u) >> 9));
                t[(size_t)(i - 1 - j)] = (int32_t)(z + (uint32_t)((int32_t)((uint32_t)p * a + 256u) >> 9));
                t[(size_t)j] = x;
            }
            t[(size_t)i] = pred[(size_t)i] * 64;
        }
        const int sh = 15 - quant;
        for (int i = 0, j = order - 1; i < order / 2; ++i, --j) {
            filter[(size_t)j] = (int16_t)((1u << (32 - sh)) - (uint32_t)((int32_t)((uint32_t)t[(size_t)i] + (1u << (sh - 1))) >> sh));
            filter[(size_t)i] = (int16_t)((1u << (32 - sh)) - (uint32_t)((int32_t)((uint32_t)t[(size_t)j] + (1u << (sh - 1))) >> sh));
        }
        // residual = prediction - target, the prediction from the target's own history
        std::vector<int16_t> res((size_t)(order + count));
        for (int i = 0; i < order + count; ++i) {
            const int32_t v = d[hist + i] >> dshift;
            res[(size_t)i] = (int16_t)v;
            if (v != (int16_t)v) st[S_WRAPS]++;
        }
        std::vector<int32_t> r((size_t)count);
        for (int i = 0; i < count; ++i) {
            uint32_t v = 1u << (quant - 1);
            for (int j = 0; j < order; ++j) v += (uint32_t)((int32_t)res[(size_t)(i + j)] * filter[(size_t)j]);
            const int32_t p = clip13((int32_t)v >> quant);
            r[(size_t)i] = (int32_t)((uint32_t)p * (1u << dshift) - (uint32_t)d[hist + order + i]);
        }
        residues(r.data(), count);
    }

    // one channel (its values after the filters, before the decorrelation), FFmpeg's decode_channel in reverse
    void channel(const int32_t* d, int shift, int lpc) {
        w.esc4(shift);
        w.sput(d[0], bits - shift);
        w.put((uint64_t)lpc, 2);
        st[S_CH_LPC] |= 1 << lpc;
        st[S_SHIFTS] |= 1 << shift;
        // subframes: boundaries v_1 < ... < v_(n-1) in units of `scale`, the last subframe longer than 0
        const int vmax = std::min(63, (nb - 2) / scale);
        int n = opt[O_NSUB] > 0 ? opt[O_NSUB] : rng.range(1, 8);
        n = std::min(n, vmax + 1);
        if (n < 1) n = 1;
        std::vector<int> v;
        while ((int)v.size() < n - 1) {
            const int x = rng.range(1, vmax);
            if (std::find(v.begin(), v.end(), x) == v.end()) v.push_back(x);
        }
        std::sort(v.begin(), v.end());
        w.put((uint64_t)(n - 1), 3);
        st[S_NSUB] |= 1 << n;
        std::vector<int> len;
        int prev = 0, left = nb - 1;
        for (int x : v) { w.put((uint64_t)x, 6); len.push_back((x - prev) * scale); left -= (x - prev) * scale; prev = x; }
        len.push_back(left);
        int at = 1, prev_len = 0;
        std::vector<int32_t> tmp;
        for (int i = 0; i < n; ++i) {
            const int sz = len[(size_t)i];
            bool filt = rng.chance(opt[O_FILTERED]);
            const bool can_cont = prev_len > 0;
            bool cont = filt && can_cont && (opt[O_CONT] < 0 ? rng.chance(50) : opt[O_CONT] > 0);
            if (filt && (cont ? prev_len : sz) < kOrders[0]) {             // no order fits: the other way, or none
                cont = !cont && can_cont && prev_len >= kOrders[0];
                filt = cont;
            }
            if (!filt) {
                w.put(0, 1);
                residues(d + at, sz);
            } else {
                w.put(1, 1);
                const int cap = cont ? prev_len : sz;
                int idx = opt[O_ORDER];
                if (idx < 0 || kOrders[idx] > cap) {
                    int hi = 0;
                    while (hi < 14 && kOrders[hi + 1] <= cap) ++hi;
                    idx = rng.range(0, hi);
                }
                const int order = kOrders[idx];
                st[S_ORDERS] |= 1 << idx;
                w.put((uint64_t)idx, 4);
                if (can_cont) w.put(cont ? 1 : 0, 1);
                if (cont) {
                    st[S_CONT]++;
                    filtered(d, at - order, order, sz);
                } else {
                    st[S_FRESH]++;
                    const int lpc_w = rng.range(0, 2);
                    st[S_SUB_LPC] |= 1 << lpc_w;
                    w.put((uint64_t)lpc_w, 2);
                    tmp.assign(d + at, d + at + order);
                    unscan(tmp.data(), lpc_w, order);
                    residues(tmp.data(), order);
                    filtered(d, at, order, sz - order);
                }
            }
            at += sz;
            prev_len = sz;
        }
    }
};

struct Decor {
    int dmode = 0, dshift = 0, dfactor = 0, order = 0, dval1 = 0, dval2 = 0;
    int16_t filter[16] = {0};
    int sizes[4] = {0};
};

// p1 changed from p2 (unchanged) by an FIR pair mode, undone: post -> pre values of p1 (both from sample 1)
void unfir(const Decor& d, int32_t* p1, const int32_t* p2, int length, Enc& e) {
    const int half = d.order / 2, length2 = length - (d.order - 1);
    for (int m = 0; m < length; ++m) {
        if (m < half) { if (d.dval1) p1[m] = (int32_t)((uint32_t)p1[m] - (uint32_t)p2[m]); }
        else if (m >= length2 + half) { if (d.dval2) p1[m] = (int32_t)((uint32_t)p1[m] - (uint32_t)p2[m]); }
        else {
            const int s = m - half;
            uint32_t v = 1u << 9;
            for (int k = 0; k < d.order; ++k) v += (uint32_t)((int32_t)(int16_t)(p2[s + k] >> d.dshift) * d.filter[k]);
            const int32_t g = e.clip13((int32_t)v >> 10);
            p1[m] = (int32_t)((uint32_t)g * (1u << d.dshift) - (uint32_t)p1[m]);
        }
    }
}

// a pair's decorrelation undone on post values a (channel c1) and b (channel c2)
void undecorrelate(const Decor& d, int32_t* a, int32_t* b, int nb, Enc& e) {
    for (int i = 1; i < nb && d.dmode <= 5; ++i) {
        switch (d.dmode) {
        case 1: b[i] = (int32_t)((uint32_t)b[i] - (uint32_t)a[i]); break;
        case 2: a[i] = (int32_t)((uint32_t)b[i] - (uint32_t)a[i]); break;
        case 3: {
            const int32_t bb = (int32_t)((uint32_t)b[i] - (uint32_t)a[i]);
            a[i] = (int32_t)((uint32_t)a[i] + (uint32_t)(bb >> 1));
            b[i] = bb;
            break;
        }
        case 4: case 5: {
            int32_t* p1 = d.dmode == 4 ? b : a;
            const int32_t* p2 = d.dmode == 4 ? a : b;
            const int32_t v = (int32_t)(d.dfactor * (uint32_t)(p2[i] >> d.dshift) + 128u) >> 8;
            p1[i] = (int32_t)(((uint32_t)v << d.dshift) - (uint32_t)p1[i]);
            break;
        }
        default: break;
        }
    }
    if (d.dmode == 7) unfir(d, a + 1, b + 1, nb - 1, e);
    if (d.dmode == 6) unfir(d, b + 1, a + 1, nb - 1, e);
}

Decor pick_decor(int dmode, Enc& e) {
    Decor d;
    d.dmode = dmode;
    if (dmode == 4 || dmode == 5) {
        d.dshift = e.rng.range(0, 16);
        d.dfactor = e.rng.range(-512, 511);
    } else if (dmode >= 6) {
        d.dshift = e.rng.range(0, 16);
        d.order = e.rng.chance(50) ? 16 : 8;
        d.dval1 = e.rng.range(0, 1);
        d.dval2 = e.rng.range(0, 1);
        for (int g = 0; g < d.order / 4; ++g) {
            d.sizes[g] = e.rng.range(0, 7);
            const int size = 14 - d.sizes[g], lim = 1 << (size - 1);
            for (int k = 0; k < 4; ++k) d.filter[4 * g + k] = (int16_t)e.rng.range(-lim, lim - 1);
        }
        e.st[S_FIR_ORDERS] |= d.order;
        e.st[S_DVALS] |= d.dval1 | d.dval2 << 1;
    }
    e.st[S_DMODES] |= 1 << dmode;
    return d;
}

void write_decor(const Decor& d, Enc& e) {
    if (d.dmode == 4 || d.dmode == 5) {
        e.w.esc4(d.dshift);
        e.w.sput(d.dfactor, 10);
    } else if (d.dmode >= 6) {
        e.w.esc4(d.dshift);
        e.w.put(d.order == 16, 1);
        e.w.put((uint64_t)d.dval1, 1);
        e.w.put((uint64_t)d.dval2, 1);
        for (int i = 0; i < d.order; ++i) {
            if (!(i & 3)) e.w.put((uint64_t)d.sizes[i / 4], 3);
            e.w.sput(d.filter[i], 14 - d.sizes[i / 4]);
        }
    }
}

}  // namespace

extern "C" {

// The data of one frame (what follows its header, up to and without the data CRC, padded to a byte) for the nb
// samples per channel of pcm (planar: channel ch at pcm[ch * nb]), at `bits` bits.  codec: 2 (mono/stereo) or 4
// (multichannel).  opt: the O_* options (-1 / 0: at random).  stats: the S_* counters, added to.  Returns the byte
// count, or -1 when out is too small.
int64_t tak_encode_data(const int32_t* pcm, int nb, int channels, int bits, int rate, int codec, uint64_t seed,
                        const int32_t* opt, uint8_t* out, int64_t cap, int64_t* stats) {
    Enc e;
    e.rng.s = seed;
    e.st = stats;
    e.opt = opt;
    e.bits = bits; e.channels = channels; e.nb = nb;
    const int units = (int)((((int64_t)rate + 511) >> 9) + 3) & ~3;
    e.uval = units << (rate < 11025 ? 3 : rate < 22050 ? 2 : rate < 44100 ? 1 : 0);
    e.scale = units << 1;
    if (nb < 16) {
        for (int ch = 0; ch < channels; ++ch)
            for (int i = 0; i < nb; ++i) e.w.sput(pcm[ch * nb + i], bits);
    } else {
        // final -> before the shift -> before the lpc scans, per channel
        std::vector<int32_t> d((size_t)channels * nb);
        std::vector<int> shift((size_t)channels), lpc((size_t)channels);
        for (int ch = 0; ch < channels; ++ch) {
            const int32_t* p = pcm + (size_t)ch * nb;
            int div = std::min(16, bits - 1);
            for (int i = 0; i < nb && div > 0; ++i)
                while (div > 0 && (p[i] & ((1 << div) - 1))) --div;
            if (opt[O_MAX_SHIFT] >= 0) div = std::min(div, opt[O_MAX_SHIFT]);
            shift[(size_t)ch] = e.rng.chance(80) ? div : e.rng.range(0, div);
            lpc[(size_t)ch] = opt[O_CH_LPC] >= 0 ? opt[O_CH_LPC] : e.rng.range(0, 3);
            int32_t* q = d.data() + (size_t)ch * nb;
            for (int i = 0; i < nb; ++i) q[i] = p[i] >> shift[(size_t)ch];
            Enc::unscan(q, lpc[(size_t)ch], nb);
        }
        auto chan = [&](int ch) { return d.data() + (size_t)ch * nb; };
        if (codec == 2) {
            Decor dec;
            if (channels == 2) {
                int dmode = opt[O_DMODE] >= 0 ? opt[O_DMODE] : e.rng.range(0, 7);
                if (dmode >= 6 && nb - 1 < 256) dmode = e.rng.range(0, 5);
                dec = pick_decor(dmode, e);
                undecorrelate(dec, chan(0), chan(1), nb, e);
            }
            for (int ch = 0; ch < channels; ++ch) e.channel(chan(ch), shift[(size_t)ch], lpc[(size_t)ch]);
            if (channels == 2) {
                const int extra = e.rng.range(0, 1);
                e.w.put((uint64_t)extra, 1);
                if (extra) e.w.put((uint64_t)e.rng.below(64), 6);
                e.w.put((uint64_t)dec.dmode, 3);
                write_decor(dec, e);
            }
        } else {
            // the pair list: each entry names a new channel (chan1), and maybe a pair: index 1 with a new chan2, the
            // others with a chan2 already decoded (in list order), possibly an earlier pair's output
            struct Entry { int c1, present, index, c2; Decor dec; };
            std::vector<Entry> list;
            const int mc = opt[O_MC];
            if (mc > 0) {
                std::vector<int> order((size_t)channels);
                for (int i = 0; i < channels; ++i) order[(size_t)i] = i;
                for (int i = channels - 1; i > 0; --i) std::swap(order[(size_t)i], order[(size_t)e.rng.below(i + 1)]);
                std::vector<int> done, changed;               // decoded channels; channels a pair has changed
                int mask = 0;
                for (int k = 0; k < channels; ++k) {
                    const int c1 = order[(size_t)k];
                    if (mask & (1 << c1)) continue;
                    Entry en{c1, 0, 0, 0, Decor()};
                    std::vector<int> fresh;
                    for (int c : order) if (!(mask & (1 << c)) && c != c1) fresh.push_back(c);
                    const bool pair = e.rng.chance(mc == 2 ? 90 : 70);
                    if (pair) {
                        std::vector<int> idx;
                        if (!fresh.empty()) idx.push_back(1);
                        if (!done.empty()) { idx.push_back(0); idx.push_back(2); if (nb - 1 >= 256) idx.push_back(3); }
                        if (!idx.empty()) {
                            en.present = 1;
                            en.index = idx[(size_t)e.rng.below((int)idx.size())];
                            if (en.index == 1) en.c2 = fresh[(size_t)e.rng.below((int)fresh.size())];
                            else if (mc == 2 && !changed.empty()) en.c2 = changed[(size_t)e.rng.below((int)changed.size())];
                            else en.c2 = done[(size_t)e.rng.below((int)done.size())];
                        }
                    }
                    if (en.present && en.index == 1) { mask |= 1 << en.c2; done.push_back(en.c2); }
                    mask |= 1 << c1;
                    done.push_back(c1);
                    if (en.present) {
                        const int dm = en.index == 0 ? 1 : en.index == 1 ? 3 : en.index == 2 ? 4 : 6;
                        en.dec = pick_decor(dm, e);
                        e.st[S_MC_INDEX] |= 1 << en.index;
                        if (en.index != 1 && std::find(changed.begin(), changed.end(), en.c2) != changed.end())
                            e.st[S_CHAINED]++;
                        changed.push_back(c1);
                        if (en.index == 1) changed.push_back(en.c2);
                    }
                    list.push_back(en);
                }
                // undone in reverse order; FFmpeg's decorrelate(c1 = chan2, c2 = chan1)
                for (size_t k = list.size(); k-- > 0;)
                    if (list[k].present) undecorrelate(list[k].dec, chan(list[k].c2), chan(list[k].c1), nb, e);
                e.w.put(1, 1);
                e.w.put((uint64_t)(list.size() - 1), 4);
                for (const Entry& en : list) {
                    e.w.put((uint64_t)en.c1, 4);
                    e.w.put((uint64_t)en.present, 1);
                    if (en.present) { e.w.put((uint64_t)en.index, 2); e.w.put((uint64_t)en.c2, 4); }
                }
            } else {
                e.w.put(0, 1);
                for (int ch = 0; ch < channels; ++ch) list.push_back(Entry{ch, 0, 0, 0, Decor()});
            }
            for (const Entry& en : list) {
                if (en.present && en.index == 1) e.channel(chan(en.c2), shift[(size_t)en.c2], lpc[(size_t)en.c2]);
                e.channel(chan(en.c1), shift[(size_t)en.c1], lpc[(size_t)en.c1]);
                if (en.present) write_decor(en.dec, e);
            }
        }
    }
    const int64_t n = (e.w.pos + 7) >> 3;
    if (n > cap) return -1;
    memset(out, 0, (size_t)n);
    memcpy(out, e.w.out.data(), e.w.out.size());
    return n;
}

}  // extern "C"
