// Packed fused lag-block kernels (engines 2-5): the same per-lag-block pipeline as sb_fused.cu
//   spectral multiply-accumulate -> Hermitian packing -> inverse FFT in shared memory -> window sums,
//   selection of the lags that can win -> fp64 evaluation of those -> one 64-bit atomicMin
// rebuilt around pairs of values.  Every value the kernels touch is one half of a float2 whose two halves go
// through identical arithmetic (add2 / mul2 / fma2: two scalar round-to-nearest instructions each on sm_90):
//
//  * Spectra are stored in a "quad" layout: 16-byte chunks A[i] = (re X[i], re X[i+B/2], im X[i], im X[i+B/2])
//    and M[i] = (re X[B-i], re X[B/2-i], im X[B-i], im X[B/2-i]), i = 0 .. B/4, in blocks of 256 A + 256 M.
//    One LDG.128 per operand feeds four fma2 for two bins; the Hermitian packing of bins (i, B-i) and
//    (i+B/2, B/2-i) is elementwise on those pairs.
//  * The first radix-2 step of the inverse FFT (decimation in frequency) is done on the packed pair itself:
//    u[i] = Z[i] + Z[i+B/2], v[i] = (Z[i] - Z[i+B/2]) * W^i.  u and v are two INDEPENDENT half-size
//    transforms with identical twiddles, X[2o] = FFT(u)[o], X[2o+1] = FFT(v)[o]; they travel together as
//    pairs (u.re, v.re), (u.im, v.im) through three radix-16 passes by decimation in frequency -- the first
//    across the CTA, the other two inside one warp each (fft_passes_dif) -- and the last radix-2 step (of
//    which only the "+" half carries valid lags) is folded into the epilogue.
//  * Twiddles of the packing stage are formed in registers from one per-thread base value, so the 64 KB
//    table sb_fused.cu streams from L2 for every item is gone; spectrum rows are 128-byte aligned.
//
// Two kernels share these pieces:
//   k_match_packed  one CTA per lag block;
//   k_match_pair    one CTA per pair of consecutive lag blocks of a query: both are multiplied at once (2P+1
//                   spectrum-row reads instead of 4P), the second product spectrum waits in an L2-resident
//                   park while the first is transformed -- the default for templates of two or more partitions.
// Values agree with sb_fused.cu to fp32 FFT rounding (~2e-7 of the curve); k_match_packed and
// k_match_pair agree bit for bit.
// Template parameters: S = sample type of the stream (uint8_t | float); EPI = body of the epilogue on uint8 streams
// (sb_set_epilogue): 3 = default since round 2 -- run-level bounds pick the runs of 8 lags that can hold a lag block's
// minimum, those leave as records and k_finish_runs evaluates them in fp64 (prep_runs_v3 / finish_item_v3); 1 = the
// first version, everything inside the match kernel (finish_item), also the only body for float32 streams and the
// bit-identical cross-check.
// Tried in earlier versions and dropped: triples of lag blocks (slower than pairs: one quad in flight per
// thread), 16-bit block-floating-point spectrum rows (the dequantisation costs more issue slots than the halved L2
// traffic returns), a persistent warp-specialised variant (multiply warps latency-bound), the Stockham form of the
// FFT passes (six CTA barriers per transform), body 2 (fp32 screening of every lag in an unrolled loop).
#include "sb_internal.h"
#include <cmath>
#include <cstdlib>
#include <vector>

#include "sb_fused_common.cuh"
#include "sb_fft_smem.cuh"

using namespace sb;
using namespace sbf;

// The prefetch of the self-mirrored quad can be compiled out to attribute a measured difference (make EXTRA=-DSB_V2_SPECIAL_PREFETCH=0).
#ifndef SB_V2_SPECIAL_PREFETCH
#define SB_V2_SPECIAL_PREFETCH 1
#endif

namespace {

constexpr int QB = 16384;                 // lags per item = half the real FFT size
constexpr int QT = 512;                   // threads per CTA
constexpr int QNW = QT / 32;
constexpr int Q4 = QB / 4;                // quads per spectrum row are i = 0 .. Q4
// Row layout (float4 units): blocks of 256 quads, each block = 256 A chunks followed by 256 M chunks (8 KB, so
// one TMA bulk copy fetches both halves of 256 quads and a warp's LDG.128 stays fully coalesced); the
// self-mirrored quad i = B/4 sits behind the 16 blocks.
constexpr int QBLK = 256;                 // quads per block
constexpr int QROW = kQuadRowF2 / 2;      // float4 per row
__host__ __device__ constexpr int qa(int i) { return i < Q4 ? (i >> 8) * (2 * QBLK) + (i & (QBLK - 1)) : 2 * Q4; }       // A chunk of quad i
__host__ __device__ constexpr int qm(int i) { return i < Q4 ? qa(i) + QBLK : 2 * Q4 + 1; }                              // M chunk of quad i
static_assert(QROW >= 2 * Q4 + 2 && (QROW * 16) % 128 == 0, "row layout");
// FFT buffer as [16][16][32] chunks with strides (529, 33, 1): element n of the transform's input sits at
// [n / 512][(n / 32) % 16][n % 32]; both strides are 1 mod 16, which makes every access pattern of the three passes
// and of the epilogue hit sixteen distinct 8-byte banks per half warp (fft_passes_dif).
constexpr int kDA = 529, kDB = 33;
constexpr int QPHYS = 16 * kDA;           // physical chunks of the padded FFT buffer
constexpr int kUU = kDA;                  // distance between elements n and n + 512

struct PackedTables {
    const float2* wb;     // [512]     exp(i*pi*t/B)                                                 (packing, per-thread base)
    const float4* d1;     // [8][512]  (W8192^(2a*t), W8192^((2a+1)*t)) as (c0, s0, c1, s1), t = 0..511   (pass 1, after the butterfly)
    const float4* d2;     // [8][32]   same with W512, l = 0..31                                           (pass 2, after the butterfly)
};

// exp(+i*pi*u/32), u = 0..7: the packing twiddle of quad i = t + 512u is wb[t] times this
__device__ constexpr float kC64[8] = {1.0f, 0.99518472667219689f, 0.98078528040323043f, 0.95694033573220882f,
                                      0.92387953251128674f, 0.88192126434835503f, 0.83146961230254524f, 0.77301045336273696f};
__device__ constexpr float kS64[8] = {0.0f, 0.098017140329560602f, 0.19509032201612825f, 0.29028467725446233f,
                                      0.38268343236508978f, 0.47139673682599764f, 0.55557023301960218f, 0.63439328416364549f};

// ---------------------------------------------------------------- packed arithmetic
struct C2 { float2 r, i; };     // two complex numbers (u, v): r = (u.re, v.re), i = (u.im, v.im)
template <bool V> struct BoolTag { static constexpr bool value = V; };

__device__ __forceinline__ float2 neg2(float2 a) { return make_float2(-a.x, -a.y); }
// Two scalar round-to-nearest operations per pair (never contracted, so mul2 followed by add2 stays two roundings)
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return add2(a, neg2(b)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 bc(float s) { return make_float2(s, s); }      // scalar-broadcast operand

__device__ __forceinline__ C2 cadd2(C2 a, C2 b) { return {add2(a.r, b.r), add2(a.i, b.i)}; }
__device__ __forceinline__ C2 csub2(C2 a, C2 b) { return {sub2(a.r, b.r), sub2(a.i, b.i)}; }
// both halves times the same complex number (c, s)
__device__ __forceinline__ C2 cmul_s(C2 a, float c, float s) {
    C2 o;
    o.r = fma2(a.r, bc(c), mul2(a.i, bc(-s)));
    o.i = fma2(a.r, bc(s), mul2(a.i, bc(c)));
    return o;
}
__device__ __forceinline__ C2 from4(float4 v) { return {make_float2(v.x, v.y), make_float2(v.z, v.w)}; }

// d * exp(+2*pi*i*q/32), q even and a compile-time constant after unrolling
__device__ __forceinline__ C2 rot32p(C2 d, int q) {
    if (q == 0) return d;
    if (q == 8) return {neg2(d.i), d.r};
    const float h = 0.70710678118654752f;
    if (q == 4) return {mul2(sub2(d.r, d.i), bc(h)), mul2(add2(d.r, d.i), bc(h))};
    if (q == 12) return {mul2(add2(d.r, d.i), bc(-h)), mul2(sub2(d.r, d.i), bc(h))};
    return cmul_s(d, kC32[q], kS32[q]);
}

// In-register inverse DFT of 16 points on both halves at once; decimation in frequency, natural order in,
// bit-reversed order out (index the result through brev<16>).
// Stages h = HI, HI/2, .., LO of the transform (the whole of it: HI = 8, LO = 1).
template <int HI = 8, int LO = 1>
__device__ __forceinline__ void dft16p(C2 (&v)[16]) {
#pragma unroll
    for (int h = HI; h >= LO; h >>= 1) {
#pragma unroll
        for (int g = 0; g < 16; g += 2 * h) {
#pragma unroll
            for (int a = 0; a < h; ++a) {
                const C2 x = v[g + a], y = v[g + a + h];
                v[g + a] = cadd2(x, y);
                v[g + a + h] = rot32p(csub2(x, y), a * (16 / h));
            }
        }
    }
}

// The FFT buffer is two arrays of float2, R[p] = (u.re, v.re) and I[p] = (u.im, v.im), p = phys(c) for chunk c
// (the register allocator does not keep the two pairs in one aligned quad, so a 128-bit store would cost four
// MOVs; 64-bit accesses cost none).  One padding slot per 16 chunks makes the stride-16 scatter of pass 1 and
// the epilogue's reads of chunks 2t, 2t+1 hit sixteen distinct 8-byte banks per half warp.
__device__ __forceinline__ constexpr int phys(int n) { return (n >> 9) * kDA + ((n >> 5) & 15) * kDB + (n & 31); }
struct Buf {
    float2* r; float2* i;
    __device__ __forceinline__ C2 ld(int p) const { return {r[p], i[p]}; }
    __device__ __forceinline__ void st(int p, C2 v) const { r[p] = v.r; i[p] = v.i; }
};

// ---------------------------------------------------------------- spectrum rows
// Addressing and loading of one quad of a row, in 16-byte units from the row's first unit.
struct Rows {
    static constexpr int STRIDE = QROW;
    // unit of quad tid + 512*uu's A chunk (its M chunk is QBLK further): qa() without the special case
    static __device__ __forceinline__ int unit(int tid, int uu) { return (tid >> 8) * (2 * QBLK) + (tid & (QBLK - 1)) + uu * (2 * QT); }
    static constexpr int USTEP = 2 * QT;             // units between the quads tid + 512*uu and tid + 512*(uu+1)
    static __device__ __forceinline__ void load(const float4* row, int u, float4& a, float4& m) { a = __ldg(row + u); m = __ldg(row + u + QBLK); }
    // predicated form (a row past the end of the stream reads as zero)
    static __device__ __forceinline__ void loadp(const float4* row, int u, bool pred, float4& a, float4& m) {
        const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
        a = pred ? __ldg(row + u) : zero4;  m = pred ? __ldg(row + u + QBLK) : zero4;
    }
    static __device__ __forceinline__ void load_special(const float4* row, float4& a, float4& m) { a = __ldg(row + qa(Q4)); m = __ldg(row + qm(Q4)); }
};
// Spectrum rows are read with plain read-only loads.  (ld.global.nc.L1::no_allocate, tried in an earlier version to
// keep the twiddle tables in L1, lowered the L2 hit rate of these rows and multiplied the kernel's DRAM traffic.)

// ---------------------------------------------------------------- packing of one quad
// a = (Y[i], Y[i+B/2]), m = (Y[B-i], Y[B/2-i]) as packed pairs, (c, s) = exp(i*pi*i/B).
// Hermitian packing (the 2B-point real inverse as a B-point complex one):
//   Z[k] = (Y[k] + conj(Y[B-k])) + i*w^k*(Y[k] - conj(Y[B-k])),  Z[B-k] = conj(e) + i*conj(o)
// then the first radix-2 step of the B-point inverse FFT, on the pair itself:
//   u[k] = Z[k] + Z[k+B/2],  v[k] = (Z[k] - Z[k+B/2]) * W^k,  W = exp(2*pi*i/B) = w^2
// for k = i (from the first slot pair) and k = B/2 - i (from the mirrored pair, W^(B/2-i) = -conj(W^i)).
__device__ __forceinline__ void pack_quad(float2 aR, float2 aI, float2 mR, float2 mI, float c, float s,
                                          C2& lo, C2& hi) {
    const float2 eR = add2(aR, mR), eI = sub2(aI, mI);
    const float2 dR = sub2(aR, mR), dI = add2(aI, mI);
    // slot 0 uses w = (c, s), slot 1 uses w^(i+B/2) = i*w = (-s, c)
    const float2 wR = make_float2(c, -s), wI = make_float2(s, c);
    const float2 oR = fma2(dR, wR, neg2(mul2(dI, wI)));
    const float2 oI = fma2(dR, wI, mul2(dI, wR));
    const float2 zloR = sub2(eR, oI), zloI = add2(eI, oR);       // (Z[i],   Z[i+B/2])
    const float2 zhiR = add2(eR, oI), zhiI = sub2(oR, eI);       // (Z[B-i], Z[B/2-i])
    const float c2 = fmaf(c, c, -s * s), s2 = 2.0f * c * s;      // W^i
    {
        const float ur = zloR.x + zloR.y, ui = zloI.x + zloI.y;
        const float dr = zloR.x - zloR.y, di = zloI.x - zloI.y;
        lo.r = make_float2(ur, dr * c2 - di * s2);  lo.i = make_float2(ui, dr * s2 + di * c2);
    }
    {
        const float ur = zhiR.y + zhiR.x, ui = zhiI.y + zhiI.x;
        const float dr = zhiR.y - zhiR.x, di = zhiI.y - zhiI.x;
        hi.r = make_float2(ur, -(dr * c2) - di * s2);  hi.i = make_float2(ui, dr * s2 - di * c2);   // times (-c2, s2)
    }
}

// ---------------------------------------------------------------- pieces shared by the two kernels
constexpr int kRounds = QB / (QT * 8);            // epilogue rounds: 8 consecutive lags per thread per round
constexpr int kLagsPerRound = QT * 8;

struct Smem {                                      // carve-up of the dynamic shared memory (both kernels)
    Buf buf;                                       // QPHYS chunks, two float2 arrays
    double2* base;                                 // [kRounds][QNW][2] exact running sums
    unsigned char* lo;                             // image[j_blk .. +QB+16)
    unsigned char* hi;                             // image[(j_blk+n)&~15 .. +QB+48)
    unsigned char* end;                            // first byte after the common part (16-byte aligned)
    __device__ __forceinline__ explicit Smem(unsigned char* raw) {
        buf.r = reinterpret_cast<float2*>(raw); buf.i = buf.r + QPHYS;
        base = reinterpret_cast<double2*>(raw + (size_t)QPHYS * 16);
        lo = reinterpret_cast<unsigned char*>(base + kRounds * QNW * 2);
        hi = lo + QB + 16;
        end = hi + QB + 48;
    }
};
constexpr int kSmallBytes = 512;                   // room behind Smem::end for the kernels' barriers, reduction scratch, park slot
constexpr size_t kSmemCommon = (size_t)QPHYS * 16 + kRounds * QNW * 2 * sizeof(double2) + (QB + 16) + (QB + 48);

struct Item {                                      // one (query, lag block)
    QueryDesc d; int q; int64_t k, j_blk;
    __device__ __forceinline__ Item(const QueryDesc& dd, int qq, int64_t kk) : d(dd), q(qq), k(kk), j_blk(kk * QB) {}
    __device__ __forceinline__ Item(const QueryDesc* desc, const int* item_query, int64_t item_first, int64_t local) {
        q = __ldg(item_query + local);
        d = desc[q];
        k = d.k0 + (item_first + local - d.itemBase);
        j_blk = k * QB;
    }
};

// uint8 streams: the two byte windows the sliding sums read go to shared memory by TMA bulk copies (one
// thread), one exact (sum, sum of squares) pair per warp-round from the fp64 running sums by cp.async.
// WARP_BASES (body 3): one pair per warp instead -- a warp owns 1024 consecutive lags there.
template <bool WARP_BASES = false>
__device__ __forceinline__ void stage_inputs(const Item& it, int tid, const uint8_t* img8, int64_t img_n,
                                             const double2* ipfx, const Smem& sm, unsigned long long* bar) {
    const int64_t hi0 = (it.j_blk + it.d.tlen) & ~(int64_t)15;
    const int64_t limit = (img_n + 16) & ~(int64_t)15;               // allocation has 16 bytes of slack
    if (tid == 0) {
        int64_t lo_bytes = limit - it.j_blk; if (lo_bytes > QB + 16) lo_bytes = QB + 16; if (lo_bytes < 0) lo_bytes = 0;
        int64_t hi_bytes = limit - hi0;      if (hi_bytes > QB + 48) hi_bytes = QB + 48; if (hi_bytes < 0) hi_bytes = 0;
        mbar_expect_tx(bar, (unsigned)(lo_bytes + hi_bytes));
        if (lo_bytes) tma_load_1d(sm.lo, img8 + it.j_blk, (unsigned)lo_bytes, bar);
        if (hi_bytes) tma_load_1d(sm.hi, img8 + hi0, (unsigned)hi_bytes, bar);
    }
    if (WARP_BASES) {
        if (tid < QNW * 2) {
            const int64_t jw = it.j_blk + (tid >> 1) * (QB / QNW);
            if (jw < it.d.lag0 + it.d.nlags) cp_async16(sm.base + tid, ipfx + jw + ((tid & 1) ? it.d.tlen : 0));
        }
    } else if (tid < kRounds * QNW * 2) {
        const int c = tid / (QNW * 2), w = (tid >> 1) % QNW, which = tid & 1;
        const int64_t jw = it.j_blk + c * kLagsPerRound + w * 256;
        if (jw < it.d.lag0 + it.d.nlags) cp_async16(sm.base + tid, ipfx + jw + (which ? it.d.tlen : 0));
    }
}

// Y += conj(T) * X on both slots of the A and the M chunk of one quad
struct QuadAcc {
    float2 aR, aI, mR, mI;
    __device__ __forceinline__ void zero() { aR = aI = mR = mI = make_float2(0.f, 0.f); }
    __device__ __forceinline__ void mac(float4 ta, float4 tm, float4 xa, float4 xm) {
        const C2 tA = from4(ta), xA = from4(xa), tM = from4(tm), xM = from4(xm);
        aR = fma2(tA.r, xA.r, aR);  aR = fma2(tA.i, xA.i, aR);
        aI = fma2(tA.r, xA.i, aI);  aI = fma2(neg2(tA.i), xA.r, aI);
        mR = fma2(tM.r, xM.r, mR);  mR = fma2(tM.i, xM.i, mR);
        mI = fma2(tM.r, xM.i, mI);  mI = fma2(neg2(tM.i), xM.r, mI);
    }
    __device__ __forceinline__ void reduce_over_lanes() {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            aR.x += __shfl_xor_sync(0xffffffffu, aR.x, o); aR.y += __shfl_xor_sync(0xffffffffu, aR.y, o);
            aI.x += __shfl_xor_sync(0xffffffffu, aI.x, o); aI.y += __shfl_xor_sync(0xffffffffu, aI.y, o);
            mR.x += __shfl_xor_sync(0xffffffffu, mR.x, o); mR.y += __shfl_xor_sync(0xffffffffu, mR.y, o);
            mI.x += __shfl_xor_sync(0xffffffffu, mI.x, o); mI.y += __shfl_xor_sync(0xffffffffu, mI.y, o);
        }
    }
};

// The self-mirrored quad i = B/4 of an item, by one warp: partitions spread over the lanes, result valid in lane 0
__device__ __forceinline__ C2 special_quad(const float4* tp, const float4* xp, int P, int lane) {
    QuadAcc acc; acc.zero();
    for (int p = lane; p < P; p += 32) {
        float4 ta, tm, xa, xm;
        Rows::load_special(tp + (int64_t)p * Rows::STRIDE, ta, tm);
        Rows::load_special(xp + (int64_t)p * Rows::STRIDE, xa, xm);
        acc.mac(ta, tm, xa, xm);
    }
    acc.reduce_over_lanes();
    const float h = 0.70710678118654752f;       // exp(i*pi/4)
    C2 lo, hi;
    pack_quad(acc.aR, acc.aI, acc.mR, acc.mI, h, h, lo, hi);
    return lo;                                    // C[B/4] (its mirror is itself)
}

// Body 3: the same quad without an L2 round trip at the end of the multiply phase, where the
// other fifteen warps already wait at the barrier.  The last warp requests the 16-byte units it needs -- two per
// row: the P template rows, then the spectrum rows k .. k+P+G-2 of the CTA's G lag blocks -- with cp.async before
// its multiply loop; afterwards the partitions are spread over the lanes and summed by the same shuffle tree as
// special_quad (same arithmetic in the same order: bit-identical), reading shared memory instead of L2.
constexpr int kSpecialBytes = 1024;                // (2 * 11 + 2) rows x 32 bytes fit
// Templates of twelve or more partitions normally take the blocked multiply route; when that route is switched off
// (sb_set_premac_mode(1)) they arrive here and their rows do not fit the area: those CTAs read the quad from L2
// (special_quad) like the first kernel body.
__device__ __forceinline__ bool special_fits(int P, int G) { return (2 * P + G - 1) * 32 <= kSpecialBytes; }
__device__ __forceinline__ void special_prefetch(float4* s_sp, const float4* tp, const float4* xp, int P, int G,
                                                 int64_t k, int64_t nblk, int lane) {
    const int u0 = qa(Q4), u1 = qm(Q4);
    for (int r = lane; r < 2 * P + G - 1; r += 32) {
        const bool is_t = r < P;
        const float4* row = is_t ? tp + (int64_t)r * Rows::STRIDE : xp + (int64_t)(r - P) * Rows::STRIDE;
        if (is_t || k + (r - P) < nblk) { cp_async16(s_sp + 2 * r, row + u0); cp_async16(s_sp + 2 * r + 1, row + u1); }
        else s_sp[2 * r] = s_sp[2 * r + 1] = make_float4(0.f, 0.f, 0.f, 0.f);     // rows past the end of the stream are zero
    }
}
__device__ __forceinline__ C2 special_from_smem(const float4* s_sp, int P, int g, int lane) {      // item g; result in lane 0
    auto units = [&](int r, float4& a, float4& m) {
        a = s_sp[2 * r]; m = s_sp[2 * r + 1];
    };
    QuadAcc acc; acc.zero();
    for (int p = lane; p < P; p += 32) {
        float4 ta, tm, xa, xm;
        units(p, ta, tm);
        units(P + g + p, xa, xm);
        acc.mac(ta, tm, xa, xm);
    }
    acc.reduce_over_lanes();
    const float h = 0.70710678118654752f;       // exp(i*pi/4)
    C2 lo, hi;
    pack_quad(acc.aR, acc.aI, acc.mR, acc.mI, h, h, lo, hi);
    return lo;
}

// Inverse FFT of the packed product spectrum: 8192 (u, v) pairs.  Afterwards chunk j of the half-size transforms
// X'[j], j < 4096 (the other half carries no valid lag), holds the correlation (times 2B) at lags 4j .. 4j+3 =
// (u.re, u.im, v.re, v.im), up to the last radix-2 step, which is the epilogue's.
// Decimation in frequency, n = 512a + 32b + 2c + m  ->  k = k1 + 16 k2 + 256 k3 + 4096 k4:
//   pass 1  thread t, over a:  y[k1][t]  = W8192^(t k1) * sum_a x[a][t] W16^(a k1)       t = 32b + 2c + m
//   pass 2  warp k1, lane l, over b:  z[k2][l] = W512^(l k2) * sum_b y[b][l] W16^(b k2)   l = 2c + m
//   pass 3  warp k1, lane (k2, m), over c:  r[k3][m] = sum_c z[c][m] W16^(c k3)           (its twiddle W32^(m k3) and
//           the last radix-2 step, of which only k4 = 0 carries valid lags, are the epilogue's:
//           X[k1 + 16 k2 + 256 k3] = r[k3][0] + W32^k3 r[k3][1])
// Every thread writes each pass's results over its own inputs (buffer [a|k1][b|k2][2(c|k3) + m]), so no pass needs a
// barrier between its loads and its stores, and after pass 1 the sixteen 512-point transforms belong to one warp
// each: passes 2 and 3 synchronise with __syncwarp only.  Two CTA-wide barriers per transform instead of six --
// and, more important, the warps drift apart between them: one warp's shared-memory loads and stores overlap the
// others' arithmetic instead of all sixteen alternating between the two pipes in lock step.  Entered after a barrier that published buf; ends with a barrier.
template <int ID>
__device__ __forceinline__ void fft_passes_dif(const Buf& buf, int tid, const PackedTables& tab, bool drain_cp_async) {
    C2 v[16];
    float4 tw[8];
    const int lane = tid & 31, warp = tid >> 5;
    {   // pass 1
#pragma unroll
        for (int a = 0; a < 8; ++a) tw[a] = __ldg(tab.d1 + a * 512 + tid);
        const int at = warp * kDB + lane;                                   // phys(tid)
#pragma unroll
        for (int a = 0; a < 16; ++a) v[a] = buf.ld(at + kDA * a);
        dft16p(v);
        buf.st(at, v[0]);
#pragma unroll
        for (int k = 1; k < 16; ++k) {
            const float4 t = tw[k >> 1];
            buf.st(at + kDA * k, (k & 1) ? cmul_s(v[brev<16>(k)], t.z, t.w) : cmul_s(v[brev<16>(k)], t.x, t.y));
        }
#pragma unroll
        for (int a = 0; a < 8; ++a) tw[a] = __ldg(tab.d2 + a * 32 + lane);
        csync<ID>();
    }
    {   // pass 2: this warp's 512 points
        const int at = warp * kDA + lane;
#pragma unroll
        for (int b = 0; b < 16; ++b) v[b] = buf.ld(at + kDB * b);
        dft16p(v);
        buf.st(at, v[0]);
#pragma unroll
        for (int k = 1; k < 16; ++k) {
            const float4 t = tw[k >> 1];
            buf.st(at + kDB * k, (k & 1) ? cmul_s(v[brev<16>(k)], t.z, t.w) : cmul_s(v[brev<16>(k)], t.x, t.y));
        }
        __syncwarp();
    }
    {   // pass 3: lane (k2 = lane % 16, m = lane / 16) of this warp
        const int at = warp * kDA + (lane & 15) * kDB + (lane >> 4);
#pragma unroll
        for (int c = 0; c < 16; ++c) v[c] = buf.ld(at + 2 * c);
        dft16p(v);
#pragma unroll
        for (int k = 0; k < 16; ++k) buf.st(at + 2 * k, v[brev<16>(k)]);
        if (drain_cp_async) cp_async_commit_wait_all();     // the staged running sums landed long ago
        csync<ID>();
    }
}

// Body 3: the constants of a query every thread needs in the epilogue -- sums of the template (two reads of its
// running sums) and the two centres (two fp64 divisions) -- by ONE thread at the start of the CTA's work on the
// query, through shared memory; the first version has all 512 threads fetch and divide them after the last FFT
// pass of every item, with the whole CTA waiting on those reads.  [0] = (sum T, sum T^2), [1] = (a, b).
__device__ __forceinline__ constexpr int kQueryConstOff() { return 384; }      // bytes behind Smem::end (small area)
template <typename S>
__device__ __forceinline__ void query_constants(double2* s_qc, const QueryDesc& d, int64_t img_n,
                                                const double2* __restrict__ ipfx, const double2* __restrict__ tpfx) {
    const double2 t_hi = tpfx[d.toff + d.tlen], t_lo = tpfx[d.toff];
    const double tsum = t_hi.x - t_lo.x, tsq = t_hi.y - t_lo.y;
    s_qc[0] = make_double2(tsum, tsq);
    s_qc[1] = make_double2((double)Acc<S>::centre(ipfx[img_n].x, (double)img_n), (double)Acc<S>::centre(tsum, (double)d.tlen));
}

// EPI 3: runs of 8 lags that can hold a lag block's minimum leave the match kernel as records -- the query, the
// run's first lag and the correlation at its 8 lags, rounded exactly like the in-kernel exact path rounds it -- and
// k_finish_runs evaluates their lags in fp64 afterwards (window sums from the running sums: the same exact
// integers).  The match kernel's epilogue then ends after the block minimum: no per-lag loop, no fp64 on the CTA's
// critical path (with the exact evaluation inside, fifteen warps wait at the closing barrier for the one warp that
// holds the candidate).  A CTA has kRunSlots slots; runs that find none
// (degenerate data: silence, constant streams) and the debug curve take the in-kernel path.
constexpr int kRunSlots = 8;
struct RunRecord { int32_t q; int32_t valid; int64_t j0; float cc[8]; };     // 48 bytes
static_assert(sizeof(RunRecord) == 48, "three 16-byte stores");
struct RunSink { RunRecord* recs; int* s_cnt; };                              // recs = this CTA's kRunSlots records (or null)
__device__ __forceinline__ constexpr int kRunCountOff() { return 256; }       // bytes behind Smem::end (small area)
__device__ __forceinline__ constexpr int kNextOff() { return 272; }           // 16 + 80 bytes: query and descriptor of the CTA's next pair (k_match_pair)

// First version of the epilogue (body 1; every sample type): window sums, fp32 screening of every lag, fp64
// evaluation of the lags that can still be the minimum, merge into the query's key.  A thread takes 8 consecutive
// lags in each of four rounds.  after_read() runs (on all 512 threads) once every thread is done with the staged windows.
template <typename S, int ID, typename AfterRead>
__device__ __forceinline__ void finish_item(const Item& it, int tid, const Smem& sm, unsigned long long* s_bar, unsigned bar_parity,
                                            unsigned long long* s_best, float* s_min,
                                            const S* __restrict__ img, int64_t img_n,
                                            const double2* __restrict__ ipfx, const double2* __restrict__ tpfx,
                                            unsigned long long* __restrict__ keys,
                                            float* __restrict__ curve_out, AfterRead after_read) {
    constexpr int B = QB, NW = QNW, LB = QB, ROUNDS = kRounds, LAGS_PER_ROUND = kLagsPerRound;
    constexpr bool is_u8 = sizeof(S) == 1;
    constexpr float kSent = 2.0f;                          // screening value of a lag outside the query's range
    const float* img32 = reinterpret_cast<const float*>(img);
    const Buf& buf = sm.buf;
    const int lane = tid & 31, warp = tid >> 5;
    const QueryDesc& d = it.d;
    const int64_t j_blk = it.j_blk;
    const int64_t n = d.tlen;
    const int64_t jlo = d.lag0, jhi = d.lag0 + d.nlags;
    const double2 t_hi = tpfx[d.toff + n], t_lo = tpfx[d.toff];
    const double tsum = t_hi.x - t_lo.x, tsq = t_hi.y - t_lo.y;
    const double a = (double)Acc<S>::centre(ipfx[img_n].x, (double)img_n);
    const double b = (double)Acc<S>::centre(tsum, (double)n);
    const double n_ab = (double)n * a * b;
    const double scale = 1.0 / (double)(2 * B);
    const double k_const = a * tsum - n_ab;
    const float f_tsq = (float)tsq, f_b = (float)b, f_scale = (float)scale;
    const bool interior = j_blk >= jlo && j_blk + LB <= jhi;

    // chunk 1024c + 2tid + e = k1 + 16 k2 + 256 k3: k1 = 2(tid % 8) + e, k2 = (tid / 8) % 16, k3 = 4c + tid / 128; its
    // two halves r[k3][0], r[k3][1] are neighbours, and the twiddle W32^k3 = W32^(tid/128) * W8^c depends on the warp only
    const int ech = 2 * (tid & 7) * kDA + ((tid >> 3) & 15) * kDB + 2 * (tid >> 7);      // + kDA*e + 8*c; second half 1 further
    const float wc0 = kC32[tid >> 7], ws0 = kS32[tid >> 7];

    float vf[ROUNDS][8];
    float tmin = kSent;
    if (is_u8) mbar_wait(s_bar, bar_parity);
#pragma unroll
    for (int c = 0; c < ROUNDS; ++c) {
        const int m0 = c * LAGS_PER_ROUND + tid * 8;
        const int64_t j0 = j_blk + m0;
        const int64_t jw = j_blk + c * LAGS_PER_ROUND + warp * 256;
        if (jw >= jhi || jw + 256 <= jlo) {                            // no valid lag in this warp-round (warp-uniform)
#pragma unroll
            for (int i = 0; i < 8; ++i) vf[c][i] = kSent;
            continue;
        }
        // correlation at the 8 lags: last radix-2 step on chunks 1024c + 2tid + {0, 1}
        float cc[8];
        float wc = wc0, ws = ws0;                                      // W32^(tid/128) times exp(2*pi*i*c/8)
        {
            const float h = 0.70710678118654752f;
            if (c == 1) { wc = (wc0 - ws0) * h; ws = (wc0 + ws0) * h; }
            if (c == 2) { wc = -ws0; ws = wc0; }
            if (c == 3) { wc = -(wc0 + ws0) * h; ws = (wc0 - ws0) * h; }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const C2 E = buf.ld(ech + kDA * e + 8 * c), O = buf.ld(ech + kDA * e + 8 * c + 1);
            const float2 xr = fma2(O.r, bc(wc), fma2(O.i, bc(-ws), E.r));
            const float2 xi = fma2(O.r, bc(ws), fma2(O.i, bc(wc), E.i));
            cc[4 * e + 0] = xr.x; cc[4 * e + 1] = xi.x; cc[4 * e + 2] = xr.y; cc[4 * e + 3] = xi.y;
        }
        float f_w0q, f_k0;
        unsigned long long lo8 = 0, hi8 = 0;
        if (is_u8) {
            // everything comes from shared memory: lane l owns the run of 8 lags starting at jw + 8l.  Window
            // sums at the head of a run = exact warp base + exclusive intra-warp scan of the runs' integer totals
            const int hi_off = (int)((j_blk + n) & 15);
            lo8 = *reinterpret_cast<const unsigned long long*>(sm.lo + m0);
            const int hb = hi_off + m0;
            const unsigned long long h0 = *reinterpret_cast<const unsigned long long*>(sm.hi + (hb & ~7));
            const unsigned long long h1 = *reinterpret_cast<const unsigned long long*>(sm.hi + (hb & ~7) + 8);
            const unsigned sh = (unsigned)(hb & 7) * 8u;
            hi8 = sh ? ((h0 >> sh) | (h1 << (64u - sh))) : h0;
            const unsigned la = (unsigned)lo8, lb = (unsigned)(lo8 >> 32), ha = (unsigned)hi8, hb2 = (unsigned)(hi8 >> 32);
            const int tq = (int)__dp4a(ha, ha, __dp4a(hb2, hb2, 0u)) - (int)__dp4a(la, la, __dp4a(lb, lb, 0u));
            const int ts = (int)__dp4a(ha, 0x01010101u, __dp4a(hb2, 0x01010101u, 0u)) - (int)__dp4a(la, 0x01010101u, __dp4a(lb, 0x01010101u, 0u));
            int iq = tq, is = ts;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int uq = __shfl_up_sync(0xffffffffu, iq, o), us = __shfl_up_sync(0xffffffffu, is, o);
                if (lane >= o) { iq += uq; is += us; }
            }
            const double2 b_lo = sm.base[(c * NW + warp) * 2], b_hi = sm.base[(c * NW + warp) * 2 + 1];
            const double w0s = (b_hi.x - b_lo.x) + (double)(is - ts);
            const double w0q = (b_hi.y - b_lo.y) + (double)(iq - tq);
            f_w0q = (float)w0q;
            f_k0 = (float)(b * w0s + k_const);
        } else {
            if (!(j0 < jhi && j0 + 8 > jlo)) {
#pragma unroll
                for (int i = 0; i < 8; ++i) vf[c][i] = kSent;
                continue;
            }
            const double2 p_hi = ipfx[j0 + n], p_lo = ipfx[j0];
            f_w0q = (float)(p_hi.y - p_lo.y);
            f_k0 = (float)(b * (p_hi.x - p_lo.x) + k_const);
        }
        int rq = 0, rs = 0;              // uint8: exact integer slide
        double dq = 0.0, ds = 0.0;       // float32: fp64 slide
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float wq = f_w0q + (is_u8 ? (float)rq : (float)dq);
            const float sit = fmaf(cc[i], f_scale, fmaf(f_b, is_u8 ? (float)rs : (float)ds, f_k0));
            const float num = fmaxf((wq + f_tsq) - 2.0f * sit, 0.0f);
            const float pr = wq * f_tsq;
            // pr == 0 (silent window or template): rsqrt -> inf, num*inf -> inf or NaN, fminf(.,1) -> 1
            const float v = fminf(num * rsqrt_fast(pr), 1.0f);
            if (interior) { vf[c][i] = v; tmin = fminf(tmin, v); }
            else if (j0 + i >= jlo && j0 + i < jhi) { vf[c][i] = v; tmin = fminf(tmin, v); }
            else vf[c][i] = kSent;                                     // sentinel: not a valid lag
            if (is_u8) {
                const int lo = (int)((lo8 >> (8 * i)) & 0xffu), hi = (int)((hi8 >> (8 * i)) & 0xffu);
                rq += hi * hi - lo * lo; rs += hi - lo;
            } else if (j0 + i + n < img_n) {
                const double lo = (double)img32[j0 + i], hi = (double)img32[j0 + i + n];
                dq += hi * hi - lo * lo; ds += hi - lo;
            }
        }
    }
    const float my_min = tmin;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tmin = fminf(tmin, __shfl_xor_sync(0xffffffffu, tmin, o));
    if (lane == 0) s_min[warp] = tmin;
    if (is_u8) fence_proxy_async();   // window reads before the next item's TMA refill
    csync<ID>();
    after_read();
    float bmin = s_min[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) bmin = fminf(bmin, s_min[w]);
    const float thr = curve_out ? 1.5f : bmin + kScreenMargin;       // debug curve: evaluate everything

    unsigned long long cand = 0;
    if (my_min <= thr) {
#pragma unroll
        for (int c = 0; c < ROUNDS; ++c)
#pragma unroll
            for (int i = 0; i < 8; ++i) cand |= (vf[c][i] <= thr) ? (1ull << (c * 8 + i)) : 0ull;
    }
    unsigned long long best = ~0ull;
    while (cand) {
        const int bit = __ffsll((long long)cand) - 1;
        cand &= cand - 1;
        const int m = (bit >> 3) * LAGS_PER_ROUND + tid * 8 + (bit & 7);
        const int64_t j = j_blk + m;
        const int jj = m >> 2;                                          // chunk of X'
        const int ca = (jj & 15) * kDA + ((jj >> 4) & 15) * kDB + 2 * (jj >> 8);
        const C2 E = buf.ld(ca), O = buf.ld(ca + 1);
        const float2 w = make_float2(kC32[jj >> 8], kS32[jj >> 8]);
        const bool second = (m & 2) != 0;                               // lags 4j+2, 4j+3 belong to v
        const float er = second ? E.r.y : E.r.x, ei = second ? E.i.y : E.i.x, orr = second ? O.r.y : O.r.x, oi = second ? O.i.y : O.i.x;
        const float xr = fmaf(orr, w.x, fmaf(oi, -w.y, er)), xi = fmaf(orr, w.y, fmaf(oi, w.x, ei));
        const double cc = (double)((m & 1) ? xi : xr) * scale;
        const double2 p_hi = ipfx[j + n], p_lo = ipfx[j];
        const float v = sqdiff_exact(cc, p_hi.x - p_lo.x, p_hi.y - p_lo.y, a, b, tsum, tsq, n_ab);
        if (curve_out) curve_out[d.curveOff + (j - jlo)] = v;
        const unsigned long long key = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned int)(j - jlo);
        best = key < best ? key : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other < best ? other : best;
    }
    if (lane == 0) s_best[warp] = best;
    csync<ID>();
    if (tid == 0) {
        for (int w = 1; w < NW; ++w) best = s_best[w] < best ? s_best[w] : best;
        if (best != ~0ull) atomicMin(keys + it.q, best);
    }
}

// Body 3 (uint8 streams).  A thread owns the 32 consecutive lags 32*tid .. 32*tid+31 of the lag block as four runs of
// 8, a warp 1024 consecutive lags: ONE intra-warp scan per lag block gives every run its exact head sums (the first
// version scans once per round of 8 lags), and the chunks 8*tid .. 8*tid+7 of the transform's output sit in sixteen
// distinct banks per half warp (k1 = 8(tid%2) + i, k2 = (tid/2)%16, k3 = warp).  Per run: cmax = the largest correlation
// value, lower / upper bound of the run's screening values (see the comment at the bounds); block minimum of the
// upper bounds; the runs whose lower bound does not exceed it leave as records for k_finish_runs.  What cannot leave
// (no slot, degenerate block, debug curve) is screened per lag and evaluated exactly here, like the first version.
template <int ID, typename AfterRead>
__device__ __forceinline__ void finish_item_v3(const Item& it, int tid, const Smem& sm, unsigned long long* s_bar, unsigned bar_parity,
                                               float* s_min, int2* s_w0, int64_t img_n,
                                               unsigned long long* __restrict__ keys, float* __restrict__ curve_out,
                                               AfterRead after_read, RunSink sink) {
    constexpr int NW = QNW, LB = QB, RUNS = 4;
    constexpr float kSent = 3.0e38f;                       // bound / screening value of "no valid lag"
    const Buf& buf = sm.buf;
    const int lane = tid & 31, warp = tid >> 5;
    const QueryDesc& d = it.d;
    const int64_t j_blk = it.j_blk, n = d.tlen, jlo = d.lag0, jhi = d.lag0 + d.nlags;
    const double2* s_qc = reinterpret_cast<const double2*>(sm.end + kQueryConstOff());     // query_constants
    const double tsum = s_qc[0].x, tsq = s_qc[0].y, a = s_qc[1].x, b = s_qc[1].y;
    const double n_ab = (double)n * a * b;
    const double scale = 1.0 / (double)(2 * QB);
    const double k_const = a * tsum - n_ab;
    const float f_tsq = (float)tsq, f_b = (float)b;
    const float m2s = -2.0f * (float)scale, m2b = -2.0f * f_b;
    const bool interior = j_blk >= jlo && j_blk + LB <= jhi;
    const int64_t jt = j_blk + 32 * tid;                   // this thread's first lag
    // over the 8 lags of a run the window terms of the screening value, rq_i - 2b*rs_i = sum over the samples that
    // left / entered the window of (hi - b)^2 - (lo - b)^2, move by at most 7 * max(b, 255 - b)^2 (f_delta, with 2 % and
    // 1024 on top: that swallows every fp32 rounding); the window energy itself by at most kRunQ
    constexpr float kRunQ = 7.0f * 255.0f * 255.0f;
    const float f_bm = fmaxf(f_b, 255.0f - f_b);
    const float f_delta = 1.02f * 7.0f * f_bm * f_bm + 1024.0f;
    const float rt = sqrtf(f_tsq), m_rt = kScreenMargin * rt, sat = (1.0f - kScreenMargin) * rt;
    const int ech = 8 * (tid & 1) * kDA + ((tid >> 1) & 15) * kDB + 2 * warp;            // chunk 8*tid + i: + kDA*i; its second half 1 further
    const float wc = kC32[warp], ws = kS32[warp];                                        // W32^k3, k3 = warp

    mbar_wait(s_bar, bar_parity);
    // ---- the 32 + 32 window bytes of this thread, the runs' integer totals, one scan
    unsigned lw[8], hw[8];
    {
        const uint4 l0 = *reinterpret_cast<const uint4*>(sm.lo + 32 * tid), l1 = *reinterpret_cast<const uint4*>(sm.lo + 32 * tid + 16);
        lw[0] = l0.x; lw[1] = l0.y; lw[2] = l0.z; lw[3] = l0.w; lw[4] = l1.x; lw[5] = l1.y; lw[6] = l1.z; lw[7] = l1.w;
        const int hi_off = (int)((j_blk + n) & 15);       // the staged copy starts at the 16-byte boundary below j_blk + n
        const uint4 h0 = *reinterpret_cast<const uint4*>(sm.hi + 32 * tid), h1 = *reinterpret_cast<const uint4*>(sm.hi + 32 * tid + 16),
                    h2 = *reinterpret_cast<const uint4*>(sm.hi + 32 * tid + 32);
        unsigned w[12] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w, h2.x, h2.y, h2.z, h2.w};
        unsigned v[10], u[9];
#pragma unroll
        for (int k = 0; k < 10; ++k) v[k] = (hi_off & 8) ? w[k + 2] : w[k];
#pragma unroll
        for (int k = 0; k < 9; ++k) u[k] = (hi_off & 4) ? v[k + 1] : v[k];
        const unsigned sh = (unsigned)(hi_off & 3) * 8u;
#pragma unroll
        for (int k = 0; k < 8; ++k) hw[k] = __funnelshift_r(u[k], u[k + 1], sh);
    }
    int tq[RUNS], ts[RUNS];
#pragma unroll
    for (int r = 0; r < RUNS; ++r) {
        tq[r] = (int)__dp4a(hw[2 * r], hw[2 * r], __dp4a(hw[2 * r + 1], hw[2 * r + 1], 0u)) - (int)__dp4a(lw[2 * r], lw[2 * r], __dp4a(lw[2 * r + 1], lw[2 * r + 1], 0u));
        ts[r] = (int)__dp4a(hw[2 * r], 0x01010101u, __dp4a(hw[2 * r + 1], 0x01010101u, 0u)) - (int)__dp4a(lw[2 * r], 0x01010101u, __dp4a(lw[2 * r + 1], 0x01010101u, 0u));
    }
    const int Tq = (tq[0] + tq[1]) + (tq[2] + tq[3]), Ts = (ts[0] + ts[1]) + (ts[2] + ts[3]);
    int iq = Tq, is = Ts;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int uq = __shfl_up_sync(0xffffffffu, iq, o), us = __shfl_up_sync(0xffffffffu, is, o);
        if (lane >= o) { iq += uq; is += us; }
    }
    // exact sums of the window at the warp's first lag (staged from the running sums), everything else as integer offsets
    const double2 b_lo = sm.base[warp * 2], b_hi = sm.base[warp * 2 + 1];
    const double Wq = b_hi.y - b_lo.y, Ws = b_hi.x - b_lo.x;
    const double Cw = Wq + tsq - 2.0 * (b * Ws + k_const);             // A at the warp's first lag
    const int bi2 = 2 * (int)b;                                          // b is an integer (Acc<uint8_t>::centre)
    float run_lb[RUNS];
    float tmin = kSent;
    int oq = iq - Tq, os = is - Ts;                                      // offsets of the run's head from the warp's first lag
#pragma unroll
    for (int r = 0; r < RUNS; ++r) {
        s_w0[r * QT + tid] = make_int2(os, oq);                          // for the in-kernel paths below
        // the 0.25 keeps a silent window (sum of squares 0) finite under rsqrt; it is below one ulp of any
        // window sum that is not within 8 samples of silence
        const float f_w0q = (float)(Wq + 0.25 + (double)oq);
        const float f_A = (float)(Cw + (double)(oq - bi2 * os));
        // correlation at the run's 8 lags: last radix-2 step on chunks 8*tid + 2r, + 1
        float cc[8];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const C2 E = buf.ld(ech + kDA * (2 * r + e)), O = buf.ld(ech + kDA * (2 * r + e) + 1);
            const float2 xr = fma2(O.r, bc(wc), fma2(O.i, bc(-ws), E.r));
            const float2 xi = fma2(O.r, bc(ws), fma2(O.i, bc(wc), E.i));
            cc[4 * e + 0] = xr.x; cc[4 * e + 1] = xi.x; cc[4 * e + 2] = xr.y; cc[4 * e + 3] = xi.y;
        }
        // Run-level bounds.  The screening value of lag i of this run is
        //   v'_i = (A + rq_i - 2b*rs_i - 2*scale*cc_i) * rsqrt(w0q + rq_i),   |rq_i - 2b*rs_i| <= delta, |rq_i| <= kRunQ,
        // so with cmax = max cc_i:   v'_i >= (A - delta - 2*scale*cmax) * rsqrt(w0q + kRunQ)   for every i  (lower bound), and
        // at the lag of cmax          v'   <= (A + delta - 2*scale*cmax) * rsqrt(w0q - kRunQ)                  (upper bound).
        // The block minimum of the upper bounds is an upper bound of the block's smallest screening value: only runs
        // whose lower bound does not exceed it (plus the margin) can hold a candidate.
        const float cmax = fmaxf(fmaxf(fmaxf(cc[0], cc[1]), fmaxf(cc[2], cc[3])), fmaxf(fmaxf(cc[4], cc[5]), fmaxf(cc[6], cc[7])));
        const int64_t j0 = jt + 8 * r;
        const bool some = interior || (j0 < jhi && j0 + 8 > jlo);          // the run has a lag of the range
        const bool inside = interior || (j0 >= jlo && j0 + 8 <= jhi);      // all of its lags are
        const float lbn = fmaf(cmax, m2s, f_A - f_delta), ubn = lbn + 2.0f * f_delta;
        const float lbv = lbn * rsqrt_fast(f_w0q + kRunQ) * 0.999999f;
        run_lb[r] = !some ? kSent : (lbn >= 0.f ? lbv : -kSent);
        const float ubv = ubn * rsqrt_fast(f_w0q - kRunQ) * 1.000001f;
        if (inside && f_w0q > 4.0f * kRunQ && ubn >= 0.f) tmin = fminf(tmin, ubv);
        oq += tq[r]; os += ts[r];
    }
    // ---- block minimum of the upper bounds
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tmin = fminf(tmin, __shfl_xor_sync(0xffffffffu, tmin, o));
    if (lane == 0) s_min[warp] = tmin;
    fence_proxy_async();              // window reads before the next item's TMA refill
    csync<ID>();
    static_assert(NW == 16, "block minimum over 16 warps");
    float bmin = s_min[lane & (NW - 1)];
#pragma unroll
    for (int o = NW / 2; o > 0; o >>= 1) bmin = fminf(bmin, __shfl_xor_sync(0xffffffffu, bmin, o));
    // a block whose minimum is (nearly) saturated -- silence, a zero template, no usable upper bound at all -- and the
    // debug curve evaluate every lag of the range in the kernel
    const float thr = bmin + m_rt;
    const bool all = curve_out != nullptr || !(bmin < sat);
    unsigned left = 0;                // runs of this thread that still need the in-kernel path
#pragma unroll
    for (int r = 0; r < RUNS; ++r) left |= (run_lb[r] <= thr || (all && run_lb[r] < kSent)) ? (1u << r) : 0u;
    // the selected runs leave as records (see RunRecord); what finds no slot stays selected
    if (left && sink.recs != nullptr && !all) {
#pragma unroll 1
        for (int r = 0; r < RUNS; ++r) {
            if (!((left >> r) & 1u)) continue;
            const int slot = atomicAdd(sink.s_cnt, 1);
            if (slot >= kRunSlots) break;
            float cc[8];
            const int k3 = warp;
#pragma unroll
            for (int e = 0; e < 2; ++e) {       // exactly as the exact path below forms them
                const C2 E = buf.ld(ech + kDA * (2 * r + e)), O = buf.ld(ech + kDA * (2 * r + e) + 1);
                const float2 w = make_float2(kC32[k3], kS32[k3]);
                const float2 xr = fma2(O.r, bc(w.x), fma2(O.i, bc(-w.y), E.r));
                const float2 xi = fma2(O.r, bc(w.y), fma2(O.i, bc(w.x), E.i));
                cc[4 * e + 0] = xr.x; cc[4 * e + 1] = xi.x; cc[4 * e + 2] = xr.y; cc[4 * e + 3] = xi.y;
            }
            float4* r4 = reinterpret_cast<float4*>(sink.recs + slot);
            const int64_t j0 = jt + 8 * r;
            *reinterpret_cast<int4*>(r4) = make_int4(it.q, 1, (int)(unsigned)(j0 & 0xffffffffll), (int)(j0 >> 32));
            r4[1] = make_float4(cc[0], cc[1], cc[2], cc[3]);
            r4[2] = make_float4(cc[4], cc[5], cc[6], cc[7]);
            left &= ~(1u << r);
        }
    }
    unsigned long long best = ~0ull;
    if (__any_sync(0xffffffffu, left != 0u)) {
        // per-lag screening of the runs that stayed (rare), everything re-read from shared memory; within a warp the
        // warp's own smallest value tightens the threshold; then the exact fp64 evaluation of the candidates
        unsigned cand = 0;            // bit 8r + i
#pragma unroll 1
        for (int r = 0; r < RUNS; ++r) {
            const bool sel = (left >> r) & 1u;
            if (!__any_sync(0xffffffffu, sel)) continue;
            const int64_t j0 = jt + 8 * r;
            float cc[8];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const C2 E = buf.ld(ech + kDA * (2 * r + e)), O = buf.ld(ech + kDA * (2 * r + e) + 1);
                const float2 xr = fma2(O.r, bc(wc), fma2(O.i, bc(-ws), E.r));
                const float2 xi = fma2(O.r, bc(ws), fma2(O.i, bc(wc), E.i));
                cc[4 * e + 0] = xr.x; cc[4 * e + 1] = xi.x; cc[4 * e + 2] = xr.y; cc[4 * e + 3] = xi.y;
            }
            const unsigned long long lo8 = *reinterpret_cast<const unsigned long long*>(sm.lo + 32 * tid + 8 * r);
            const int hb = (int)((j_blk + n) & 15) + 32 * tid + 8 * r;
            const unsigned long long h0 = *reinterpret_cast<const unsigned long long*>(sm.hi + (hb & ~7));
            const unsigned long long h1 = *reinterpret_cast<const unsigned long long*>(sm.hi + (hb & ~7) + 8);
            const unsigned shb = (unsigned)(hb & 7) * 8u;
            const unsigned long long hi8 = shb ? ((h0 >> shb) | (h1 << (64u - shb))) : h0;
            const int2 off = s_w0[r * QT + tid];
            const float f_w0q = (float)(Wq + 0.25 + (double)off.y);
            const float f_A = (float)(Cw + (double)(off.y - bi2 * off.x));
            float v8[8];
            float vmin = kSent;
            int rq = 0, rs = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float frq = (float)rq;
                const float num = fmaf(cc[i], m2s, fmaf(m2b, (float)rs, f_A + frq));
                const float v = num * rsqrt_fast(f_w0q + frq);
                const bool valid = sel && j0 + i >= jlo && j0 + i < jhi;
                v8[i] = valid ? v : kSent;
                vmin = fminf(vmin, v8[i]);
                const int lo = (int)((lo8 >> (8 * i)) & 0xffu), hi = (int)((hi8 >> (8 * i)) & 0xffu);
                const int dd = hi - lo;
                rq += (hi + lo) * dd; rs += dd;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
            const float thrw = fminf(thr, vmin + m_rt);
#pragma unroll
            for (int i = 0; i < 8; ++i) cand |= (v8[i] < kSent && (v8[i] <= thrw || all)) ? (1u << (r * 8 + i)) : 0u;   // (a block without a usable upper bound has thr = kSent)
        }
        while (cand) {
            const int bit = __ffs((int)cand) - 1;
            cand &= cand - 1;
            const int r = bit >> 3, i = bit & 7;
            const int m = 32 * tid + bit;
            const int64_t j = j_blk + m;
            const int jj = m >> 2;                                          // chunk of X'
            const int ca = (jj & 15) * kDA + ((jj >> 4) & 15) * kDB + 2 * (jj >> 8);
            const C2 E = buf.ld(ca), O = buf.ld(ca + 1);
            const float2 w = make_float2(kC32[jj >> 8], kS32[jj >> 8]);
            const bool second = (m & 2) != 0;                               // lags 4j+2, 4j+3 belong to v
            const float er = second ? E.r.y : E.r.x, ei = second ? E.i.y : E.i.x, orr = second ? O.r.y : O.r.x, oi = second ? O.i.y : O.i.x;
            const float xr = fmaf(orr, w.x, fmaf(oi, -w.y, er)), xi = fmaf(orr, w.y, fmaf(oi, w.x, ei));
            const double cc = (double)((m & 1) ? xi : xr) * scale;
            // exact window sums without touching HBM: the run's head sums plus the integer slide over the first i samples
            const unsigned long long lo8 = *reinterpret_cast<const unsigned long long*>(sm.lo + 32 * tid + 8 * r);
            const int hb = (int)((j_blk + n) & 15) + 32 * tid + 8 * r;
            const unsigned long long h0 = *reinterpret_cast<const unsigned long long*>(sm.hi + (hb & ~7));
            const unsigned long long h1 = *reinterpret_cast<const unsigned long long*>(sm.hi + (hb & ~7) + 8);
            const unsigned shb = (unsigned)(hb & 7) * 8u;
            const unsigned long long hi8 = shb ? ((h0 >> shb) | (h1 << (64u - shb))) : h0;
            const unsigned long long keep = i ? (~0ull >> (8 * (8 - i))) : 0ull;      // samples 0 .. i-1
            const unsigned la = (unsigned)(lo8 & keep), lb = (unsigned)((lo8 & keep) >> 32), ha = (unsigned)(hi8 & keep), hb2 = (unsigned)((hi8 & keep) >> 32);
            const int rq = (int)__dp4a(ha, ha, __dp4a(hb2, hb2, 0u)) - (int)__dp4a(la, la, __dp4a(lb, lb, 0u));
            const int rs = (int)__dp4a(ha, 0x01010101u, __dp4a(hb2, 0x01010101u, 0u)) - (int)__dp4a(la, 0x01010101u, __dp4a(lb, 0x01010101u, 0u));
            const int2 off = s_w0[r * QT + tid];
            const double wsum = (Ws + (double)off.x) + (double)rs, wsq = (Wq + (double)off.y) + (double)rq;
            const float v = sqdiff_exact(cc, wsum, wsq, a, b, tsum, tsq, n_ab);
            if (curve_out) curve_out[d.curveOff + (j - jlo)] = v;
            const unsigned long long key = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned int)(j - jlo);
            best = key < best ? key : best;
        }
        if (best != ~0ull) atomicMin(keys + it.q, best);
    }
    fence_proxy_async();              // the in-kernel paths' window reads, again before the refill
    csync<ID>();                      // everyone is done with the FFT buffer and the staged windows
    after_read();
}

// Multi-stream calls: the streams of query q (processing order) from the call's stream table -- image slot .x, template
// slot .y -- in place of the kernel's stream arguments.
template <typename S> struct QueryStreams { const float4* Xhat; int64_t nblk; const S* img; int64_t img_n; const double2* ipfx; const double2* tpfx; };
template <typename S>
__device__ __forceinline__ QueryStreams<S> select_streams(const StreamEntry* streams, const int2* slots, int q) {
    const int2 sl = slots[q];
    const StreamEntry si = streams[sl.x];
    return {reinterpret_cast<const float4*>(si.specq), si.nblk, static_cast<const S*>(si.raw), si.n, si.pfx, streams[sl.y].pfx};
}
#define SB_SELECT_STREAMS(q) do { const QueryStreams<S> qs__ = select_streams<S>(streams, slots, (q)); \
    Xhat = qs__.Xhat; nblk = qs__.nblk; img = qs__.img; img_n = qs__.img_n; ipfx = qs__.ipfx; tpfx = qs__.tpfx; } while (0)

// ---------------------------------------------------------------- kernel A: one CTA per item
template <typename S, int EPI, bool MULTI = false>
__global__ void __launch_bounds__(QT, 1)
k_match_packed(const float4* __restrict__ That, int64_t part_first,
               const float4* __restrict__ Xhat, int64_t nblk,
               const S* __restrict__ img, int64_t img_n,
               const double2* __restrict__ ipfx, const double2* __restrict__ tpfx,
               const QueryDesc* __restrict__ desc, const int* __restrict__ item_query, int64_t item_first,
               PackedTables tab, unsigned long long* __restrict__ keys, float* __restrict__ curve_out,
               RunRecord* __restrict__ recs, int* __restrict__ rec_count,
               const StreamEntry* __restrict__ streams = nullptr, const int2* __restrict__ slots = nullptr) {
    constexpr int T = QT, NW = QNW;
    constexpr bool is_u8 = sizeof(S) == 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const Smem sm(smem_raw);
    unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(sm.end);
    unsigned long long* s_best = s_bar + 1;                                // [NW]
    float* s_min = reinterpret_cast<float*>(s_best + NW);                  // [NW]
    int* s_cnt = reinterpret_cast<int*>(sm.end + kRunCountOff());          // EPI 3: records written by this CTA
    const RunSink sink = {EPI == 3 && recs ? recs + (size_t)blockIdx.x * kRunSlots : nullptr, s_cnt};
    float4* s_sp = reinterpret_cast<float4*>(sm.end + kSmallBytes);        // body 3: units of the self-mirrored quads
    int2* s_w0 = EPI >= 2 && is_u8 ? reinterpret_cast<int2*>(sm.end + kSmallBytes + kSpecialBytes) : nullptr;   // [kRounds][QT]
    const Buf& buf = sm.buf;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const Item it(desc, item_query, item_first, blockIdx.x);
    const QueryDesc& d = it.d;
    if constexpr (MULTI) SB_SELECT_STREAMS(it.q);

    // ---------------- 0. stage what the epilogue needs; the latency hides behind the MAC and the FFT
    if (is_u8) {
        if (tid == 0) mbar_init(s_bar, 1);
        stage_inputs<EPI == 3>(it, tid, reinterpret_cast<const uint8_t*>(img), img_n, ipfx, sm, s_bar);
    }
    if (EPI == 3 && tid == 96) *s_cnt = 0;
    if (EPI >= 2 && tid == 64) query_constants<S>(reinterpret_cast<double2*>(sm.end + kQueryConstOff()), d, img_n, ipfx, tpfx);

    // ---------------- 1+2. spectral multiply-accumulate, packing, first radix-2 step --------
    {
        int P = d.P;
        if (it.k + P > nblk) P = (int)(nblk - it.k);      // rows past the end of the stream are zero
        typedef Rows R;
        const float4* tp = That + (d.partBase - part_first) * (int64_t)R::STRIDE;
        const float4* xp = Xhat + it.k * (int64_t)R::STRIDE;
        const float2 wbase = __ldg(tab.wb + tid);
        const int tm = (T - tid) & (T - 1);           // mirrored chunks C[B/2 - i] live in thread tm's column
        const int col = phys(tid), mcol = phys(tm);
        const bool sp_pref = EPI >= 2 && SB_V2_SPECIAL_PREFETCH && special_fits(d.P, 1);
        if (sp_pref && warp == NW - 1) special_prefetch(s_sp, tp, xp, d.P, 1, it.k, nblk, lane);
        constexpr int U = 4;                          // quads in flight per thread
#pragma unroll 1
        for (int half = 0; half < 2; ++half) {
            const int i0 = R::unit(tid, half * U);    // unit of quad tid + 512*(half*U + u) = i0 + u*USTEP
            QuadAcc acc[U];
#pragma unroll
            for (int u = 0; u < U; ++u) acc[u].zero();
#pragma unroll 1
            for (int p = 0; p < P; ++p) {
                const float4* t = tp + (int64_t)p * R::STRIDE;
                const float4* x = xp + (int64_t)p * R::STRIDE;
                float4 ta[U], tmm[U], xa[U], xm[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    R::load(t, i0 + u * R::USTEP, ta[u], tmm[u]);
                    R::load(x, i0 + u * R::USTEP, xa[u], xm[u]);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) acc[u].mac(ta[u], tmm[u], xa[u], xm[u]);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int uu = half * U + u;          // i = tid + 512*uu
                const float c = wbase.x * kC64[uu] - wbase.y * kS64[uu];
                const float s = wbase.x * kS64[uu] + wbase.y * kC64[uu];
                C2 lo, hi;
                pack_quad(acc[u].aR, acc[u].aI, acc[u].mR, acc[u].mI, c, s, lo, hi);
                buf.st(col + kUU * uu, lo);                       // C[i]
                // C[B/2 - i]: chunk (T - tid) + 512*(15 - uu), or 512*(16 - uu) for tid = 0 (none for i = 0)
                if (tid != 0) buf.st(mcol + kUU * (15 - uu), hi);
                else if (uu != 0) buf.st(mcol + kUU * (16 - uu), hi);
            }
        }
        if (warp == NW - 1) {                       // the self-mirrored quad i = B/4
            if (sp_pref) {
                cp_async_commit_wait_all();
                __syncwarp();
                const C2 lo = special_from_smem(s_sp, d.P, 0, lane);
                if (lane == 0) buf.st(phys(Q4), lo);
            } else {
                const C2 lo = special_quad(tp, xp, P, lane);
                if (lane == 0) buf.st(phys(Q4), lo);
            }
        }
    }
    csync<0>();

    // ---------------- 3. inverse FFT, 4. epilogue ---------------------------------------------
    fft_passes_dif<0>(buf, tid, tab, is_u8);
    if constexpr (EPI == 3) finish_item_v3<0>(it, tid, sm, s_bar, 0u, s_min, s_w0, img_n, keys, curve_out, [] {}, sink);
    else finish_item<S, 0>(it, tid, sm, s_bar, 0u, s_best, s_min, img, img_n, ipfx, tpfx, keys, curve_out, [] {});
    if (EPI == 3 && rec_count && tid == 0) rec_count[blockIdx.x] = *s_cnt < kRunSlots ? *s_cnt : kRunSlots;    // behind the closing barrier of finish_item
}

// The park of one CTA: [2 * uu + h][QT] float4, h = 0 for the chunk C[i], 1 for C[B/2 - i] (i = tid + 512*uu), so
// a warp's store or load of one (uu, h) is 512 contiguous bytes.
constexpr int kParkF4 = 16 * QT;

// A parked product spectrum back into the FFT buffer: this thread's 16 park entries hold, quad by quad, the chunks
// C[i] and C[B/2 - i] it packed.
__device__ __forceinline__ void unpark(const float4* pk, const Buf& buf, int col, int mcol, int tid) {
#pragma unroll
    for (int uu = 0; uu < 8; ++uu) {
        const C2 lo = from4(park_ld(pk + (2 * uu) * QT)), hi = from4(park_ld(pk + (2 * uu + 1) * QT));
        buf.st(col + kUU * uu, lo);
        if (tid != 0) buf.st(mcol + kUU * (15 - uu), hi);
        else if (uu != 0) buf.st(mcol + kUU * (16 - uu), hi);
    }
}

// ---------------------------------------------------------------- kernel A2: one CTA per PAIR of lag blocks
// The multiply phase of k_match_packed runs at the SM's L2 read rate (each item pulls 2 x P rows of 131 KB).
// Two consecutive lag blocks k, k+1 of one query use the same template rows T^_p and overlapping spectrum rows
// (block k+1 at step p needs X^_{k+1+p}, which block k needs at step p+1): multiplying both at once costs
// 2P + 1 row reads instead of 4P.  The second product spectrum (128 KB) has nowhere to wait in shared memory
// (the FFT buffer and the epilogue's arrays take 170-188 KB of the 227 KB), so it is parked in global memory:
// one 128 KB slot per resident CTA (park_acquire), written and read with L2-only accesses, which L2 keeps
// (132 slots = 17 MB of the 50 MB).  Every thread reads back exactly what it wrote, so the park needs no barrier.
template <typename S, int EPI, bool MULTI = false>
__global__ void __launch_bounds__(QT, 1)
k_match_pair(const float4* __restrict__ That, int64_t part_first,
             const float4* __restrict__ Xhat, int64_t nblk,
             const S* __restrict__ img, int64_t img_n,
             const double2* __restrict__ ipfx, const double2* __restrict__ tpfx,
             const QueryDesc* __restrict__ desc, const int* __restrict__ pair_query, int64_t pair_first, int64_t n_pairs,
             float4* __restrict__ park, int* __restrict__ park_busy, int park_slots,
             PackedTables tab, unsigned long long* __restrict__ keys, float* __restrict__ curve_out,
             RunRecord* __restrict__ recs, int* __restrict__ rec_count,
             const StreamEntry* __restrict__ streams = nullptr, const int2* __restrict__ slots = nullptr) {
    constexpr int T = QT, NW = QNW;
    constexpr bool is_u8 = sizeof(S) == 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const Smem sm(smem_raw);
    unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(sm.end);
    unsigned long long* s_best = s_bar + 1;                                // [NW]
    float* s_min = reinterpret_cast<float*>(s_best + NW);                  // [NW]
    int* s_slot = reinterpret_cast<int*>(s_min + NW);                       // park slot of this CTA
    int* s_cnt = reinterpret_cast<int*>(sm.end + kRunCountOff());          // EPI 3: records written for the current pair (both items)
    int* s_next_q = reinterpret_cast<int*>(sm.end + kNextOff());           // query of the CTA's next pair ...
    QueryDesc* s_next_d = reinterpret_cast<QueryDesc*>(sm.end + kNextOff() + 16);     // ... and its descriptor (fetched during this pair)
    float4* s_sp = reinterpret_cast<float4*>(sm.end + kSmallBytes);        // body 3: units of the self-mirrored quads
    int2* s_w0 = EPI >= 2 && is_u8 ? reinterpret_cast<int2*>(sm.end + kSmallBytes + kSpecialBytes) : nullptr;   // [kRounds][QT]
    const Buf& buf = sm.buf;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // The kernel is persistent: a CTA walks the pairs blockIdx.x, blockIdx.x + gridDim.x, ... (the launcher starts one
    // CTA per SM).  The park slot, the barrier and the per-thread constants are set up once; the descriptor of the
    // next pair is fetched while this one is transformed, so no pair but the first starts with two dependent global
    // reads.
    if (tid == 64) *s_slot = park_acquire(park_busy, park_slots, (int)(blockIdx.x % (unsigned)park_slots));
    if (is_u8 && tid == 0) mbar_init(s_bar, 1);
    if (EPI == 3 && tid == 32) *s_cnt = 0;
    csync<0>();
    float4* const pk = park + (size_t)*s_slot * kParkF4 + tid;      // this thread's entries, QT float4 apart
    const int tm = (T - tid) & (T - 1);               // mirrored chunks C[B/2 - i] live in thread tm's column
    const int col = phys(tid), mcol = phys(tm);
    const float2 wbase = __ldg(tab.wb + tid);
    unsigned phase = 0;                               // completed phases of s_bar (one per staged item)

    // (body 3 only: the first-version instantiations sit at the register limit -- carrying the loop's state across a
    // pair makes them spill -- and keep one CTA per pair; their launcher starts n_pairs CTAs)
    constexpr bool kPersistent = EPI == 3, kPrefetch = kPersistent;
    int64_t pi = blockIdx.x;                          // the grid never exceeds n_pairs
    do {                                              // uniform over the CTA
    const bool first = !kPrefetch || pi == (int64_t)blockIdx.x;
    const int q = first ? __ldg(pair_query + pi) : *s_next_q;
    const QueryDesc d = first ? desc[q] : *s_next_d;
    // a CTA's walk crosses query boundaries, and with them stream boundaries: every pair reads its query's entries
    if constexpr (MULTI) SB_SELECT_STREAMS(q);
    const int64_t pi_next = pi + gridDim.x;
    int q_next = 0;
    if (kPrefetch && tid == 32 && pi_next < n_pairs) q_next = __ldg(pair_query + pi_next);      // used after the multiply phase: no wait here
    const int lp = (int)(pair_first + pi - d.groupBase);                  // pair number inside the query
    const bool has2 = 2 * lp + 1 < d.nk;
    const Item it0(d, q, d.k0 + 2 * lp), it1(d, q, d.k0 + 2 * lp + 1);
    const RunSink sink = {EPI == 3 && recs ? recs + (size_t)pi * kRunSlots : nullptr, s_cnt};

    if (is_u8) stage_inputs<EPI == 3>(it0, tid, reinterpret_cast<const uint8_t*>(img), img_n, ipfx, sm, s_bar);
    if (EPI >= 2 && tid == 64) query_constants<S>(reinterpret_cast<double2*>(sm.end + kQueryConstOff()), d, img_n, ipfx, tpfx);
    C2 sp1 = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};             // C[B/4] of the second item (warp NW-1, lane 0)
    // ---------------- 1+2. multiply-accumulate for both items, packing, first radix-2 step ----
    {
        typedef Rows R;
        const int64_t k = it0.k;
        const float4* tp = That + (d.partBase - part_first) * (int64_t)R::STRIDE;
        const float4* xp = Xhat + k * (int64_t)R::STRIDE;
        const bool sp_pref = EPI >= 2 && SB_V2_SPECIAL_PREFETCH && special_fits(d.P, 2);
        if (sp_pref && warp == NW - 1) special_prefetch(s_sp, tp, xp, d.P, 2, k, nblk, lane);
        constexpr int U = 2;                          // quads in flight per thread (two accumulator sets each)
#pragma unroll 1
        for (int grp = 0; grp < 8 / U; ++grp) {
            const int i0 = R::unit(tid, grp * U);     // unit of quad tid + 512*(grp*U + u) = i0 + u*USTEP
            QuadAcc a0[U], a1[U];
            float4 xa[U], xm[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                a0[u].zero(); a1[u].zero();
                R::load(xp, i0 + u * R::USTEP, xa[u], xm[u]);     // row k < nblk
            }
#pragma unroll 2                               // two partition steps in flight
            for (int p = 0; p < d.P; ++p) {
                const float4* t = tp + (int64_t)p * R::STRIDE;
                const float4* x = xp + (int64_t)(p + 1) * R::STRIDE;
                const bool next_row = k + p + 1 < nblk;           // rows past the end of the stream are zero
                float4 ta[U], tmm[U], xna[U], xnm[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    R::load(t, i0 + u * R::USTEP, ta[u], tmm[u]);
                    R::loadp(x, i0 + u * R::USTEP, next_row, xna[u], xnm[u]);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    a0[u].mac(ta[u], tmm[u], xa[u], xm[u]);       // block k   : row k + p
                    a1[u].mac(ta[u], tmm[u], xna[u], xnm[u]);     // block k+1 : row k + 1 + p
                    xa[u] = xna[u]; xm[u] = xnm[u];
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int uu = grp * U + u;           // i = tid + 512*uu
                const float c = wbase.x * kC64[uu] - wbase.y * kS64[uu];
                const float s = wbase.x * kS64[uu] + wbase.y * kC64[uu];
                C2 lo, hi;
                pack_quad(a0[u].aR, a0[u].aI, a0[u].mR, a0[u].mI, c, s, lo, hi);
                buf.st(col + kUU * uu, lo);                       // C[i]
                if (tid != 0) buf.st(mcol + kUU * (15 - uu), hi); // C[B/2 - i]
                else if (uu != 0) buf.st(mcol + kUU * (16 - uu), hi);
                pack_quad(a1[u].aR, a1[u].aI, a1[u].mR, a1[u].mI, c, s, lo, hi);
                park_st(pk + (2 * uu) * QT, make_float4(lo.r.x, lo.r.y, lo.i.x, lo.i.y));
                park_st(pk + (2 * uu + 1) * QT, make_float4(hi.r.x, hi.r.y, hi.i.x, hi.i.y));
            }
        }
        if (warp == NW - 1) {                         // the self-mirrored quad i = B/4 of both items
            if (sp_pref) {
                cp_async_commit_wait_all();
                __syncwarp();
                const C2 lo = special_from_smem(s_sp, d.P, 0, lane);
                if (lane == 0) buf.st(phys(Q4), lo);
                if (has2) sp1 = special_from_smem(s_sp, d.P, 1, lane);
            } else {
                int P0 = d.P; if (k + P0 > nblk) P0 = (int)(nblk - k);
                const C2 lo = special_quad(tp, xp, P0, lane);
                if (lane == 0) buf.st(phys(Q4), lo);
                if (has2) {
                    int P1 = d.P; if (k + 1 + P1 > nblk) P1 = (int)(nblk - k - 1);
                    sp1 = special_quad(tp, xp + R::STRIDE, P1, lane);
                }
            }
        }
    }
    csync<0>();
    // the next pair's descriptor travels while this pair is transformed (every reader of the slot is past the barrier)
    if (kPrefetch && tid == 32 && pi_next < n_pairs) {
        *s_next_q = q_next;
        const float4* src = reinterpret_cast<const float4*>(desc + q_next);
        static_assert(sizeof(QueryDesc) == 80, "five 16-byte copies");
#pragma unroll
        for (int k = 0; k < 5; ++k) cp_async16(reinterpret_cast<float4*>(s_next_d) + k, src + k);
    }

    // ---------------- first item: inverse FFT + epilogue ---------------------------------------
    fft_passes_dif<0>(buf, tid, tab, true);          // drains this thread's asynchronous copies in front of its last barrier
    auto stage_second = [&] { if (is_u8 && has2) stage_inputs<EPI == 3>(it1, tid, reinterpret_cast<const uint8_t*>(img), img_n, ipfx, sm, s_bar); };
    if constexpr (EPI == 3) finish_item_v3<0>(it0, tid, sm, s_bar, phase & 1u, s_min, s_w0, img_n, keys, curve_out, stage_second, sink);
    else finish_item<S, 0>(it0, tid, sm, s_bar, phase & 1u, s_best, s_min, img, img_n, ipfx, tpfx, keys, curve_out, stage_second);
    ++phase;

    // ---------------- second item: out of the park, then the same ---------------------------------
    if (has2) {                                       // uniform over the CTA
        unpark(pk, buf, col, mcol, tid);
        if (tid == (NW - 1) * 32) buf.st(phys(Q4), sp1);
        csync<0>();
        fft_passes_dif<0>(buf, tid, tab, is_u8);
        if constexpr (EPI == 3) finish_item_v3<0>(it1, tid, sm, s_bar, phase & 1u, s_min, s_w0, img_n, keys, curve_out, [] {}, sink);
        else finish_item<S, 0>(it1, tid, sm, s_bar, phase & 1u, s_best, s_min, img, img_n, ipfx, tpfx, keys, curve_out, [] {});
        ++phase;
    }
    // end of the pair (behind the closing barrier of the last epilogue, which also separates this pair's readers of the
    // shared arrays from the next pair's writers): the record count leaves.  The next descriptor became visible with
    // the barrier that ended the first transform (thread 32 drained its copies in front of it).
    if (EPI == 3 && rec_count && tid == 32) { rec_count[pi] = *s_cnt < kRunSlots ? *s_cnt : kRunSlots; *s_cnt = 0; }
    } while (kPersistent && (pi += gridDim.x) < n_pairs);   // pairs of this CTA
    csync<0>();
    if (tid == 64) park_release(park_busy + *s_slot);
}

// EPI 3, second step: one thread per record slot evaluates the 8 lags of its run exactly (fp64) and merges the best
// into the query's key -- the arithmetic of finish_item's exact path, with the window sums taken from the running
// sums (for uint8 streams the same exact integers the match kernel slides on its staged bytes).
template <typename S, bool MULTI = false>
__global__ void __launch_bounds__(128)
k_finish_runs(const RunRecord* __restrict__ recs, const int* __restrict__ rec_count, int64_t n_ctas,
              const QueryDesc* __restrict__ desc, const double2* __restrict__ ipfx, int64_t img_n,
              const double2* __restrict__ tpfx, unsigned long long* __restrict__ keys,
              const StreamEntry* __restrict__ streams = nullptr, const int2* __restrict__ slots = nullptr) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t cta = idx / kRunSlots;
    const int slot = (int)(idx - cta * kRunSlots);
    if (cta >= n_ctas || slot >= rec_count[cta]) return;
    const float4* r4 = reinterpret_cast<const float4*>(recs + cta * kRunSlots + slot);
    const int4 head = *reinterpret_cast<const int4*>(r4);
    const float4 c0 = r4[1], c1 = r4[2];
    const float cc[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const int q = head.x;
    const int64_t j0 = (int64_t)(unsigned)head.z | ((int64_t)head.w << 32);
    if constexpr (MULTI) {
        const int2 sl = slots[q];
        ipfx = streams[sl.x].pfx; img_n = streams[sl.x].n; tpfx = streams[sl.y].pfx;
    }
    const QueryDesc d = desc[q];
    const int64_t n = d.tlen, jlo = d.lag0, jhi = d.lag0 + d.nlags;
    const double2 t_hi = tpfx[d.toff + n], t_lo = tpfx[d.toff];
    const double tsum = t_hi.x - t_lo.x, tsq = t_hi.y - t_lo.y;
    const double a = (double)Acc<S>::centre(ipfx[img_n].x, (double)img_n);
    const double b = (double)Acc<S>::centre(tsum, (double)n);
    const double n_ab = (double)n * a * b;
    const double scale = 1.0 / (double)(2 * QB);
    unsigned long long best = ~0ull;
#pragma unroll 1
    for (int i = 0; i < 8; ++i) {
        const int64_t j = j0 + i;
        if (j < jlo || j >= jhi) continue;
        const double2 p_hi = ipfx[j + n], p_lo = ipfx[j];
        const float v = sqdiff_exact((double)cc[i] * scale, p_hi.x - p_lo.x, p_hi.y - p_lo.y, a, b, tsum, tsq, n_ab);
        const unsigned long long key = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned int)(j - jlo);
        best = key < best ? key : best;
    }
    if (best != ~0ull) atomicMin(keys + q, best);
}

// pair_query[i] = query of pair (pair_first + i): one CTA per query fills its own range
__global__ void k_fill_pair_query(const QueryDesc* __restrict__ desc, int q_begin, int64_t pair_first, int* __restrict__ pair_query, int group) {
    const int q = q_begin + blockIdx.x;
    const int64_t base = desc[q].groupBase - pair_first;
    const int np = (desc[q].nk + group - 1) / group;           // pairs of lag blocks
    for (int i = threadIdx.x; i < np; i += blockDim.x) pair_query[base + i] = q;
}

// ---------------------------------------------------------------- forward spectra, quad layout
// Same transform as k_forward_rows in sb_fused.cu (gather + centring + 2B-point real FFT through the
// shared-memory inverse passes run backwards); only the output stage differs: bins leave as the chunks
// A[i] = (X[i], X[i+B/2]) and M[i] = (X[B-i], X[B/2-i]) the packed kernel multiplies.
// MULTI: MODE 0 builds the rows row_list[i] = (slot, row) of several streams, each into its own stream's rows; MODE 1
// reads every query's template from its template slot.
// Persistent: a CTA walks the launch's rows i = blockIdx.x, + gridDim.x, .. < rows, so the FFT's twiddle tables
// travel to shared memory once per CTA (rows < 0: the CTA builds row blockIdx.x only, a launch of one CTA per row).  In MODE 1 a row's query is found by the whole CTA, 512 descriptors per step
// (two steps of dependent loads for up to 262 144 queries instead of one thread's binary search).
template <typename S, int MODE, bool MULTI = false>
__global__ void __launch_bounds__(Cfg<14>::T, 1)
k_forward_quad(const S* __restrict__ src, int64_t src_n, const double2* __restrict__ pfx,
               const QueryDesc* __restrict__ desc, int q_begin, int q_end, int64_t row_first,
               FusedTables tab, float4* __restrict__ out,
               const StreamEntry* __restrict__ streams = nullptr, const int2* __restrict__ slots = nullptr,
               const int2* __restrict__ row_list = nullptr, int64_t rows = -1) {
    typedef Cfg<14> C;
    constexpr int N = C::N, T = C::T, B = C::N;
    constexpr int NT2 = C::R2 * 32, NT3 = C::R3 * 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* buf = reinterpret_cast<float2*>(smem_raw);
    float2* s_t2 = buf + pad(N) + 1;
    float2* s_a3 = s_t2 + NT2;
    float2* s_b3 = s_a3 + NT3;
    int* s_q = reinterpret_cast<int*>(s_b3 + NT3);           // in the 64 bytes behind the tables
    const int tid = threadIdx.x;
    for (int i = tid; i < NT2; i += T) s_t2[i] = __ldg(tab.t2 + i);
    for (int i = tid; i < NT3; i += T) { s_a3[i] = __ldg(tab.a3 + i); s_b3[i] = __ldg(tab.b3 + i); }

    for (int64_t item = blockIdx.x; rows < 0 ? item == blockIdx.x : item < rows; item += gridDim.x) {
        const S* xs = src;
        const double2* xpfx = pfx;
        float4* xout = out;
        int64_t off, len;          // samples [off, off+len) of xs, zero beyond
        float centre;
        int64_t row = row_first + item, out_row = item;
        if constexpr (MULTI && MODE == 0) {
            const int2 rl = row_list[item];
            const StreamEntry se = streams[rl.x];
            xs = static_cast<const S*>(se.raw); xpfx = se.pfx;
            xout = reinterpret_cast<float4*>(se.specq);
            row = out_row = rl.y;
            off = row * B;
            len = se.n - off; if (len > 2 * B) len = 2 * B; if (len < 0) len = 0;
            centre = Acc<S>::centre(xpfx[se.n].x, (double)se.n);
        } else if (MODE == 0) {
            off = row * B;
            len = src_n - off; if (len > 2 * B) len = 2 * B; if (len < 0) len = 0;
            centre = Acc<S>::centre(pfx[src_n].x, (double)src_n);
        } else {
            // largest q in [q_begin, q_end) with partBase <= row: each step tests the candidates lo + t*s, t < m, and the
            // one thread whose candidate is the last that passes writes its t
            int lo = q_begin, n = q_end - q_begin;
            while (n > 1) {
                const int s = (n + T - 1) / T, m = (n + s - 1) / s;
                auto le = [&](int t) { return t == 0 || (t < m && desc[lo + t * s].partBase <= row); };
                if (le(tid) && !le(tid + 1)) *s_q = tid;
                __syncthreads();
                const int c = *s_q;
                __syncthreads();            // s_q is written again by the next step
                lo += c * s;
                n = c == m - 1 ? n - c * s : s;
            }
            const int q = lo;
            const QueryDesc d = desc[q];
            if constexpr (MULTI) { xs = static_cast<const S*>(streams[slots[q].y].raw); xpfx = streams[slots[q].y].pfx; }
            const int64_t seg0 = (row - d.partBase) * B;
            off = d.toff + seg0;
            len = d.tlen - seg0; if (len > B) len = B;
            centre = Acc<S>::centre(xpfx[d.toff + d.tlen].x - xpfx[d.toff].x, (double)d.tlen);
        }
        const S* x = xs + off;
        // all 64 sample loads of a thread in flight at once (the previous row's output stage has read buf: the barrier
        // at the end of the loop body)
#pragma unroll
        for (int k = 0; k < B / T; ++k) {
            const int n = tid + k * T;
            const int64_t i0 = 2 * (int64_t)n;
            const float a = i0 < len ? (float)x[i0] - centre : 0.f;
            const float b = i0 + 1 < len ? (float)x[i0 + 1] - centre : 0.f;
            buf[pad(n)] = make_float2(a, -b);            // conj(z[n])
        }
        __syncthreads();
        ifft_smem<C::R3, false>(buf, s_t2, s_a3, s_b3);   // buf = conj(Z)
        // bins k and B-k from Z[k], Z[B-k]:  X[k] = Xe + conj(w^k)*Xo,  X[B-k] = conj(Xe - conj(w^k)*Xo)
        auto bins = [&](int k, float2& xk, float2& xbk) {
            const float2 zk = buf[pad(k)];
            const float2 zp = buf[pad(k == 0 ? 0 : B - k)];
            const float2 A = make_float2(zk.x, -zk.y), P = make_float2(zp.x, zp.y);     // Z[k], conj(Z[B-k])
            const float2 xe = make_float2(0.5f * (A.x + P.x), 0.5f * (A.y + P.y));
            const float2 dd = make_float2(A.x - P.x, A.y - P.y);
            const float2 xo = make_float2(0.5f * dd.y, -0.5f * dd.x);                   // -i*dd/2
            const float2 w = __ldg(tab.w + k);
            const float2 tv = cmul(make_float2(w.x, -w.y), xo);
            xk = make_float2(xe.x + tv.x, xe.y + tv.y);
            xbk = make_float2(xe.x - tv.x, -(xe.y - tv.y));
        };
        float4* o = xout + out_row * QROW;
        for (int i = tid; i <= Q4; i += T) {
            float2 x_i, x_bi, x_h, x_hb;
            bins(i, x_i, x_bi);                          // X[i], X[B-i]
            bins(B / 2 - i, x_h, x_hb);                  // X[B/2-i], X[B/2+i]
            o[qa(i)] = make_float4(x_i.x, x_hb.x, x_i.y, x_hb.y);
            o[qm(i)] = make_float4(x_bi.x, x_h.x, x_bi.y, x_h.y);
        }
        __syncthreads();           // buf is the next row's
    }
}

size_t forward_smem_bytes14() {
    typedef Cfg<14> C;
    return ((size_t)(C::N + (C::N >> 5) + 1) + C::R2 * 32 + 2 * C::R3 * 32) * sizeof(float2) + 64;
}

// layout of the small area behind Smem::end: barrier (8) | s_best [16] (128) | s_min [16] (64) | park slot (4) ... |
// record counter at 256 | next pair's query + descriptor at 272 (96) | query constants at 384 (32) | end at kSmallBytes
static_assert(8 + QNW * 8 + QNW * 4 + 4 <= kRunCountOff() && kRunCountOff() + 4 <= kNextOff() &&
              kNextOff() + 16 + (int)sizeof(QueryDesc) <= kQueryConstOff() && kQueryConstOff() + 32 <= kSmallBytes, "small shared-memory area");
size_t packed_smem_bytes(int epi = 1) {      // body 3 keeps the runs' exact head sums next to the small arrays
    return epi >= 2 ? kSmemCommon + kSmallBytes + kSpecialBytes + (size_t)kRounds * QT * sizeof(int2)
                    : kSmemCommon + kSmallBytes;           // the small area holds the barrier, the reduction scratch, the park slot and (pair kernel) the next pair's descriptor
}

// Values of the tables of PackedTables, in one array: offsets of wb, d1, d2 in `off` (floats)
constexpr int kPackedTableCount = 3;
std::vector<float> packed_table_values(size_t (&off)[kPackedTableCount]) {
    const double pi = 3.14159265358979323846;
    const size_t nb = 512 * 2, nd1 = 8 * 512 * 4, nd2 = 8 * 32 * 4;
    off[0] = 0; off[1] = nb; off[2] = nb + nd1;
    std::vector<float> h(off[2] + nd2);
    // (W_N^((2a)*k), W_N^((2a+1)*k)) as (c0, s0, c1, s1), a = 0..7, k = 0..K-1
    auto pairs = [&](size_t at, int K, double N) {
        for (int a = 0; a < 8; ++a)
            for (int k = 0; k < K; ++k)
                for (int e = 0; e < 2; ++e) {
                    const double ang = 2.0 * pi * (double)((2 * a + e) * k) / N;
                    h[at + ((size_t)a * K + k) * 4 + 2 * e] = (float)cos(ang); h[at + ((size_t)a * K + k) * 4 + 2 * e + 1] = (float)sin(ang);
                }
    };
    for (int t = 0; t < 512; ++t) { h[off[0] + 2 * t] = (float)cos(pi * t / QB); h[off[0] + 2 * t + 1] = (float)sin(pi * t / QB); }
    pairs(off[1], 512, 8192.0);
    pairs(off[2], 32, 512.0);
    return h;
}

PackedTables packed_tables_at(const float* base, const size_t (&off)[kPackedTableCount]) {
    PackedTables t;
    t.wb = reinterpret_cast<const float2*>(base + off[0]);
    t.d1 = reinterpret_cast<const float4*>(base + off[1]);
    t.d2 = reinterpret_cast<const float4*>(base + off[2]);
    return t;
}

#ifndef SB_EMULATE      // ---- everything below launches kernels or calls the CUDA runtime (not part of tests/emu)
float* g_ptab_dev = nullptr;
PackedTables g_ptab;

int ensure_packed_tables(PackedTables* out) {
    if (!g_ptab_dev) {
        size_t off[kPackedTableCount];
        const std::vector<float> h = packed_table_values(off);
        SB_CUDA(cudaMalloc(&g_ptab_dev, h.size() * sizeof(float)));
        SB_CUDA(cudaMemcpy(g_ptab_dev, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
        g_ptab = packed_tables_at(g_ptab_dev, off);
    }
    *out = g_ptab;
    return SB_OK;
}

__global__ void k_fill_item_query2(const QueryDesc* __restrict__ desc, int q_begin, int64_t item_first,
                                   int* __restrict__ item_query) {
    const int q = q_begin + blockIdx.x;
    const int64_t base = desc[q].itemBase - item_first;
    const int nk = desc[q].nk;
    for (int i = threadIdx.x; i < nk; i += blockDim.x) item_query[base + i] = q;
}

int* g_item_query2 = nullptr;
int64_t g_item_query2_cap = 0;

template <typename S, int MODE, bool MULTI = false>
int launch_forward_quad_typed(const sb_stream* src, const QueryDesc* d_desc, int q_begin, int q_end,
                              int64_t row_first, int64_t rows, float2* out, const MultiArgs* m = nullptr,
                              const int2* row_list = nullptr) {
    Ctx& c = ctx();
    FusedTables tab;
    SB_TRY(fused_tables(&tab));
    static bool attr_set = false;
    const size_t smem = forward_smem_bytes14();
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_forward_quad<S, MODE, MULTI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    const int64_t grid = std::min<int64_t>(rows, c.sm_count);       // persistent: one CTA per SM walks the rows
    k_forward_quad<S, MODE, MULTI><<<(unsigned)grid, Cfg<14>::T, smem, c.stream>>>(
        static_cast<const S*>(src->d_raw), src->n, src->d_pfx, d_desc, q_begin, q_end, row_first, tab,
        reinterpret_cast<float4*>(out), MULTI ? m->d_streams : nullptr, MULTI ? m->d_slots : nullptr, row_list, rows);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// item -> query map of the current launch (one int per CTA), grown on demand
int ensure_item_query(int64_t n) {
    if (g_item_query2_cap < n) {
        cudaStreamSynchronize(ctx().stream);
        cudaFree(g_item_query2); g_item_query2 = nullptr; g_item_query2_cap = 0;
        SB_CUDA(cudaMalloc(&g_item_query2, sizeof(int) * (size_t)n));
        g_item_query2_cap = n;
    }
    return SB_OK;
}

// EPI 3: record slots of the current launch (kRunSlots per CTA) and the CTAs' record counts, grown on demand
RunRecord* g_run_recs = nullptr;
int* g_run_count = nullptr;
int64_t g_run_cap = 0;          // CTAs
constexpr int64_t kRunChunk = 1 << 19;    // CTAs per launch when records are written: 201 MB of slots

int ensure_run_records(int64_t n_ctas) {
    if (g_run_cap < n_ctas) {
        cudaStreamSynchronize(ctx().stream);
        cudaFree(g_run_recs); cudaFree(g_run_count); g_run_recs = nullptr; g_run_count = nullptr; g_run_cap = 0;
        SB_CUDA(cudaMalloc(&g_run_recs, sizeof(RunRecord) * (size_t)n_ctas * kRunSlots));
        SB_CUDA(cudaMalloc(&g_run_count, sizeof(int) * (size_t)n_ctas));
        g_run_cap = n_ctas;
    }
    return SB_OK;
}

// k_match_pair's park: one slot per SM (the kernel's shared memory allows one resident CTA per SM) and a busy flag
// per slot
float4* g_park = nullptr;
int* g_park_busy = nullptr;
int g_park_slots = 0;

int ensure_park() {
    Ctx& c = ctx();
    if (g_park_slots != c.sm_count) {
        cudaStreamSynchronize(c.stream);
        cudaFree(g_park); cudaFree(g_park_busy); g_park = nullptr; g_park_busy = nullptr; g_park_slots = 0;
        SB_CUDA(cudaMalloc(&g_park, sizeof(float4) * kParkF4 * (size_t)c.sm_count));
        SB_CUDA(cudaMalloc(&g_park_busy, sizeof(int) * (size_t)c.sm_count));
        SB_CUDA(cudaMemsetAsync(g_park_busy, 0, sizeof(int) * (size_t)c.sm_count, c.stream));
        g_park_slots = c.sm_count;
    }
    return SB_OK;
}

// Stand-in for the image / template arguments of a multi-stream launch (the kernels read the table instead)
const sb_stream kNoStream{};

template <typename S, bool MULTI>
int launch_finish_runs(const sb_stream* image, const sb_stream* tmpl, const QueryDesc* d_desc, int64_t n_ctas, unsigned long long* d_keys,
                       const MultiArgs* m) {
    Ctx& c = ctx();
    const int64_t threads = n_ctas * kRunSlots;
    k_finish_runs<S, MULTI><<<(unsigned)((threads + 127) / 128), 128, 0, c.stream>>>(g_run_recs, g_run_count, n_ctas, d_desc, image->d_pfx, image->n,
                                                                                   tmpl->d_pfx, d_keys, MULTI ? m->d_streams : nullptr,
                                                                                   MULTI ? m->d_slots : nullptr);
    c.launches += 1;
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// Launchers of the three match kernels.  `Kernel` is one instantiation (sample type x epilogue variant); its
// dynamic shared memory limit is raised once.  The uint8 kernels exist with both epilogues (Ctx::epilogue),
// float32 streams have the first one only.
template <typename S, int EPI, bool MULTI>
int launch_packed_typed(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first,
                        const QueryDesc* d_desc, int64_t item_first, int64_t n_items, const PackedTables& tab,
                        unsigned long long* d_keys, float* d_curve, const MultiArgs* m) {
    Ctx& c = ctx();
    static bool attr_set = false;
    const size_t smem = packed_smem_bytes(EPI);
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_match_packed<S, EPI, MULTI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    const bool records = EPI == 3 && d_curve == nullptr;             // the debug curve evaluates every lag in the kernel
    const int64_t max_grid = records ? kRunChunk : (int64_t)1 << 30;
    for (int64_t i0 = 0; i0 < n_items; i0 += max_grid) {
        const int64_t ni = std::min<int64_t>(max_grid, n_items - i0);
        if (records) SB_TRY(ensure_run_records(ni));
        k_match_packed<S, EPI, MULTI><<<(unsigned)ni, QT, smem, c.stream>>>(
            reinterpret_cast<const float4*>(d_parts), part_first, reinterpret_cast<const float4*>(image->d_specq), image->nblkq,
            static_cast<const S*>(image->d_raw), image->n, image->d_pfx, tmpl->d_pfx, d_desc, g_item_query2 + i0, item_first + i0,
            tab, d_keys, d_curve, records ? g_run_recs : nullptr, records ? g_run_count : nullptr,
            MULTI ? m->d_streams : nullptr, MULTI ? m->d_slots : nullptr);
        if (records) SB_TRY((launch_finish_runs<S, MULTI>(image, tmpl, d_desc, ni, d_keys, m)));
    }
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

template <typename S, int EPI, bool MULTI>
int launch_pair_typed(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first,
                      const QueryDesc* d_desc, int64_t pair_first, int64_t n_pairs, const PackedTables& tab,
                      unsigned long long* d_keys, float* d_curve, const MultiArgs* m) {
    Ctx& c = ctx();
    static bool attr_set = false;
    const size_t smem = packed_smem_bytes(EPI) + 16;
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_match_pair<S, EPI, MULTI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    const bool records = EPI == 3 && d_curve == nullptr;             // the debug curve evaluates every lag in the kernel
    const int64_t max_grid = records ? kRunChunk : (int64_t)1 << 30;
    for (int64_t i0 = 0; i0 < n_pairs; i0 += max_grid) {
        const int64_t ni = std::min<int64_t>(max_grid, n_pairs - i0);
        if (records) SB_TRY(ensure_run_records(ni));
        const int64_t grid = EPI == 3 ? std::min<int64_t>(ni, c.sm_count) : ni;      // body 3 is persistent: one CTA per SM walks the pairs
        k_match_pair<S, EPI, MULTI><<<(unsigned)grid, QT, smem, c.stream>>>(
            reinterpret_cast<const float4*>(d_parts), part_first, reinterpret_cast<const float4*>(image->d_specq), image->nblkq,
            static_cast<const S*>(image->d_raw), image->n, image->d_pfx, tmpl->d_pfx, d_desc, g_item_query2 + i0, pair_first + i0, ni,
            g_park, g_park_busy, g_park_slots, tab, d_keys, d_curve, records ? g_run_recs : nullptr, records ? g_run_count : nullptr,
            MULTI ? m->d_streams : nullptr, MULTI ? m->d_slots : nullptr);
        SB_CUDA(cudaGetLastError());
        if (records) SB_TRY((launch_finish_runs<S, MULTI>(image, tmpl, d_desc, ni, d_keys, m)));
    }
    return SB_OK;
}

// One instantiation per (sample type, epilogue, multi-stream): float32 streams have the first screening loop only.
#define SB_DISPATCH_MATCH1(FN, M, dtype, ...) \
    ((dtype) != SB_U8        ? FN<float, 1, M>(__VA_ARGS__) \
     : ctx().epilogue == 3   ? FN<uint8_t, 3, M>(__VA_ARGS__) : FN<uint8_t, 1, M>(__VA_ARGS__))
#define SB_DISPATCH_MATCH(FN, image, tmpl, multi, ...) \
    ((multi) ? SB_DISPATCH_MATCH1(FN, true, (multi)->dtype, &kNoStream, &kNoStream, __VA_ARGS__, multi) \
             : SB_DISPATCH_MATCH1(FN, false, (image)->dtype, image, tmpl, __VA_ARGS__, multi))

}  // namespace

namespace sb {

int launch_match_packed(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first,
                        const QueryDesc* d_desc, int q_begin, int q_end, int64_t item_first, int64_t n_items,
                        unsigned long long* d_keys, float* d_curve, const MultiArgs* multi) {
    Ctx& c = ctx();
    PackedTables tab;
    SB_TRY(ensure_packed_tables(&tab));
    SB_TRY(ensure_item_query(n_items));
    k_fill_item_query2<<<(unsigned)(q_end - q_begin), 128, 0, c.stream>>>(d_desc, q_begin, item_first, g_item_query2);
    c.launches += 1;
    return SB_DISPATCH_MATCH(launch_packed_typed, image, tmpl, multi, d_parts, part_first, d_desc, item_first, n_items, tab, d_keys, d_curve);
}

int launch_match_pair(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first,
                      const QueryDesc* d_desc, int q_begin, int q_end, int64_t pair_first, int64_t n_pairs,
                      unsigned long long* d_keys, float* d_curve, const MultiArgs* multi) {
    Ctx& c = ctx();
    PackedTables tab;
    SB_TRY(ensure_packed_tables(&tab));
    SB_TRY(ensure_item_query(n_pairs));
    SB_TRY(ensure_park());
    k_fill_pair_query<<<(unsigned)(q_end - q_begin), 128, 0, c.stream>>>(d_desc, q_begin, pair_first, g_item_query2, 2);
    c.launches += 1;
    return SB_DISPATCH_MATCH(launch_pair_typed, image, tmpl, multi, d_parts, part_first, d_desc, pair_first, n_pairs, tab, d_keys, d_curve);
}

int launch_block_spectra_quad(const sb_stream* s, int64_t k_first, int64_t rows, float2* out) {
    return s->dtype == SB_U8 ? launch_forward_quad_typed<uint8_t, 0>(s, nullptr, 0, 0, k_first, rows, out)
                             : launch_forward_quad_typed<float, 0>(s, nullptr, 0, 0, k_first, rows, out);
}

int launch_block_spectra_quad_multi(const MultiArgs& m, const int2* d_row_list, int64_t n_rows) {
    return m.dtype == SB_U8 ? launch_forward_quad_typed<uint8_t, 0, true>(&kNoStream, nullptr, 0, 0, 0, n_rows, nullptr, &m, d_row_list)
                            : launch_forward_quad_typed<float, 0, true>(&kNoStream, nullptr, 0, 0, 0, n_rows, nullptr, &m, d_row_list);
}

int launch_part_spectra_quad(const sb_stream* tmpl, const QueryDesc* d_desc, int q_begin, int q_end,
                             int64_t part_first, int64_t rows, float2* out, const MultiArgs* multi) {
    if (multi)
        return multi->dtype == SB_U8 ? launch_forward_quad_typed<uint8_t, 1, true>(&kNoStream, d_desc, q_begin, q_end, part_first, rows, out, multi)
                                     : launch_forward_quad_typed<float, 1, true>(&kNoStream, d_desc, q_begin, q_end, part_first, rows, out, multi);
    return tmpl->dtype == SB_U8 ? launch_forward_quad_typed<uint8_t, 1>(tmpl, d_desc, q_begin, q_end, part_first, rows, out)
                                : launch_forward_quad_typed<float, 1>(tmpl, d_desc, q_begin, q_end, part_first, rows, out);
}

void packed_release_tables() {
    if (g_ptab_dev) cudaFree(g_ptab_dev);
    g_ptab_dev = nullptr;
    cudaFree(g_item_query2); g_item_query2 = nullptr; g_item_query2_cap = 0;
    cudaFree(g_run_recs); cudaFree(g_run_count); g_run_recs = nullptr; g_run_count = nullptr; g_run_cap = 0;
    cudaFree(g_park); cudaFree(g_park_busy); g_park = nullptr; g_park_busy = nullptr; g_park_slots = 0;
}

}  // namespace sb
#else
}  // namespace (tests/emu includes this file and adds its entry points behind it)
#endif  // SB_EMULATE
