// Fused lag-block kernel: for one (query, lag block) item a CTA
//   1. accumulates Y[bin] = sum_p conj(T^_p[bin]) * X^_{k+p}[bin] straight from L2 into registers,
//   2. packs the Hermitian half spectrum into a half-size complex sequence in shared memory,
//   3. runs the inverse FFT entirely in shared memory (Stockham, radix 32 x {32|16} x 16),
//   4. slides the window sums through its lags, screens every lag in fp32 and evaluates only the
//      lags that can still be the minimum with OpenCV's rule in fp64, and
//   5. merges its (value, first index) into the query's result with one 64-bit atomicMin.
// The B-long correlation block never touches HBM; the only global traffic is the spectra (L2
// resident) and 2 B per lag of raw samples.  See DESIGN.md section 4 for the roofline of each phase.
#include "sb_internal.h"
#include <cmath>
#include <cstdlib>
#include <vector>

#include "sb_fused_common.cuh"
#include "sb_fft_smem.cuh"

using namespace sb;
using namespace sbf;

namespace {

typedef Cfg<14> C;
static_assert(C::N == kLagBlock, "the FFT half-size is the lag block");

// ---------------------------------------------------------------- the kernel
template <typename S>
__global__ void __launch_bounds__(C::T, C::MINB)
k_match_fused(const float2* __restrict__ That, int64_t part_first, const float2* __restrict__ Ypre,
              const float2* __restrict__ Xhat, int64_t nblk,
              const S* __restrict__ img, int64_t img_n,
              const double2* __restrict__ ipfx, const double2* __restrict__ tpfx,
              const QueryDesc* __restrict__ desc, const int* __restrict__ item_query, int64_t item_first,
              FusedTables tab, unsigned long long* __restrict__ keys, float* __restrict__ curve_out) {
    constexpr int N = C::N, T = C::T, B = C::N;
    constexpr int NB = B + 1;                       // bins per spectrum row
    // geometry: real FFT of 2B points; hop = partition length = B; an item yields the LB = B lags
    // that the circular correlation gets right
    constexpr int LB = B;
    constexpr int LAGS_PER_ROUND = T * 8;           // 8 consecutive lags per thread per round
    constexpr int ROUNDS = LB / LAGS_PER_ROUND;     // 4
    constexpr int KEEP3 = C::R3 * LB / (2 * B);     // outputs of a last-pass butterfly that carry valid lags
    static_assert(LB % LAGS_PER_ROUND == 0 && ROUNDS * 8 <= 64, "epilogue tiling");
    constexpr int NW = T / 32;
    constexpr int NT2 = C::R2 * 32, NT3 = C::R3 * 32;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* buf = reinterpret_cast<float2*>(smem_raw);                  // pad(N) complex values
    float2* s_t2 = buf + pad(N) + 1;                                    // twiddle tables
    float2* s_a3 = s_t2 + NT2;
    float2* s_b3 = s_a3 + NT3;
    // 16-byte aligned staging area for cp.async (the padded FFT buffer has an odd number of float2)
    unsigned char* stage = smem_raw + (((size_t)(pad(N) + 1 + NT2 + 2 * NT3) * sizeof(float2) + 15) & ~(size_t)15);
    double2* s_base = reinterpret_cast<double2*>(stage);                // [ROUNDS][NW][2] exact running sums
    unsigned char* s_lo = reinterpret_cast<unsigned char*>(s_base + ROUNDS * NW * 2);   // image[j_blk .. +B+16)
    unsigned char* s_hi = s_lo + LB + 16;                               // image[(j_blk+n)&~15 .. +LB+48)
    unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(s_hi + LB + 48);  // mbarrier of the TMA copies
    unsigned long long* s_best = s_bar + 1;                             // [NW]
    float* s_min = reinterpret_cast<float*>(s_best + NW);               // [NW]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t item = item_first + blockIdx.x;
    const int q = __ldg(item_query + blockIdx.x);     // which query this lag block belongs to
    // stage the FFT twiddle tables (16 KB); first needed in pass 2, several barriers from here
    for (int i = tid; i < NT2; i += T) s_t2[i] = __ldg(tab.t2 + i);
    for (int i = tid; i < NT3; i += T) { s_a3[i] = __ldg(tab.a3 + i); s_b3[i] = __ldg(tab.b3 + i); }
    const QueryDesc d = desc[q];
    const int64_t k = d.k0 + (item - d.itemBase);

    // ---------------- 0. stage what the epilogue needs (uint8 streams) ----------------------
    // The two byte windows the sliding sums read (image[j] and image[j+n] over this lag block) go to
    // shared memory by TMA bulk copies, one exact (sum, sum of squares) pair per warp-round from the
    // fp64 running sums by cp.async -- all issued now; their latency hides behind the MAC and the FFT.
    if (sizeof(S) == 1) {
        const unsigned char* img8 = reinterpret_cast<const unsigned char*>(img);
        const int64_t j_blk0 = k * LB, hi0 = (j_blk0 + d.tlen) & ~(int64_t)15;
        const int64_t limit = (img_n + 16) & ~(int64_t)15;               // allocation has 16 bytes of slack
        if (tid == 0) {
            // the two windows: one TMA bulk copy each (1-D cp.async.bulk), completion on an mbarrier
            int64_t lo_bytes = limit - j_blk0; if (lo_bytes > LB + 16) lo_bytes = LB + 16; if (lo_bytes < 0) lo_bytes = 0;
            int64_t hi_bytes = limit - hi0;    if (hi_bytes > LB + 48) hi_bytes = LB + 48; if (hi_bytes < 0) hi_bytes = 0;
            mbar_init(s_bar, 1);
            mbar_expect_tx(s_bar, (unsigned)(lo_bytes + hi_bytes));
            if (lo_bytes) tma_load_1d(s_lo, img8 + j_blk0, (unsigned)lo_bytes, s_bar);
            if (hi_bytes) tma_load_1d(s_hi, img8 + hi0, (unsigned)hi_bytes, s_bar);
        }
        if (tid < ROUNDS * NW * 2) {                                      // 16-byte pieces: plain cp.async
            const int c = tid / (NW * 2), w = (tid >> 1) % NW, which = tid & 1;
            const int64_t jw = j_blk0 + c * LAGS_PER_ROUND + w * 256;    // first lag of warp w in round c
            if (jw < d.lag0 + d.nlags) cp_async16(s_base + tid, ipfx + jw + (which ? d.tlen : 0));
        }
    }

    // ---------------- 1+2. spectral multiply-accumulate and Hermitian packing ---------------
    {
        int P = d.P;
        const int64_t row0 = k;                     // block-spectrum row of partition 0
        if (row0 + P > nblk) P = (int)(nblk - row0);    // rows past the end of the stream are zero
        const float2* tp = That + (d.partBase - part_first) * (int64_t)NB;
        const float2* xp = Xhat + row0 * (int64_t)NB;
        constexpr int U = 8;                        // bin pairs in flight per thread
        static_assert((B / 2) % (U * T) == 0, "pair loop must tile B/2");
        // pairs (m, B-m), m = 1 .. B/2-1, plus m = 0 whose partner is the Nyquist bin B
        for (int m0 = tid; m0 < B / 2; m0 += U * T) {
            float2 ym[U], yp[U];
#pragma unroll
            for (int u = 0; u < U; ++u) { ym[u] = make_float2(0.f, 0.f); yp[u] = make_float2(0.f, 0.f); }
            if (Ypre) {                             // products already formed by k_mac_blocked (long templates)
                const float2* y = Ypre + (int64_t)blockIdx.x * NB;
#pragma unroll
                for (int u = 0; u < U; ++u) { const int m = m0 + u * T; ym[u] = __ldg(y + m); yp[u] = __ldg(y + (B - m)); }
            } else
            for (int p = 0; p < P; ++p) {
                const float2* t = tp + (int64_t)p * NB;
                const float2* x = xp + (int64_t)p * NB;
                float2 t1[U], x1[U], t2[U], x2[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int m = m0 + u * T;
                    t1[u] = __ldg(t + m); x1[u] = __ldg(x + m);
                    t2[u] = __ldg(t + (B - m)); x2[u] = __ldg(x + (B - m));
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    ym[u].x += t1[u].x * x1[u].x + t1[u].y * x1[u].y;  ym[u].y += t1[u].x * x1[u].y - t1[u].y * x1[u].x;
                    yp[u].x += t2[u].x * x2[u].x + t2[u].y * x2[u].y;  yp[u].y += t2[u].x * x2[u].y - t2[u].y * x2[u].x;
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int m = m0 + u * T;
                const float2 w = __ldg(tab.w + m);                     // exp(+i*pi*m/B)
                // Z[m]   = (Ym + conj(Yp)) + i*(Ym - conj(Yp))*w
                const float2 e = make_float2(ym[u].x + yp[u].x, ym[u].y - yp[u].y);
                const float2 o = cmul(make_float2(ym[u].x - yp[u].x, ym[u].y + yp[u].y), w);
                buf[pad(m0) + u * (T / 32 * 33)] = make_float2(e.x - o.y, e.y + o.x);
                // Z[B-m] = conj(e) + i*conj(o)   (w^(B-m) = -conj(w^m))
                if (m > 0) buf[pad(B - m0) - u * (T / 32 * 33)] = make_float2(e.x + o.y, -e.y + o.x);
            }
        }
        if (tid < 32) {                             // the self-paired bin m = B/2 (w = i): Z = 2*conj(Y)
            float2 y = make_float2(0.f, 0.f);
            if (Ypre) { if (lane == 0) y = __ldg(Ypre + (int64_t)blockIdx.x * NB + B / 2); }
            else
            for (int p = lane; p < P; p += 32) {
                const float2 t1 = __ldg(tp + (int64_t)p * NB + B / 2), x1 = __ldg(xp + (int64_t)p * NB + B / 2);
                y.x += t1.x * x1.x + t1.y * x1.y;  y.y += t1.x * x1.y - t1.y * x1.x;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { y.x += __shfl_xor_sync(0xffffffffu, y.x, o); y.y += __shfl_xor_sync(0xffffffffu, y.y, o); }
            if (lane == 0) buf[pad(B / 2)] = make_float2(2.f * y.x, -2.f * y.y);
        }
    }
    __syncthreads();

    // ---------------- 3. inverse FFT of N complex points in shared memory -------------------
    ifft_smem<KEEP3, true>(buf, s_t2, s_a3, s_b3);
    // now buf[pad(i)] = (x[2i], x[2i+1]) for i < N/2: correlation at lags 2i, 2i+1 (times 2B)

    // ---------------- 4. window sums, fp32 screening, fp64 exact evaluation -----------------
    // Every thread owns runs of 8 consecutive lags.  The exact window sums at the first lag of a
    // run come from the interleaved fp64 running sums (two 16-byte loads per run); inside the run
    // the window slides on the raw samples: W[j+1] = W[j] + I[j+n]^k - I[j]^k.
    const int64_t n = d.tlen;
    const int64_t jlo = d.lag0, jhi = d.lag0 + d.nlags;
    const int64_t j_blk = k * LB;
    const double2 t_hi = tpfx[d.toff + n], t_lo = tpfx[d.toff];
    const double tsum = t_hi.x - t_lo.x, tsq = t_hi.y - t_lo.y;
    const double a = (double)Acc<S>::centre(ipfx[img_n].x, (double)img_n);
    const double b = (double)Acc<S>::centre(tsum, (double)n);
    const double n_ab = (double)n * a * b;
    const double scale = 1.0 / (double)(2 * B);
    const double k_const = a * tsum - n_ab;
    const float f_tsq = (float)tsq, f_b = (float)b, f_scale = (float)scale;
    const bool interior = j_blk >= jlo && j_blk + LB <= jhi;          // every lag of the item is valid

    float vf[ROUNDS][8];
    float tmin = 2.0f;
    if (sizeof(S) == 1) mbar_wait(s_bar, 0);                          // TMA copies of step 0 (long done)
    if (sizeof(S) == 1) {
        // uint8: everything comes from shared memory.  Per round each warp covers 256 consecutive lags;
        // lane l owns the run of 8 lags starting at jw + 8l.  Window sums at the head of a run = exact
        // warp base + exclusive intra-warp scan of the runs' integer totals (dp4a), then slide by 1.
        const int hi_off = (int)((j_blk + n) & 15);
#pragma unroll
        for (int c = 0; c < ROUNDS; ++c) {
            const int m0 = c * LAGS_PER_ROUND + tid * 8;
            const int64_t j0 = j_blk + m0;
            const int64_t jw = j_blk + c * LAGS_PER_ROUND + warp * 256;
            if (jw >= jhi || jw + 256 <= jlo) {                       // no valid lag in this warp-round (warp-uniform)
#pragma unroll
                for (int i = 0; i < 8; ++i) vf[c][i] = 2.0f;
                continue;
            }
            const unsigned long long lo8 = *reinterpret_cast<const unsigned long long*>(s_lo + m0);
            const int hb = hi_off + m0;                                // byte offset into s_hi, any alignment
            const unsigned long long h0 = *reinterpret_cast<const unsigned long long*>(s_hi + (hb & ~7));
            const unsigned long long h1 = *reinterpret_cast<const unsigned long long*>(s_hi + (hb & ~7) + 8);
            const unsigned sh = (unsigned)(hb & 7) * 8u;
            const unsigned long long hi8 = sh ? ((h0 >> sh) | (h1 << (64u - sh))) : h0;
            const unsigned la = (unsigned)lo8, lb = (unsigned)(lo8 >> 32), ha = (unsigned)hi8, hb2 = (unsigned)(hi8 >> 32);
            int tq = (int)__dp4a(ha, ha, __dp4a(hb2, hb2, 0u)) - (int)__dp4a(la, la, __dp4a(lb, lb, 0u));
            int ts = (int)__dp4a(ha, 0x01010101u, __dp4a(hb2, 0x01010101u, 0u)) - (int)__dp4a(la, 0x01010101u, __dp4a(lb, 0x01010101u, 0u));
            int iq = tq, is = ts;                                      // inclusive scan over the lanes
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int uq = __shfl_up_sync(0xffffffffu, iq, o), us = __shfl_up_sync(0xffffffffu, is, o);
                if (lane >= o) { iq += uq; is += us; }
            }
            const double2 b_lo = s_base[(c * NW + warp) * 2], b_hi = s_base[(c * NW + warp) * 2 + 1];
            const double w0s = (b_hi.x - b_lo.x) + (double)(is - ts);
            const double w0q = (b_hi.y - b_lo.y) + (double)(iq - tq);
            const float f_w0q = (float)w0q;
            const float f_k0 = (float)(b * w0s + k_const);
            float cc[8];
#pragma unroll
            for (int h = 0; h < 4; ++h) { const float2 z = buf[pad(m0 >> 1) + h]; cc[2 * h] = z.x; cc[2 * h + 1] = z.y; }
            int rq = 0, rs = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float wq = f_w0q + (float)rq;
                const float sit = fmaf(cc[i], f_scale, fmaf(f_b, (float)rs, f_k0));
                const float num = fmaxf((wq + f_tsq) - 2.0f * sit, 0.0f);
                const float pr = wq * f_tsq;
                // pr == 0 (silent window or template): rsqrt -> inf, num*inf -> inf or NaN, fminf(.,1) -> 1
                const float v = fminf(num * rsqrt_fast(pr), 1.0f);
                if (interior) { vf[c][i] = v; tmin = fminf(tmin, v); }
                else if (j0 + i >= jlo && j0 + i < jhi) { vf[c][i] = v; tmin = fminf(tmin, v); }
                else vf[c][i] = 2.0f;                                  // sentinel: not a valid lag
                const int lo = (int)((lo8 >> (8 * i)) & 0xffu), hi = (int)((hi8 >> (8 * i)) & 0xffu);
                rq += hi * hi - lo * lo; rs += hi - lo;
            }
        }
    } else {
        // float32 streams: exact fp64 base per run straight from the running sums, slide in fp64
#pragma unroll
        for (int c = 0; c < ROUNDS; ++c) {
            const int m0 = c * LAGS_PER_ROUND + tid * 8;
            const int64_t j0 = j_blk + m0;
#pragma unroll
            for (int i = 0; i < 8; ++i) vf[c][i] = 2.0f;
            if (!(j0 < jhi && j0 + 8 > jlo)) continue;
            const double2 p_hi = ipfx[j0 + n], p_lo = ipfx[j0];
            const float f_w0q = (float)(p_hi.y - p_lo.y);
            const float f_k0 = (float)(b * (p_hi.x - p_lo.x) + k_const);
            float cc[8];
#pragma unroll
            for (int h = 0; h < 4; ++h) { const float2 z = buf[pad(m0 >> 1) + h]; cc[2 * h] = z.x; cc[2 * h + 1] = z.y; }
            double rq = 0.0, rs = 0.0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t j = j0 + i;
                const float wq = f_w0q + (float)rq;
                const float sit = fmaf(cc[i], f_scale, fmaf(f_b, (float)rs, f_k0));
                const float num = fmaxf((wq + f_tsq) - 2.0f * sit, 0.0f);
                const float pr = wq * f_tsq;
                const float v = fminf(num * rsqrt_fast(pr), 1.0f);
                if (j >= jlo && j < jhi) { vf[c][i] = v; tmin = fminf(tmin, v); }
                if (j + n < img_n) {
                    const double lo = (double)img[j], hi = (double)img[j + n];
                    rq += hi * hi - lo * lo; rs += hi - lo;
                }
            }
        }
    }
    const float my_min = tmin;                                        // this thread's own best
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tmin = fminf(tmin, __shfl_xor_sync(0xffffffffu, tmin, o));
    if (lane == 0) s_min[warp] = tmin;
    __syncthreads();
    float bmin = s_min[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) bmin = fminf(bmin, s_min[w]);
    const float thr = curve_out ? 1.5f : bmin + kScreenMargin;       // debug curve: evaluate everything

    // lags that can still be the minimum (bit c*8+i), then ONE copy of the fp64 path
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
        const float2 z = buf[pad(m >> 1)];
        const double cc = (double)((m & 1) ? z.y : z.x) * scale;
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
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < NW; ++w) best = s_best[w] < best ? s_best[w] : best;
        if (best != ~0ull) atomicMin(keys + q, best);
    }
}

// ---------------------------------------------------------------- forward spectra
// Real-to-complex transform of 2B centred samples per row, written as the B+1 bins every other
// kernel expects (same layout and scaling as an unnormalised R2C of size 2B).  It is the inverse
// kernel's machinery run backwards: z[n] = x[2n] + i*x[2n+1], Z = conj(IFFT(conj(z))), then
//   X[k] = Xe + conj(w^k)*Xo,  X[B-k] = conj(Xe - conj(w^k)*Xo),
//   Xe = (Z[k] + conj(Z[B-k]))/2,  Xo = -i*(Z[k] - conj(Z[B-k]))/2,  w = exp(i*pi/B).
// Rows are either the lag blocks of a stream (MODE 0: samples [kB, kB+2B), centred on the stream
// mean) or the partitions of the batch's templates (MODE 1: B samples + B zeros, centred on the
// template's own mean) -- the gather, the centring and the FFT are one pass over the data.
template <typename S, int MODE>
__global__ void __launch_bounds__(C::T, C::MINB)
k_forward_rows(const S* __restrict__ src, int64_t src_n, const double2* __restrict__ pfx,
               const QueryDesc* __restrict__ desc, int q_begin, int q_end, int64_t row_first,
               FusedTables tab, float2* __restrict__ out) {
    constexpr int N = C::N, T = C::T, B = C::N, NB = B + 1;   // rows are B samples apart
    constexpr int NT2 = C::R2 * 32, NT3 = C::R3 * 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* buf = reinterpret_cast<float2*>(smem_raw);
    float2* s_t2 = buf + pad(N) + 1;
    float2* s_a3 = s_t2 + NT2;
    float2* s_b3 = s_a3 + NT3;
    __shared__ int s_q;
    const int tid = threadIdx.x;
    for (int i = tid; i < NT2; i += T) s_t2[i] = __ldg(tab.t2 + i);
    for (int i = tid; i < NT3; i += T) { s_a3[i] = __ldg(tab.a3 + i); s_b3[i] = __ldg(tab.b3 + i); }

    int64_t off, len;          // samples [off, off+len) of src, zero beyond
    float centre;
    const int64_t row = row_first + blockIdx.x;
    if (MODE == 0) {
        off = row * B;
        len = src_n - off; if (len > 2 * B) len = 2 * B; if (len < 0) len = 0;
        centre = Acc<S>::centre(pfx[src_n].x, (double)src_n);
    } else {
        if (tid == 0) {        // largest q with partBase <= row
            int lo = q_begin, hi = q_end - 1;
            while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (desc[mid].partBase <= row) lo = mid; else hi = mid - 1; }
            s_q = lo;
        }
        __syncthreads();
        const QueryDesc d = desc[s_q];
        const int64_t seg0 = (row - d.partBase) * B;
        off = d.toff + seg0;
        len = d.tlen - seg0; if (len > B) len = B;
        centre = Acc<S>::centre(pfx[d.toff + d.tlen].x - pfx[d.toff].x, (double)d.tlen);
    }
    const S* x = src + off;
#pragma unroll 4
    for (int n = tid; n < B; n += T) {
        const int64_t i0 = 2 * (int64_t)n;
        const float a = i0 < len ? (float)x[i0] - centre : 0.f;
        const float b = i0 + 1 < len ? (float)x[i0 + 1] - centre : 0.f;
        buf[pad(n)] = make_float2(a, -b);            // conj(z[n])
    }
    __syncthreads();
    ifft_smem<C::R3, false>(buf, s_t2, s_a3, s_b3);   // buf = conj(Z)
    float2* o = out + (int64_t)blockIdx.x * NB;
    for (int k = tid; k <= B / 2; k += T) {
        const float2 zk = buf[pad(k)];
        const float2 zp = buf[pad(k == 0 ? 0 : B - k)];
        const float2 A = make_float2(zk.x, -zk.y), P = make_float2(zp.x, zp.y);     // Z[k], conj(Z[B-k])
        const float2 xe = make_float2(0.5f * (A.x + P.x), 0.5f * (A.y + P.y));
        const float2 dd = make_float2(A.x - P.x, A.y - P.y);
        const float2 xo = make_float2(0.5f * dd.y, -0.5f * dd.x);                   // -i*dd/2
        const float2 w = __ldg(tab.w + k);
        const float2 tv = cmul(make_float2(w.x, -w.y), xo);
        o[k] = make_float2(xe.x + tv.x, xe.y + tv.y);
        if (k != B / 2) o[B - k] = make_float2(xe.x - tv.x, -(xe.y - tv.y));
    }
}

size_t forward_smem_bytes() {
    return ((size_t)(C::N + (C::N >> 5) + 1) + C::R2 * 32 + 2 * C::R3 * 32) * sizeof(float2) + 64;
}

// ---------------------------------------------------------------- host side
size_t fused_smem_bytes() {
    const size_t padded = (size_t)(C::N + (C::N >> 5) + 1);
    const size_t nw = C::T / 32;
    const size_t LB = C::N;
    const size_t rounds = LB / (C::T * 8);
    return (padded + C::R2 * 32 + 2 * C::R3 * 32) * sizeof(float2) + nw * sizeof(unsigned long long)
         + 16 + rounds * nw * 2 * sizeof(double2) + (LB + 16) + (LB + 48) + 8 + nw * sizeof(float) + 64;
}

struct TableSet { float2* dev = nullptr; FusedTables tab; };
TableSet g_tables;

int ensure_tables(FusedTables* out) {
    TableSet& ts = g_tables;
    if (!ts.dev) {
        const int N = C::N;
        const size_t nw = N / 2 + 1, n2 = (size_t)C::R2 * 32, n3 = (size_t)C::R3 * 32;
        std::vector<float2> h(nw + n2 + 2 * n3);
        const double pi = 3.14159265358979323846;
        for (size_t m = 0; m < nw; ++m) h[m] = make_float2((float)cos(pi * m / N), (float)sin(pi * m / N));
        for (int r = 0; r < C::R2; ++r)
            for (int k = 0; k < 32; ++k) {
                const double ang = 2.0 * pi * r * k / (32.0 * C::R2);
                h[nw + r * 32 + k] = make_float2((float)cos(ang), (float)sin(ang));
            }
        for (int r = 0; r < C::R3; ++r)
            for (int k = 0; k < 32; ++k) {
                const double al = 2.0 * pi * r * k / N, ah = 2.0 * pi * r * (k * 32.0) / N;
                h[nw + n2 + r * 32 + k] = make_float2((float)cos(al), (float)sin(al));
                h[nw + n2 + n3 + r * 32 + k] = make_float2((float)cos(ah), (float)sin(ah));
            }
        SB_CUDA(cudaMalloc(&ts.dev, h.size() * sizeof(float2)));
        SB_CUDA(cudaMemcpy(ts.dev, h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice));
        ts.tab.w = ts.dev; ts.tab.t2 = ts.dev + nw; ts.tab.a3 = ts.dev + nw + n2; ts.tab.b3 = ts.dev + nw + n2 + n3;
    }
    *out = ts.tab;
    return SB_OK;
}

// item_query[i] = query of item (item_first + i): one CTA per query fills its own range
__global__ void k_fill_item_query(const QueryDesc* __restrict__ desc, int q_begin, int64_t item_first,
                                  int* __restrict__ item_query) {
    const int q = q_begin + blockIdx.x;
    const int64_t base = desc[q].itemBase - item_first;
    const int nk = desc[q].nk;
    for (int i = threadIdx.x; i < nk; i += blockDim.x) item_query[base + i] = q;
}

int* g_item_query = nullptr;
int64_t g_item_query_cap = 0;

template <typename S>
int launch_typed(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first, const float2* d_premac,
                 const QueryDesc* d_desc, int q_begin, int q_end, int64_t item_first, int64_t n_items,
                 unsigned long long* d_keys, float* d_curve) {
    Ctx& c = ctx();
    FusedTables tab;
    SB_TRY(ensure_tables(&tab));
    static bool attr_set = false;
    const size_t smem = fused_smem_bytes();
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_match_fused<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    if (g_item_query_cap < n_items) {
        cudaStreamSynchronize(c.stream);
        cudaFree(g_item_query); g_item_query = nullptr; g_item_query_cap = 0;
        SB_CUDA(cudaMalloc(&g_item_query, sizeof(int) * (size_t)n_items));
        g_item_query_cap = n_items;
    }
    k_fill_item_query<<<(unsigned)(q_end - q_begin), 128, 0, c.stream>>>(d_desc, q_begin, item_first, g_item_query);
    c.launches += 1;
    const int64_t max_grid = 1 << 30;
    for (int64_t i0 = 0; i0 < n_items; i0 += max_grid) {
        const int64_t ni = std::min<int64_t>(max_grid, n_items - i0);
        k_match_fused<S><<<(unsigned)ni, C::T, smem, c.stream>>>(
            d_parts, part_first, d_premac ? d_premac + i0 * (int64_t)(C::N + 1) : nullptr, image->d_spec, image->nblk,
            static_cast<const S*>(image->d_raw), image->n,
            image->d_pfx, tmpl->d_pfx, d_desc, g_item_query + i0, item_first + i0,
            tab, d_keys, d_curve);
    }
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

template <typename S, int MODE>
int launch_forward_typed(const sb_stream* src, const QueryDesc* d_desc, int q_begin, int q_end,
                         int64_t row_first, int64_t rows, float2* out) {
    Ctx& c = ctx();
    FusedTables tab;
    SB_TRY(ensure_tables(&tab));
    static bool attr_set = false;
    const size_t smem = forward_smem_bytes();
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_forward_rows<S, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    k_forward_rows<S, MODE><<<(unsigned)rows, C::T, smem, c.stream>>>(
        static_cast<const S*>(src->d_raw), src->n, src->d_pfx, d_desc, q_begin, q_end, row_first, tab, out);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

template <int MODE>
int launch_forward(const sb_stream* src, const QueryDesc* d_desc, int q_begin, int q_end,
                   int64_t row_first, int64_t rows, float2* out) {
    if (src->dtype == SB_U8) return launch_forward_typed<uint8_t, MODE>(src, d_desc, q_begin, q_end, row_first, rows, out);
    return launch_forward_typed<float, MODE>(src, d_desc, q_begin, q_end, row_first, rows, out);
}

}  // namespace

namespace sb {

int launch_match_fused(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first, const float2* d_premac,
                       const QueryDesc* d_desc, int q_begin, int q_end, int64_t item_first, int64_t n_items,
                       unsigned long long* d_keys, float* d_curve) {
    if (image->dtype == SB_U8)
        return launch_typed<uint8_t>(image, tmpl, d_parts, part_first, d_premac, d_desc, q_begin, q_end, item_first, n_items, d_keys, d_curve);
    return launch_typed<float>(image, tmpl, d_parts, part_first, d_premac, d_desc, q_begin, q_end, item_first, n_items, d_keys, d_curve);
}

// Block spectra of a stream: rows [k_first, k_first + rows) into out (row stride B+1)
int launch_block_spectra(const sb_stream* s, int64_t k_first, int64_t rows, float2* out) {
    return launch_forward<0>(s, nullptr, 0, 0, k_first, rows, out);
}
// Partition spectra of the templates of queries [q_begin, q_end): global part rows [part_first, +rows)
int launch_part_spectra(const sb_stream* tmpl, const QueryDesc* d_desc, int q_begin, int q_end,
                        int64_t part_first, int64_t rows, float2* out) {
    return launch_forward<1>(tmpl, d_desc, q_begin, q_end, part_first, rows, out);
}

int fused_tables(FusedTables* out) { return ensure_tables(out); }

void fused_release_tables() {
    if (g_tables.dev) cudaFree(g_tables.dev);
    g_tables.dev = nullptr;
    cudaFree(g_item_query); g_item_query = nullptr; g_item_query_cap = 0;
}

}  // namespace sb
