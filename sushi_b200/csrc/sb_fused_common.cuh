// Device helpers of the fused lag-block kernel (sb_fused.cu): complex arithmetic, in-register DFTs,
// the exact per-lag formula, async-copy wrappers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifdef SB_EMULATE
#include "emu_ptx.h"      // tests/emu: host stand-ins for the inline PTX (test infrastructure)
#else
#include "sb_ptx.cuh"
#endif

namespace sbf {

// ---------------------------------------------------------------- small complex helpers
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// exp(+2*pi*i*q/32), q = 0..15
__device__ constexpr float kC32[16] = {
    1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
    0.70710678118654752f, 0.55557023301960218f, 0.38268343236508978f, 0.19509032201612825f,
    0.0f, -0.19509032201612825f, -0.38268343236508978f, -0.55557023301960218f,
    -0.70710678118654752f, -0.83146961230254524f, -0.92387953251128674f, -0.98078528040323043f};
__device__ constexpr float kS32[16] = {
    0.0f, 0.19509032201612825f, 0.38268343236508978f, 0.55557023301960218f,
    0.70710678118654752f, 0.83146961230254524f, 0.92387953251128674f, 0.98078528040323043f,
    1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
    0.70710678118654752f, 0.55557023301960218f, 0.38268343236508978f, 0.19509032201612825f};

// d * exp(+2*pi*i*q/32) with q a compile-time constant after unrolling.  The roundings are spelled out: with the
// butterflies unrolled, a plain product would be free to fuse into the next stage's sum, and the spectra would
// change in the last bit.
__device__ __forceinline__ float2 rot32(float2 d, int q) {
    if (q == 0) return d;
    if (q == 8) return make_float2(-d.y, d.x);
    const float h = 0.70710678118654752f;
    if (q == 4) return make_float2(__fmul_rn(d.x - d.y, h), __fmul_rn(d.x + d.y, h));
    if (q == 12) return make_float2(__fmul_rn(d.x + d.y, -h), __fmul_rn(d.x - d.y, h));
    return make_float2(__fmaf_rn(d.x, kC32[q], -__fmul_rn(d.y, kS32[q])), __fmaf_rn(d.y, kC32[q], __fmul_rn(d.x, kS32[q])));
}

// In-register inverse DFT of R points (sign +, unnormalised), decimation in frequency: natural
// order in, bit-reversed order out (the caller indexes the outputs through brev<R>).
template <int R> __device__ __forceinline__ constexpr int brev(int r) {
    int o = 0;
    for (int b = 1; b < R; b <<= 1) { o = (o << 1) | (r & 1); r >>= 1; }
    return o;
}

// With KEEP < R only the outputs X[0 .. KEEP) are produced (KEEP >= R/2): position g of the
// bit-reversed result holds X[brev(g)], so in the last stage the pair (g, g+1) holds X[r] and
// X[r + R/2], r = brev(g), and the subtraction is skipped when r + R/2 >= KEEP.
// Each stage is its own instantiation with a constant trip count: written as nested loops over h, g and a, the
// compiler left the inner loops of the radix-32 and radix-16 passes rolled, with v[] in local memory and the
// twiddles loaded from global memory in every butterfly.
template <int R, int KEEP, int H>
__device__ __forceinline__ void dft_dif_stage(float2 (&v)[R]) {
#pragma unroll
    for (int i = 0; i < R / 2; ++i) {
        const int g = (i / H) * (2 * H), a = i % H;
        const float2 x = v[g + a], y = v[g + a + H];
        v[g + a] = cadd(x, y);
        if (!(H == 1 && brev<R>(g) + R / 2 >= KEEP)) v[g + a + H] = rot32(csub(x, y), a * (16 / H));
    }
    if constexpr (H > 1) dft_dif_stage<R, KEEP, H / 2>(v);
}
template <int R, int KEEP = R>
__device__ __forceinline__ void dft_dif(float2 (&v)[R]) {
    static_assert(KEEP >= R / 2 && KEEP <= R, "KEEP out of range");
    dft_dif_stage<R, KEEP, R / 2>(v);
}

// one padding slot per 32 complex values keeps the radix-32 scatter of pass 1 conflict free
__device__ __forceinline__ int pad(int i) { return i + (i >> 5); }

// ---------------------------------------------------------------- exact per-lag value (fp64)
// OpenCV's rule for TM_SQDIFF_NORMED (imgproc/templmatch.cpp, common_matchTemplate; behaviour pinned by
// tests/golden): with corr the float32-rounded sum(I*T),
//   num = max(wnd - 2*corr + tsum2, 0);  t = sqrt(wnd) * sqrt(tsum2)  (t = 0 if wnd is ~0)
//   out = |num| < t ? num/t : 1           -> float32
// One rsqrt replaces the sqrt+divide pair: t = p*rsqrt(p), num/t = num*rsqrt(p), p = wnd*tsum2.
__device__ __forceinline__ float sqdiff_exact(double corr_centred, double wsum, double wsq,
                                              double a, double b, double tsum, double tsq, double n_ab) {
    const double sit = corr_centred + b * wsum + a * tsum - n_ab;
    const double corr = (double)(float)sit;          // OpenCV keeps sum(I*T) as float32
    double num = wsq - 2.0 * corr + tsq;
    num = fmax(num, 0.0);
    const double p = wsq * tsq;
    if (!(wsq > 0.0) || wsq <= fmin(0.5, 10.0 * 1.1920928955078125e-07 * wsq) || !(p > 0.0)) return 1.0f;
    const double r = rsqrt(p);
    const double t = p * r;
    return (num < t) ? (float)(num * r) : 1.0f;
}

template <typename S> struct Acc;
template <> struct Acc<uint8_t> {
    typedef int type;
    static __device__ __forceinline__ int sq(uint8_t hi, uint8_t lo) { return (int)hi * hi - (int)lo * lo; }
    static __device__ __forceinline__ int ln(uint8_t hi, uint8_t lo) { return (int)hi - (int)lo; }
    static __device__ __forceinline__ float centre(double sum, double cnt) { return (float)rint(sum / cnt); }
};
template <> struct Acc<float> {
    typedef double type;
    static __device__ __forceinline__ double sq(float hi, float lo) { return (double)hi * hi - (double)lo * lo; }
    static __device__ __forceinline__ double ln(float hi, float lo) { return (double)hi - (double)lo; }
    static __device__ __forceinline__ float centre(double sum, double cnt) { return (float)(sum / cnt); }
};

constexpr float kScreenMargin = 8e-6f;   // > 2 x fp32 screening error + one float32 ulp at 1.0

// 8 consecutive samples starting at element index e (any alignment) as one 64-bit word
__device__ __forceinline__ unsigned long long load8(const uint8_t* __restrict__ p, int64_t e) {
    const int64_t a8 = e & ~(int64_t)7;
    const unsigned sh = (unsigned)(e & 7) * 8u;
    const unsigned long long w0 = __ldg(reinterpret_cast<const unsigned long long*>(p + a8));
    if (sh == 0) return w0;
    const unsigned long long w1 = __ldg(reinterpret_cast<const unsigned long long*>(p + a8 + 8));
    return (w0 >> sh) | (w1 << (64u - sh));
}


}  // namespace sbf
