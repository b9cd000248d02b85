// Shared-memory FFT machinery of the fused engines: geometry, twiddle tables and the in-place
// Stockham inverse transform of N = B = 16384 complex points (used by sb_fused.cu and, for the
// forward spectra, sb_fused2.cu).
#pragma once
#include "sb_fused_common.cuh"

namespace sbf {

// ---------------------------------------------------------------- configuration
template <int LOG2N> struct Cfg;
template <> struct Cfg<14> {   // B = 16384 lags per item
    static constexpr int N = 16384, T = 512, R1 = 32, R2 = 32, R3 = 16, MINB = 1;
};

struct FusedTables {
    const float2* w;      // [N/2+1]   exp(+i*pi*m/N)            (Hermitian unpacking)
    const float2* t2;     // [R2][32]  exp(+2*pi*i*r*k/(32*R2))   (pass 2, k = lane)
    const float2* a3;     // [R3][32]  exp(+2*pi*i*r*k/N), k = lane            (pass 3, low part)
    const float2* b3;     // [R3][32]  exp(+2*pi*i*r*kh*32/N), kh = k / 32     (pass 3, high part)
};

// ---------------------------------------------------------------- the FFT
// Unnormalised inverse DFT (sign +) of N complex points held in shared memory in the padded layout
// buf[pad(i)].  Stockham passes: butterfly j reads in[j + r*N/R], twiddles by exp(2*pi*i*r*k/(Ns*R)),
// k = j mod Ns, and writes out[(j-k)*R + k + r*Ns]; every value sits in a register between the two
// barriers of a pass, so the transform is in place and the output is in natural order.
// Must be entered after a barrier that made buf visible; ends with a barrier.
template <int KEEP3, bool FUSED>
__device__ __forceinline__ void ifft_smem(float2* __restrict__ buf, const float2* __restrict__ s_t2,
                                          const float2* __restrict__ s_a3, const float2* __restrict__ s_b3) {
    typedef Cfg<14> C;
    constexpr int N = C::N, T = C::T;
    const int tid = threadIdx.x, lane = tid & 31;
    // Stockham passes: butterfly j reads in[j + r*N/R], twiddles by exp(2*pi*i*r*k/(Ns*R)),
    // k = j mod Ns, and writes out[(j-k)*R + k + r*Ns]; every value sits in a register between
    // the two barriers, so the pass is in place.
    {   // pass 1: R1 = 32, Ns = 1 (no twiddles); one butterfly per thread
        constexpr int R = C::R1;
        static_assert(N / R == T, "pass 1: one butterfly per thread");
        float2 v[R];
        // pad(i + 32c) = pad(i) + 33c: every address below is one base plus a compile-time offset
        {
            const float2* src = buf + pad(tid);
#pragma unroll
            for (int r = 0; r < R; ++r) v[r] = src[r * ((N / R) + (N / R) / 32)];
        }
        __syncthreads();
        dft_dif<R>(v);
        {
            float2* dst = buf + tid * (R + 1);              // pad(tid*32 + r) = 33*tid + r
#pragma unroll
            for (int r = 0; r < R; ++r) dst[r] = v[brev<R>(r)];
        }
        __syncthreads();
    }
    {   // pass 2: Ns = 32, k = lane
        constexpr int R = C::R2, Ns = C::R1, PER = (N / R) / T;
        float2 v[PER][R];
#pragma unroll
        for (int b = 0; b < PER; ++b)
#pragma unroll
            for (int r = 0; r < R; ++r) v[b][r] = buf[pad(tid) + (b * T + r * (N / R)) / 32 * 33];
        __syncthreads();
#pragma unroll
        for (int b = 0; b < PER; ++b) {
            const int j = tid + b * T;
#pragma unroll
            for (int r = 1; r < R; ++r) v[b][r] = cmul(v[b][r], s_t2[r * 32 + lane]);
            dft_dif<R>(v[b]);
            const int j0 = (j - lane) * R + lane;
#pragma unroll
            for (int r = 0; r < R; ++r) buf[pad(j0) + r * (Ns / 32 * 33)] = v[b][brev<R>(r)];
        }
        __syncthreads();
    }
    {   // pass 3: Ns = R1*R2, k = j (j < Ns).  Only outputs r < KEEP3 of each butterfly are needed
        // (the fused kernel reads z[0 .. LB/2): the valid lags of the 2B-point real sequence)
        constexpr int R = C::R3, Ns = C::R1 * C::R2, PER = (N / R) / T;
        static_assert(N / R == Ns, "pass 3 is the last pass");
        float2 v[PER][R];
#pragma unroll
        for (int b = 0; b < PER; ++b)
#pragma unroll
            for (int r = 0; r < R; ++r) v[b][r] = buf[pad(tid) + (b * T + r * (N / R)) / 32 * 33];
        __syncthreads();
#pragma unroll
        for (int b = 0; b < PER; ++b) {
            const int j = tid + b * T;
            const int kh = j >> 5;
#pragma unroll
            for (int r = 1; r < R; ++r)
                v[b][r] = cmul(v[b][r], cmul(s_a3[r * 32 + lane], s_b3[r * 32 + kh]));
            dft_dif<R, KEEP3>(v[b]);
#pragma unroll
            for (int r = 0; r < KEEP3; ++r) buf[pad(tid) + (b * T + r * Ns) / 32 * 33] = v[b][brev<R>(r)];
        }
        if (FUSED) cp_async_commit_wait_all();      // the fused kernel's staged copies landed long ago; the barrier publishes them
        __syncthreads();
    }
}

}  // namespace sbf

namespace sb {
// device-resident twiddle tables of Cfg<14>; built on first use
int fused_tables(sbf::FusedTables* out);
}
