// sb_pcm_swr: the ffmpeg command line's `-ac 1 -ar <rate>` conversion of a decoded sb_pcm (sb_swr.cuh has the
// arithmetic and what it is pinned to).
//   swr_mix       equal rates: one thread per frame, the integer Q15 downmix of its interleaved samples
//   swr_resample  a CTA per tile of outputs: per channel of the mono row, the tile's input window (mirrored edges
//                 included) is staged in shared memory as float, each thread filters its output from it with the bank
//                 row of its phase (global memory, read through the read-only cache), and the remix accumulates in
//                 registers; the last channel's pass writes int16.
#include "sb_internal.h"
#include "sb_swr.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int kSmemBytes = 48 * 1024;

__global__ void __launch_bounds__(256)
k_swr_mix(const int16_t* __restrict__ in, int64_t frames, sbswr::Mix mix, int16_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < frames; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = sbswr::mix_int(in + i * mix.channels, mix);
}

__global__ void __launch_bounds__(256)
k_swr_resample(const int16_t* __restrict__ in, sbswr::Plan p, const float* __restrict__ bank,
               int16_t* __restrict__ out) {
    extern __shared__ float win[];
    const int tile = blockDim.x;
    const int64_t t0 = (int64_t)blockIdx.x * tile;
    const int64_t t = t0 + threadIdx.x;
    const int64_t last = (t0 + tile < p.out_frames ? t0 + tile : p.out_frames) - 1;
    int64_t s0, s1, s, frac, f;
    int phase;
    sbswr::position(p.rs, t0, &s0, &phase, &frac);
    sbswr::position(p.rs, last, &s1, &phase, &frac);
    sbswr::position(p.rs, t, &s, &phase, &frac);
    const int width = (int)(s1 - s0) + p.rs.filter_alloc;
    float v = 0.f;
    for (int k = 0; k < p.mix.count; ++k) {
        const int c = p.mix.index[k];
        if (k) __syncthreads();
        for (int i = threadIdx.x; i < width; i += tile) {
            f = sbswr::source_frame(p, s0 + i);
            win[i] = f < 0 ? 0.f : (float)in[f * p.channels + c] * (1.0f / 32768);
        }
        __syncthreads();
        if (t <= last) {
            const float y = sbswr::resample_one(p.rs, bank, win + (s - s0), phase, frac);
            v = sbswr::fadd(v, sbswr::fmul(y, p.mix.flt[c]));
        }
    }
    if (t <= last) out[t] = sbswr::to_s16(v);
}

}  // namespace

extern "C" int sb_pcm_swr(const sb_pcm* in, uint64_t layout, int out_rate, sb_pcm** out) {
    Ctx& c = ctx();
    const char* who = "sb_pcm_swr";
    if (!c.inited) SB_FAIL(SB_ESTATE, "%s: library not initialised (call sb_init)", who);
    if (!in || !out) SB_FAIL(SB_EINVAL, "%s: NULL argument", who);
    sbswr::Plan p;
    char msg[160];
    if (!sbswr::make_plan(layout, in->channels, in->rate, out_rate, in->frames, &p, msg, sizeof msg))
        SB_FAIL(SB_EINVAL, "%s: %s", who, msg);
    int tile = 256, width = 0;
    if (p.resample) {
        for (; tile >= 32; tile /= 2) {                      // the widest window any tile of `tile` outputs stages
            const int64_t span = ((int64_t)(tile - 1) * p.rs.dst_incr / p.rs.src_incr) / p.rs.phase_count + 2;
            if ((span + p.rs.filter_alloc) * (int64_t)sizeof(float) <= kSmemBytes) {
                width = (int)(span + p.rs.filter_alloc);
                break;
            }
        }
        if (!width)
            SB_FAIL(SB_EINVAL, "%s: sample rates %d -> %d need too wide a filter window", who, in->rate, out_rate);
    }
    int16_t* d_out = nullptr;
    float* d_bank = nullptr;
    SB_TRY(pool_alloc((void**)&d_out, sizeof(int16_t) * (size_t)p.out_frames + 16));
    cudaError_t e = cudaSuccess;
    const int64_t n = p.out_frames;
    std::vector<float> bank;
    if (!p.resample && n > 0) {
        ProfScope ps("swr_mix");
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)c.sm_count * 16));
        k_swr_mix<<<grid, 256, 0, c.stream>>>(in->d_pcm, n, p.mix, d_out);
        e = cudaGetLastError();
    } else if (n > 0) {
        sbswr::float_bank(p.rs, bank);
        int rc = pool_alloc((void**)&d_bank, sizeof(float) * bank.size() + 16);
        if (rc != SB_OK) { pool_free(d_out); return rc; }
        e = cudaMemcpyAsync(d_bank, bank.data(), sizeof(float) * bank.size(), cudaMemcpyHostToDevice, c.stream);
        if (e == cudaSuccess) {
            ProfScope ps("swr_resample");
            const int64_t grid = (n + tile - 1) / tile;
            k_swr_resample<<<(unsigned)grid, tile, sizeof(float) * width, c.stream>>>(in->d_pcm, p, d_bank, d_out);
            e = cudaGetLastError();
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);           // before the host bank goes
    pool_free(d_bank);
    if (e != cudaSuccess) { pool_free(d_out); SB_FAIL(SB_ECUDA, "%s: %s", who, cudaGetErrorString(e)); }
    return pcm_handle(d_out, n, 1, out_rate, out);
}
