// Monkey's Audio input: the frames of a raw .ape file (version 3.99), decoded on the GPU into the interleaved int16 PCM
// that sb_load_pcm decodes from a WAV file.  An APE frame holds up to 294 912 samples per channel, and at the higher
// compression levels each goes through up to three adaptive filters of up to 1280 taps, so the decode runs in FFmpeg's
// stage order, one kernel per stage, over an int32 scratch of every sample:
//   k_ape_entropy    one thread per frame: the frame header, then the range decoder's residuals, both channels
//                    interleaved as the stream codes them (serial within a frame);
//   k_ape_nn         one warp per (frame, coded channel): each NN filter of the level in turn over the channel, in
//                    place; the taps are spread across the lanes (lane l holds taps l, l + 32, ...), the dot product is
//                    a warp reduction, the weight update is lane-local, and the history and adapt values sit in a
//                    shared-memory ring per warp;
//   k_ape_predictor  one thread per frame: the predictor (which couples the two channels) and the decorrelation; the
//                    output samples back into the scratch, their top 16 bits at the frame's sample position;
//   k_ape_crc        one warp per frame: the CRC-32 of the frame's output bytes as 32 slices joined by the zlib combine
//                    rule, checked against the frame header.
// The per-frame arithmetic is in sb_ape.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
#include "sb_ape.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int kThreads = 32;
constexpr int kNnWarps = 4;
constexpr size_t kNnSmem = (size_t)kNnWarps * 2 * sbape::kRing * sizeof(int16_t);        // 32 KB

__global__ void __launch_bounds__(kThreads)
k_ape_entropy(const uint8_t* __restrict__ buf, const sbape::Frame* __restrict__ frames, int64_t n, sbape::Config c,
              int32_t* __restrict__ scratch, int32_t* __restrict__ kind, uint32_t* __restrict__ crc,
              int32_t* __restrict__ status) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    int32_t kd;
    uint32_t w = 0;
    status[k] = sbape::entropy_frame(buf, frames[k], c, scratch, &kd, &w);
    kind[k] = kd;
    crc[k] = w;
}

// One filter of `order` taps (T per lane) over `blocks` samples of one channel, in place.
template <int T>
__device__ void nn_filter(int32_t* __restrict__ d, int64_t stride, int32_t blocks, int order, int frac,
                          const sbape::NnShared& s, int lane) {
    for (int i = lane; i < sbape::kRing; i += 32) {
        s.hist[i] = 0;
        s.adapt[i] = 0;
    }
    int32_t w[T];
    SBA_UNROLL
    for (int k = 0; k < T; ++k) w[k] = 0;
    int32_t avg = 0;
    __syncwarp();
    for (int32_t base = 0; base < blocks; base += 32) {
        // 32 inputs at a time, one per lane, handed round by shuffles; each lane keeps the output of its own step
        const int32_t mine = base + lane < blocks ? d[(int64_t)(base + lane) * stride] : 0;
        int32_t out_mine = 0;
        const int m = min(32, blocks - base);
        for (int j = 0; j < m; ++j) {
            const int64_t t = base + j;
            const int32_t in = __shfl_sync(0xffffffffu, mine, j);
            const uint32_t part = sbape::lane_step<T>(w, lane, order, s, t, sbape::sign_neg(in));
            const uint32_t dot = __reduce_add_sync(0xffffffffu, part);
            int16_t h, a;
            const int32_t out = sbape::finish(dot, frac, in, avg, h, a);
            __syncwarp();
            if (lane == 0) {
                s.hist[t & (sbape::kRing - 1)] = h;
                s.adapt[t & (sbape::kRing - 1)] = a;
            }
            if (lane == j) out_mine = out;
            __syncwarp();
        }
        if (lane < m) d[(int64_t)(base + lane) * stride] = out_mine;
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kNnWarps * 32)
k_ape_nn(const sbape::Frame* __restrict__ frames, int64_t n, sbape::Config c, int32_t* __restrict__ scratch,
         const int32_t* __restrict__ kind, const int32_t* __restrict__ status) {
    extern __shared__ int16_t nn_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t job = (int64_t)blockIdx.x * kNnWarps + warp;
    if (job >= n * c.channels) return;
    const int64_t f = job / c.channels;
    const int ch = (int)(job % c.channels);
    if (status[f] != sbape::kOk || kind[f] == sbape::kSilence || (kind[f] == sbape::kMono && ch > 0)) return;
    sbape::NnShared s;
    s.hist = nn_smem + (size_t)warp * 2 * sbape::kRing;
    s.adapt = s.hist + sbape::kRing;
    const sbape::Frame fr = frames[f];
    int32_t* d = scratch + fr.sample * c.channels + ch;
    for (int l = 0; l < sbape::kLevels; ++l) {
        const int order = sbape::filter_order(c.fset, l), frac = sbape::filter_frac(c.fset, l);
        if (!order) break;
        switch (order) {
        case 16: nn_filter<1>(d, c.channels, fr.blocks, order, frac, s, lane); break;
        case 32: nn_filter<1>(d, c.channels, fr.blocks, order, frac, s, lane); break;
        case 64: nn_filter<2>(d, c.channels, fr.blocks, order, frac, s, lane); break;
        case 256: nn_filter<8>(d, c.channels, fr.blocks, order, frac, s, lane); break;
        default: nn_filter<40>(d, c.channels, fr.blocks, order, frac, s, lane); break;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_ape_predictor(const sbape::Frame* __restrict__ frames, int64_t n, sbape::Config c, int32_t* __restrict__ scratch,
                const int32_t* __restrict__ kind, int16_t* __restrict__ pcm, int32_t* __restrict__ status) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n || status[k] != sbape::kOk) return;
    status[k] = sbape::predictor_frame(frames[k], c, kind[k], scratch, pcm);
}

__global__ void __launch_bounds__(kThreads)
k_ape_crc(const sbape::Frame* __restrict__ frames, int64_t n, sbape::Config c, const int32_t* __restrict__ scratch,
          const uint32_t* __restrict__ stored, int32_t* __restrict__ status) {
    __shared__ uint32_t table[256];
    const int lane = threadIdx.x;
    for (int i = lane; i < 256; i += 32) table[i] = sbape::crc_entry((uint32_t)i);
    __syncwarp();
    const int64_t f = blockIdx.x;
    if (status[f] != sbape::kOk) return;
    const sbape::Frame fr = frames[f];
    const int64_t total = (int64_t)fr.blocks * c.channels;
    const int64_t per = (total + 31) / 32;
    const int64_t lo = min(total, per * lane), hi = min(total, lo + per);
    uint32_t crc = sbape::crc_bytes(scratch + fr.sample * c.channels, lo, hi, c.bits, table);
    int64_t len = (hi - lo) * (c.bits / 8);
    // join the slices pairwise: lane l takes lane l + s's CRC and length when l is a multiple of 2 s
    for (int s = 1; s < 32; s <<= 1) {
        const uint32_t rc = __shfl_down_sync(0xffffffffu, crc, s);
        const int64_t rl = __shfl_down_sync(0xffffffffu, len, s);
        if ((lane & (2 * s - 1)) == 0 && lane + s < 32) {
            crc = rl ? sbape::crc_combine(crc, rc, rl) : crc;
            len += rl;
        }
    }
    if (lane == 0) status[f] = sbape::check_crc(crc, stored[f]);
}

}  // namespace

extern "C" {

int sb_ape_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                         const int32_t* config, sb_pcm** out) {
    const char* who = "sb_ape_decode_frames";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, buf && offsets && file_offsets && config && out));
    sbape::Config cfg;
    int32_t rate = 0;
    char msg[256];
    if (!sbape::parse_config(config, &cfg, &rate, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    if (nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_ape_decode_frames: bad stream parameters");
    std::vector<sbape::Frame> frames;
    int64_t samples = 0;
    if (!sbape::frame_table(offsets, file_offsets, n, nbytes, cfg, frames, &samples, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    sbape::Frame* d_frames = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t *d_scratch = nullptr, *d_kind = nullptr, *d_status = nullptr;
    uint32_t* d_crc = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, buf, nbytes, who));
    SB_TRY(blocks.alloc(&d_frames, (size_t)n));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)samples * cfg.channels));
    SB_TRY(blocks.alloc(&d_scratch, (size_t)samples * cfg.channels));
    SB_TRY(blocks.alloc(&d_kind, (size_t)n));
    SB_TRY(blocks.alloc(&d_crc, (size_t)n));
    SB_TRY(blocks.alloc(&d_status, (size_t)n));
    std::vector<int32_t> status((size_t)n);
    const unsigned grid = (unsigned)((n + kThreads - 1) / kThreads);
    cudaError_t e = cudaFuncSetAttribute(k_ape_nn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kNnSmem);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(d_frames, frames.data(), sizeof(sbape::Frame) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("ape_entropy");
        k_ape_entropy<<<grid, kThreads, 0, c.stream>>>(d_buf, d_frames, n, cfg, d_scratch, d_kind, d_crc, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && sbape::filter_order(cfg.fset, 0)) {
        ProfScope ps("ape_nn");
        const int64_t jobs = n * cfg.channels;
        k_ape_nn<<<(unsigned)((jobs + kNnWarps - 1) / kNnWarps), kNnWarps * 32, kNnSmem, c.stream>>>(
            d_frames, n, cfg, d_scratch, d_kind, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("ape_predictor");
        k_ape_predictor<<<grid, kThreads, 0, c.stream>>>(d_frames, n, cfg, d_scratch, d_kind, d_pcm, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("ape_crc");
        k_ape_crc<<<(unsigned)n, 32, 0, c.stream>>>(d_frames, n, cfg, d_scratch, d_crc, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, n, who));
    if (!sbframes::first_failure(status.data(), n, "APE frame", file_offsets, 1, sbape::error_text, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return pcm_handle(blocks.take(d_pcm), samples, cfg.channels, rate, out);
}

}  // extern "C"
