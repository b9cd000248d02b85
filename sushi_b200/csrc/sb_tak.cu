// TAK input: the frames of a raw .tak file, decoded on the GPU into the interleaved int16 PCM that sb_load_pcm decodes
// from a WAV file.  A TAK frame holds up to 16384 samples per channel, each channel coded as subframes with prediction
// filters of up to 256 taps, so the decode runs in FFmpeg's stage order, one kernel per stage, over an int32 scratch of
// every sample:
//   k_tak_sync       every byte position where FFmpeg's tak parser starts a frame (sync word, a header that parses,
//                    its CRC-24); the host chains them into the frame table (sbtak::frame_table);
//   k_tak_entropy    one thread per frame: the residual codes of every channel into the scratch, planar per frame,
//                    and where each filtered subframe's and each decorrelated pair's parameters start (serial within a
//                    frame);
//   k_tak_filter     one warp per (frame, channel): each filtered subframe in turn, in place: the predictors turned
//                    into the filter across the lanes, then the filter (lane l holds taps l, l + 32, ...; the dot
//                    product is a warp reduction in 32-bit wrap-around; the int16 history sits in a shared-memory ring
//                    per warp);
//   k_tak_finish     one CTA per frame: the decorrelation pairs in list order and the channel lpc modes as nested block
//                    scans, all sample-parallel, then the sample shift and the int16 store;
//   k_tak_crc        one warp per frame: the CRC-24 of the frame's data as 32 slices joined by the combine rule,
//                    checked against the stored CRC.
// The per-frame arithmetic is in sb_tak.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
#include "sb_tak.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int kThreads = 32;
constexpr int kFilterWarps = 4;
constexpr int kFinishThreads = 256;

__global__ void __launch_bounds__(256)
k_tak_sync(const uint8_t* __restrict__ file, int64_t start, int64_t end, sbtak::Config c,
           sbtak::Candidate* __restrict__ out, unsigned long long* __restrict__ count, int64_t cap) {
    const int64_t words = (end + 3) >> 2;                          // the buffer is zero-padded past its bytes
    for (int64_t w = (start >> 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < words;
         w += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(file) + w);
        if (!(((v & 0xFF) == 0xFF) | (((v >> 8) & 0xFF) == 0xFF) | (((v >> 16) & 0xFF) == 0xFF) | ((v >> 24) == 0xFF)))
            continue;
        for (int k = 0; k < 4; ++k) {
            const int64_t i = 4 * w + k;
            if (i < start || ((v >> (8 * k)) & 0xFF) != 0xFF) continue;
            sbtak::Candidate h;
            if (!sbtak::parse_header(file, end, i, c, &h)) continue;
            const unsigned long long slot = atomicAdd(count, 1ull);
            if ((int64_t)slot < cap) out[slot] = h;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_tak_entropy(const uint8_t* __restrict__ file, int64_t nbytes, const sbtak::Frame* __restrict__ frames, int64_t n,
              sbtak::Config c, int32_t* __restrict__ scratch, sbtak::Sub* __restrict__ subs,
              sbtak::State* __restrict__ state, int32_t* __restrict__ status) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    sbtak::State s;
    status[f] = sbtak::entropy_frame(file, nbytes, frames[f], c, scratch,
                                     subs + f * c.channels * sbtak::kMaxSubframes, &s);
    state[f] = s;
}

struct FilterSmem {
    int16_t ring[sbtak::kRing];
    int16_t filter[sbtak::kMaxOrder];
    int16_t pred[sbtak::kMaxOrder];
    int32_t t[sbtak::kMaxOrder];
};

// one filtered subframe of channel d, in place, by one warp
__device__ void filter_sub(const uint8_t* __restrict__ file, int64_t nbytes, const sbtak::Sub& u, int32_t* __restrict__ d,
                           FilterSmem& s, int lane) {
    const int order = u.order;
    sbtak::FilterParams p;
    int st = 0;
    if (lane == 0) st = sbtak::read_filter(file, nbytes, u.bits, order, s.pred, &p);
    st = __shfl_sync(0xffffffffu, st, 0);
    p.dshift = __shfl_sync(0xffffffffu, p.dshift, 0);
    p.quant = __shfl_sync(0xffffffffu, p.quant, 0);
    (void)st;                                          // the entropy stage read the same bits without fault
    __syncwarp();
    // the predictors' filter: FFmpeg's recurrence, the pairs of each step across the lanes
    if (lane == 0 && order > 0) s.t[0] = s.pred[0] * 64;
    __syncwarp();
    for (int i = 1; i < order; ++i) {
        for (int j = lane; j < (i + 1) / 2; j += 32) sbtak::taps_pair(s.t, i, j, s.pred[i]);
        if (lane == 0) s.t[i] = s.pred[i] * 64;
        __syncwarp();
    }
    for (int k = lane; k < order; k += 32) s.filter[k] = sbtak::tap(s.t, order, p.quant, k);
    for (int k = lane; k < order; k += 32) s.ring[k] = (int16_t)(d[u.hist + k] >> p.dshift);
    __syncwarp();
    int32_t* out = d + u.hist + order;
    for (int base = 0; base < u.count; base += 32) {
        // 32 residuals at a time, one per lane, handed round by shuffles; each lane keeps the output of its own step
        const int32_t mine = base + lane < u.count ? out[base + lane] : 0;
        int32_t out_mine = 0;
        const int m = min(32, u.count - base);
        for (int j = 0; j < m; ++j) {
            const int64_t t = base + j;
            const int32_t resid = __shfl_sync(0xffffffffu, mine, j);
            const uint32_t dot = __reduce_add_sync(0xffffffffu, sbtak::lane_part(s.ring, s.filter, order, t, lane));
            const int32_t v = sbtak::finish_sample(dot, p.quant, p.dshift, resid);
            if (lane == 0) s.ring[(t + order) & (sbtak::kRing - 1)] = (int16_t)(v >> p.dshift);
            if (lane == j) out_mine = v;
            __syncwarp();
        }
        if (lane < m) out[base + lane] = out_mine;
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kFilterWarps * 32)
k_tak_filter(const uint8_t* __restrict__ file, int64_t nbytes, const sbtak::Frame* __restrict__ frames, int64_t n,
             sbtak::Config c, int32_t* __restrict__ scratch, const sbtak::Sub* __restrict__ subs,
             const sbtak::State* __restrict__ state, const int32_t* __restrict__ status) {
    __shared__ FilterSmem smem[kFilterWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t job = (int64_t)blockIdx.x * kFilterWarps + warp;
    if (job >= n * c.channels) return;
    const int64_t f = job / c.channels;
    const int ch = (int)(job % c.channels);
    if (status[f] != sbtak::kOk) return;
    const int nsub = state[f].nsub[ch];
    const sbtak::Frame fr = frames[f];
    int32_t* d = scratch + fr.sample * c.channels + (int64_t)ch * fr.nb;
    const sbtak::Sub* u = subs + (f * c.channels + ch) * sbtak::kMaxSubframes;
    for (int k = 0; k < nsub; ++k) filter_sub(file, nbytes, u[k], d, smem[warp], lane);
}

// inclusive prefix sum of d[lo, hi) in 32-bit wrap-around, by the whole CTA
__device__ void block_scan(int32_t* __restrict__ d, int lo, int hi, uint32_t* __restrict__ warp_sums) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int len = hi - lo, per = (len + kFinishThreads - 1) / kFinishThreads;
    const int a = min(hi, lo + tid * per), b = min(hi, a + per);
    uint32_t sum = 0;
    for (int i = a; i < b; ++i) sum += (uint32_t)d[i];
    uint32_t inc = sum;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    uint32_t acc = inc - sum;
    for (int w = 0; w < warp; ++w) acc += warp_sums[w];
    for (int i = a; i < b; ++i) {
        acc += (uint32_t)d[i];
        d[i] = (int32_t)acc;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kFinishThreads)
k_tak_finish(const uint8_t* __restrict__ file, int64_t nbytes, const sbtak::Frame* __restrict__ frames, sbtak::Config c,
             int32_t* __restrict__ scratch, const sbtak::State* __restrict__ state, const int32_t* __restrict__ status,
             int16_t* __restrict__ pcm) {
    __shared__ sbtak::Decor dec;
    __shared__ uint32_t warp_sums[kFinishThreads / 32];
    const int64_t f = blockIdx.x;
    if (status[f] != sbtak::kOk) return;
    const sbtak::Frame fr = frames[f];
    const int nb = fr.nb;
    int32_t* base = scratch + fr.sample * c.channels;
    const sbtak::State& s = state[f];
    if (!s.raw) {
        for (int k = 0; k < s.npairs; ++k) {
            if (threadIdx.x == 0) sbtak::read_decor(file, nbytes, s.pair[k], &dec);
            __syncthreads();
            int32_t* a = base + (int64_t)s.pair[k].c1 * nb;
            int32_t* b = base + (int64_t)s.pair[k].c2 * nb;
            for (int i = threadIdx.x; i < nb; i += kFinishThreads) sbtak::decorrelate_sample(dec, a, b, nb, i);
            __syncthreads();
        }
        for (int ch = 0; ch < c.channels; ++ch) {
            const int mode = s.lpc[ch];
            if (nb < 2) continue;
            for (int l = 1; l <= mode; ++l) block_scan(base + (int64_t)ch * nb, mode - l, nb, warp_sums);
        }
    }
    for (int64_t k = threadIdx.x; k < (int64_t)nb * c.channels; k += kFinishThreads) {
        const int i = (int)(k / c.channels), ch = (int)(k % c.channels);
        pcm[(fr.sample + i) * c.channels + ch] = sbtak::store(base[(int64_t)ch * nb + i], s.raw ? 0 : s.shift[ch], c.bits);
    }
}

__global__ void __launch_bounds__(32)
k_tak_crc(const uint8_t* __restrict__ file, const sbtak::Frame* __restrict__ frames, const sbtak::State* __restrict__ state,
          int32_t* __restrict__ status) {
    __shared__ uint32_t table[256];
    const int lane = threadIdx.x;
    for (int i = lane; i < 256; i += 32) table[i] = sbtak::crc_entry((uint32_t)i);
    __syncwarp();
    const int64_t f = blockIdx.x;
    if (status[f] != sbtak::kOk) return;
    const sbtak::Frame fr = frames[f];
    const int64_t lo0 = fr.start + fr.hsize, hi0 = state[f].data_end - 3, total = hi0 - lo0;
    const int64_t per = (total + 31) / 32;
    const int64_t lo = lo0 + min(total, per * lane), hi = min(hi0, lo + per);
    uint32_t crc = sbtak::crc_bytes(file, lo, hi, lane == 0 ? sbtak::kCrcInit : 0u, table);
    int64_t len = hi - lo;
    // join the slices pairwise: lane l takes lane l + s's CRC and length when l is a multiple of 2 s
    for (int s = 1; s < 32; s <<= 1) {
        const uint32_t rc = __shfl_down_sync(0xffffffffu, crc, s);
        const int64_t rl = __shfl_down_sync(0xffffffffu, len, s);
        if ((lane & (2 * s - 1)) == 0 && lane + s < 32) {
            crc = rl ? sbtak::crc_combine(crc, rc, rl) : crc;
            len += rl;
        }
    }
    if (lane == 0 && crc != sbtak::stored_crc(file + hi0)) status[f] = sbtak::kCrc;
}

}  // namespace

extern "C" {

int sb_tak_decode_file(const void* file, int64_t nbytes, int64_t audio_start, int64_t audio_end, const int32_t* config,
                       sb_pcm** out) {
    const char* who = "sb_tak_decode_file";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, file && config && out));
    sbtak::Config cfg;
    char msg[256];
    if (!sbtak::parse_config(config, &cfg, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    if (nbytes < 1 || audio_start < 0 || audio_end <= audio_start || audio_end > nbytes)
        SB_FAIL(SB_EINVAL, "sb_tak_decode_file: bad stream parameters");
    Blocks blocks;
    uint8_t* d_file = nullptr;
    SB_TRY(upload_padded(blocks, &d_file, file, nbytes, who));

    // candidates: a frame has at least 11 bytes; real files hold one frame per few kB and false syncs are rarer still
    std::vector<sbtak::Candidate> cand;
    SB_TRY(scan_candidates(nbytes / 256 + 4096, "tak_sync", who, [&](sbtak::Candidate* d_cand, unsigned long long* d_count, int64_t cap) {
        const int64_t words = (audio_end - audio_start + 3) / 4 + 1;
        const int grid = (int)std::min<int64_t>((words + 255) / 256, (int64_t)c.sm_count * 16);
        k_tak_sync<<<std::max(grid, 1), 256, 0, c.stream>>>(d_file, audio_start, audio_end, cfg, d_cand, d_count, cap);
    }, cand));
    std::sort(cand.begin(), cand.end(),
              [](const sbtak::Candidate& a, const sbtak::Candidate& b) { return a.offset < b.offset; });
    std::vector<sbtak::Frame> frames;
    int64_t samples = 0;
    if (!sbtak::frame_table(cand.data(), (int64_t)cand.size(), audio_start, audio_end, cfg, frames, &samples, msg,
                            sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    const int64_t n = (int64_t)frames.size();
    std::vector<int64_t> where((size_t)n);
    for (int64_t f = 0; f < n; ++f) where[(size_t)f] = frames[(size_t)f].start;

    sbtak::Frame* d_frames = nullptr;
    sbtak::Sub* d_subs = nullptr;
    sbtak::State* d_state = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t *d_scratch = nullptr, *d_status = nullptr;
    SB_TRY(blocks.alloc(&d_frames, (size_t)n));
    SB_TRY(blocks.alloc(&d_subs, (size_t)n * cfg.channels * sbtak::kMaxSubframes));
    SB_TRY(blocks.alloc(&d_state, (size_t)n));
    SB_TRY(blocks.alloc(&d_scratch, (size_t)samples * cfg.channels));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)samples * cfg.channels));
    SB_TRY(blocks.alloc(&d_status, (size_t)n));
    std::vector<int32_t> status((size_t)n);
    cudaError_t e = cudaMemcpyAsync(d_frames, frames.data(), sizeof(sbtak::Frame) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("tak_entropy");
        k_tak_entropy<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, c.stream>>>(
            d_file, nbytes, d_frames, n, cfg, d_scratch, d_subs, d_state, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("tak_filter");
        const int64_t jobs = n * cfg.channels;
        k_tak_filter<<<(unsigned)((jobs + kFilterWarps - 1) / kFilterWarps), kFilterWarps * 32, 0, c.stream>>>(
            d_file, nbytes, d_frames, n, cfg, d_scratch, d_subs, d_state, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("tak_finish");
        k_tak_finish<<<(unsigned)n, kFinishThreads, 0, c.stream>>>(d_file, nbytes, d_frames, cfg, d_scratch, d_state,
                                                                   d_status, d_pcm);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("tak_crc");
        k_tak_crc<<<(unsigned)n, 32, 0, c.stream>>>(d_file, d_frames, d_state, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, n, who));
    if (!sbframes::first_failure(status.data(), n, "TAK frame", where.data(), 1, sbtak::error_text, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return pcm_handle(blocks.take(d_pcm), samples, cfg.channels, cfg.rate, out);
}

}  // extern "C"
