// MPEG audio layer II input: the frames of a Matroska A_MPEG/L2 track or of a transport stream's MPEG audio PID,
// decoded on the GPU into interleaved int16 PCM, FFmpeg's fixed-point `mp2` decoder bit for bit.
// mp2_decode (sb_mp2_decode_frames, and sb_ts_finish for SB_TS_MP2):
//   frame_table      host: the header chain (sb_mp2.cuh)
//   k_mp2_unpack     one thread per frame: allocations, SCFSI, scalefactors, samples, requantisation and CRC into
//                    subband-sample scratch, channel-major
//   k_mp2_dct        one thread per time slot of a channel: the 32-point DCT in place
//   k_mp2_window<0>  one CTA per frame and channel (288 threads, 4 slots a warp): the slots' synthesis rows and the 15
//                    rows before them staged in shared memory, every output's window sum; the CTA's sum of their low
//                    32 bits
//   k_mp2_tiles      one CTA: exclusive scan of those sums in FFmpeg's order (frame, then channel)
//   k_mp2_window<1>  the same sums again, scanned in emission order on top of the CTA's prefix: every output's
//                    rounding remainder, and the sample
// The per-frame arithmetic is in sb_mp2.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
#include "sb_mp2.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int kThreads = 256;
constexpr int kWinThreads = 288;                      // 9 warps, 4 slots each
constexpr int kRows = sbmp2::kSlots + 15;             // a frame's slots and the 15 its window reaches back to

__global__ void __launch_bounds__(kThreads)
k_mp2_unpack(const uint8_t* __restrict__ buf, int64_t nbytes, const sbmp2::Frame* __restrict__ frames, int64_t n,
             sbmp2::Scales sc, int32_t* __restrict__ sb, int32_t* __restrict__ status) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    status[k] = sbmp2::unpack_frame(buf, nbytes, frames[k], k, n, sc, sb);
}

__global__ void __launch_bounds__(kThreads)
k_mp2_dct(int32_t* __restrict__ sb, int64_t rows) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    int32_t in[32];
    const int4* p = reinterpret_cast<const int4*>(sb + r * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int4 q = p[i];
        in[4 * i] = q.x; in[4 * i + 1] = q.y; in[4 * i + 2] = q.z; in[4 * i + 3] = q.w;
    }
    int32_t out[32];
    sbmp2::dct32(out, in);
    int4* o = reinterpret_cast<int4*>(sb + r * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = make_int4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
}

struct SmemRows {
    const int32_t* rows;                               // row 0 is slot t0 - 15
    int64_t t0;
    __device__ int32_t operator()(int64_t t, int m) const { return rows[(t - t0 + 15) * 32 + m]; }
};

// kWrite 0: tile_sum[tile] = the CTA's outputs' window sums, summed mod 2^32.  kWrite 1: the outputs, with
// tile_sum[tile] now the exclusive prefix of those sums over the tiles before.
template <int kWrite>
__global__ void __launch_bounds__(kWinThreads)
k_mp2_window(const int32_t* __restrict__ v, int64_t n_frames, int channels, uint32_t* __restrict__ tile_sum,
             int16_t* __restrict__ pcm) {
    __shared__ int32_t rows[kRows * 32];
    __shared__ uint32_t warp_total[kWinThreads / 32];
    const int64_t tile = blockIdx.x;
    const int64_t f = tile / channels;
    const int c = (int)(tile % channels);
    const int64_t t0 = f * sbmp2::kSlots;
    const int32_t* base = v + (int64_t)c * n_frames * sbmp2::kFrameSamples;
    for (int i = threadIdx.x; i < kRows * 32; i += blockDim.x) {
        const int64_t t = t0 - 15 + i / 32;
        rows[i] = t < 0 ? 0 : base[t * 32 + (i & 31)];
    }
    __syncthreads();
    const SmemRows r{rows, t0};
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int j = sbmp2::emitted(lane);
    int64_t sum[4];
    uint32_t run = 0, before[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        sum[s] = sbmp2::window_sum(r, t0 + w * 4 + s, j);
        uint32_t x = (uint32_t)sum[s];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
            if (lane >= o) x += y;
        }
        before[s] = run + x - (uint32_t)sum[s];          // exclusive within the warp's slots
        run += __shfl_sync(0xFFFFFFFFu, x, 31);
    }
    if (lane == 0) warp_total[w] = run;
    __syncthreads();
    if (!kWrite) {
        if (threadIdx.x == 0) {
            uint32_t t = 0;
            for (int k = 0; k < kWinThreads / 32; ++k) t += warp_total[k];
            tile_sum[tile] = t;
        }
        return;
    }
    uint32_t prefix = tile_sum[tile];
    for (int k = 0; k < w; ++k) prefix += warp_total[k];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const int64_t t = t0 + w * 4 + s;
        pcm[(t * 32 + j) * channels + c] = sbmp2::round_sample(prefix + before[s], sum[s]);
    }
}

// exclusive scan of n uint32 in place (mod 2^32), one CTA
__global__ void __launch_bounds__(1024)
k_mp2_tiles(uint32_t* __restrict__ v, int64_t n) {
    __shared__ uint32_t warp_sums[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t base = 0;
    for (int64_t i0 = 0; i0 < n; i0 += blockDim.x) {
        const int64_t i = i0 + threadIdx.x;
        const uint32_t x0 = i < n ? v[i] : 0;
        uint32_t x = x0;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sums[w] = x;
        __syncthreads();
        if (w == 0) {
            uint32_t s = warp_sums[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, s, o);
                if (lane >= o) s += y;
            }
            warp_sums[lane] = s;
        }
        __syncthreads();
        if (i < n) v[i] = base + (w > 0 ? warp_sums[w - 1] : 0) + x - x0;
        base += warp_sums[31];
        __syncthreads();
    }
}

}  // namespace

namespace sb {

// Decode the MP2 stream in `host` (nbytes bytes), which is also on the device at d_buf with the zero tail of
// sb_decode.h.  where(b): the file offset of stream byte b, for messages.  *cut: 1 when the last frame is cut short (decoded with zeros).
int mp2_decode(const uint8_t* host, const uint8_t* d_buf, int64_t nbytes, const std::function<int64_t(int64_t)>& where,
               int32_t* cut, sb_pcm** out) {
    const char* who = "mp2_decode";
    Ctx& c = ctx();
    std::vector<sbmp2::Frame> frames;
    sbmp2::Stream s;
    char msg[256];
    if (!sbmp2::frame_table(host, nbytes, where, frames, &s, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    *cut = s.cut;
    const int64_t n = (int64_t)frames.size();
    if (n < 1) SB_FAIL(SB_EINVAL, "MP2 frame 0 at byte offset %lld: the only frame is not decoded (bytes before it)",
                       (long long)where(s.first));
    const int64_t rows = n * s.channels * sbmp2::kSlots;
    Blocks blocks;
    sbmp2::Frame* d_frames = nullptr;
    int32_t* d_sb = nullptr;
    int32_t* d_status = nullptr;
    uint32_t* d_tiles = nullptr;
    int16_t* d_pcm = nullptr;
    SB_TRY(blocks.alloc(&d_frames, (size_t)n));
    SB_TRY(blocks.alloc(&d_sb, (size_t)rows * 32));
    SB_TRY(blocks.alloc(&d_status, (size_t)n));
    SB_TRY(blocks.alloc(&d_tiles, (size_t)n * s.channels));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)n * sbmp2::kFrameSamples * s.channels));
    std::vector<int32_t> status((size_t)n);
    cudaError_t e = cudaMemcpyAsync(d_frames, frames.data(), sizeof(sbmp2::Frame) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("mp2_unpack");
        k_mp2_unpack<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, c.stream>>>(
            d_buf, nbytes, d_frames, n, sbmp2::make_scales(), d_sb, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, n, who));
    std::vector<int64_t> at((size_t)n);
    for (int64_t f = 0; f < n; ++f) at[(size_t)f] = where(frames[(size_t)f].offset);
    if (!sbframes::first_failure(status.data(), n, "MP2 frame", at.data(), 1, sbmp2::error_text, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    const unsigned tiles = (unsigned)(n * s.channels);
    {
        ProfScope ps("mp2_dct");
        k_mp2_dct<<<(unsigned)((rows + kThreads - 1) / kThreads), kThreads, 0, c.stream>>>(d_sb, rows);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("mp2_window", 3);
        k_mp2_window<0><<<tiles, kWinThreads, 0, c.stream>>>(d_sb, n, s.channels, d_tiles, d_pcm);
        k_mp2_tiles<<<1, 1024, 0, c.stream>>>(d_tiles, tiles);
        k_mp2_window<1><<<tiles, kWinThreads, 0, c.stream>>>(d_sb, n, s.channels, d_tiles, d_pcm);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    return pcm_handle(blocks.take(d_pcm), n * sbmp2::kFrameSamples, s.channels, s.rate, out);
}

}  // namespace sb

extern "C" {

int sb_mp2_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets,
                         int64_t n, sb_pcm** out) {
    const char* who = "sb_mp2_decode_frames";
    SB_TRY(entry_check(who, buf && offsets && file_offsets && out));
    if (nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_mp2_decode_frames: bad stream parameters");
    for (int64_t k = 0; k < n; ++k)
        if (offsets[k] < 0 || offsets[k] > nbytes || (k && offsets[k] < offsets[k - 1]))
            SB_FAIL(SB_EINVAL, "sb_mp2_decode_frames: block offsets out of order");
    const uint8_t* host = static_cast<const uint8_t*>(buf);
    // the blocks back to back, walked as one stream, then held to FFmpeg's one packet per block below; messages
    // name the file offset of the block holding a frame's header
    auto where = [&](int64_t b) -> int64_t {
        const int64_t k = std::upper_bound(offsets, offsets + n, b) - offsets - 1;
        return file_offsets[k < 0 ? 0 : k];
    };
    // FFmpeg decodes each block as a packet: a block must hold whole frames, the last one's end cut at most
    std::vector<sbmp2::Frame> frames;
    sbmp2::Stream st;
    char msg[256];
    if (!sbmp2::frame_table(host, nbytes, where, frames, &st, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    for (size_t f = 0, k = 0; k < (size_t)n; ++k) {
        const int64_t end = k + 1 < (size_t)n ? offsets[k + 1] : nbytes;
        if (offsets[k] == end) continue;
        if (f >= frames.size() || frames[f].offset != offsets[k])
            SB_FAIL(SB_EINVAL, "MP2 block at byte offset %lld: the block does not start with a frame header (FFmpeg "
                    "refuses such a block)", (long long)file_offsets[k]);
        while (f < frames.size() && frames[f].offset < end) {
            if (frames[f].offset + frames[f].size > end)
                SB_FAIL(SB_EINVAL, "MP2 frame %lld at byte offset %lld: the frame runs past its block (FFmpeg decodes "
                        "the blocks one by one)", (long long)f, (long long)where(frames[f].offset));
            ++f;
        }
    }
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, host, nbytes, who));
    int32_t cut = 0;
    return mp2_decode(host, d_buf, nbytes, where, &cut, out);
}

int sb_mp2_decode_stream(const void* buf, int64_t nbytes, int64_t file_offset, int32_t* cut, sb_pcm** out) {
    const char* who = "sb_mp2_decode_stream";
    SB_TRY(entry_check(who, buf && cut && out));
    if (nbytes < 1 || file_offset < 0) SB_FAIL(SB_EINVAL, "sb_mp2_decode_stream: bad stream parameters");
    const uint8_t* host = static_cast<const uint8_t*>(buf);
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, host, nbytes, who));
    return mp2_decode(host, d_buf, nbytes, [&](int64_t b) { return file_offset + b; }, cut, out);
}

}  // extern "C"
