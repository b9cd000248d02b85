// TTA input: the frames of a raw .tta file or a Matroska A_TTA1 track, decoded on the GPU into the interleaved int16
// PCM that sb_load_pcm decodes from a WAV file.
// sb_tta_decode_frames:
//   k_tta_decode   one thread per frame: every sample through the Rice code, the filter and the predictor, channel by
//                  channel, then the decorrelation and the top-16-bit store at the frame's sample position; then the
//                  frame's CRC-32.  Each thread keeps its channels' state in a column of shared memory, and its CTA
//                  shares one slice-by-4 CRC table there; nothing is kept per frame in global scratch, so every frame
//                  goes in one launch.
// The per-frame arithmetic is in sb_tta.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
#include "sb_tta.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int kThreads = 32;

size_t smem_bytes(int channels) {
    return sizeof(uint32_t) * (sbtta::kCrcWords + (size_t)kThreads * channels * sbtta::kStateWords);
}

__global__ void __launch_bounds__(kThreads)
k_tta_decode(const uint8_t* __restrict__ buf, const sbtta::Frame* __restrict__ frames, int64_t n, sbtta::Config c,
             int16_t* __restrict__ pcm, int32_t* __restrict__ status) {
    extern __shared__ uint32_t smem[];
    uint32_t* crc = smem;
    for (int i = threadIdx.x; i < sbtta::kCrcWords; i += blockDim.x) sbtta::crc_table_entry(crc, i);
    __syncthreads();
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    sbtta::State s;
    s.p = (int32_t*)(smem + sbtta::kCrcWords) + threadIdx.x;
    s.stride = blockDim.x;
    status[k] = sbtta::decode_frame(buf, frames[k], c, s, crc, pcm);
}

}  // namespace

extern "C" {

int sb_tta_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                         const int32_t* config, sb_pcm** out) {
    const char* who = "sb_tta_decode_frames";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, buf && offsets && file_offsets && config && out));
    sbtta::Config cfg;
    int32_t rate = 0;
    char msg[256];
    if (!sbtta::parse_config(config, &cfg, &rate, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    if (nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_tta_decode_frames: bad stream parameters");
    std::vector<sbtta::Frame> frames;
    int64_t samples = 0;
    if (!sbtta::frame_table(offsets, file_offsets, n, nbytes, cfg, frames, &samples, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    sbtta::Frame* d_frames = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, buf, nbytes, who));
    SB_TRY(blocks.alloc(&d_frames, (size_t)n));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)samples * cfg.channels));
    SB_TRY(blocks.alloc(&d_status, (size_t)n));
    std::vector<int32_t> status((size_t)n);
    const size_t smem = smem_bytes(cfg.channels);
    cudaError_t e = cudaFuncSetAttribute(k_tta_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_frames, frames.data(), sizeof(sbtta::Frame) * n, cudaMemcpyHostToDevice,
                                              c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("tta_decode");
        k_tta_decode<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, smem, c.stream>>>(d_buf, d_frames, n, cfg,
                                                                                                d_pcm, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, n, who));
    if (!sbframes::first_failure(status.data(), n, "TTA frame", file_offsets, 1, sbtta::error_text, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return pcm_handle(blocks.take(d_pcm), samples, cfg.channels, rate, out);
}

}  // extern "C"
