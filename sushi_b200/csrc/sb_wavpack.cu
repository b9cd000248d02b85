// WavPack input: the blocks a raw .wv file or a Matroska A_WAVPACK4 track holds, decoded on the GPU into the interleaved
// int16 PCM that sb_load_pcm decodes from a WAV file.
// sb_wavpack_decode_blocks:
//   k_wavpack_decode   one thread per block: its metadata sub-blocks, then every sample through the entropy decoder and
//                      all decorrelation terms at once, as FFmpeg's decoder runs them, stored as the top 16 bits at the
//                      block's sample position and channel offset.  Each thread keeps its 16 terms' weights and histories
//                      in a column of shared memory; nothing is kept per block in global scratch, so every block goes in
//                      one launch.
// The per-block arithmetic is in sb_wavpack.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
#include "sb_wavpack.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int kThreads = 32;
constexpr int kSmemBytes = kThreads * sbwv::kMaxTerms * sbwv::kTermWords * 4;      // 38912

__global__ void __launch_bounds__(kThreads)
k_wavpack_decode(const uint8_t* __restrict__ buf, const sbwv::Block* __restrict__ blocks, int64_t n, int channels,
                 int16_t* __restrict__ pcm, int32_t* __restrict__ status) {
    extern __shared__ int32_t terms[];
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    sbwv::Terms ts;
    ts.p = terms + threadIdx.x;
    ts.stride = blockDim.x;
    status[k] = sbwv::decode_block(buf, blocks[k], channels, ts, pcm);
}

}  // namespace

extern "C" {

int sb_wavpack_decode_blocks(const void* buf, int64_t nbytes, const int64_t* table, int64_t n, int32_t channels,
                             int32_t rate, sb_pcm** out) {
    const char* who = "sb_wavpack_decode_blocks";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, buf && table && out));
    if (channels < 1 || channels > 8) SB_FAIL(SB_EINVAL, "WavPack with %d channels is not supported (1 to 8)", channels);
    if (rate < 1 || nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_wavpack_decode_blocks: bad stream parameters");
    std::vector<sbwv::Block> blocks_h;
    int64_t samples = 0;
    char msg[256];
    if (!sbwv::block_table(table, n, nbytes, channels, blocks_h, &samples, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    sbwv::Block* d_blocks = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, buf, nbytes, who));
    SB_TRY(blocks.alloc(&d_blocks, (size_t)n));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)samples * channels));
    SB_TRY(blocks.alloc(&d_status, (size_t)n));
    std::vector<int32_t> status((size_t)n);
    cudaError_t e = cudaMemcpyAsync(d_blocks, blocks_h.data(), sizeof(sbwv::Block) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_pcm, 0, sizeof(int16_t) * (size_t)samples * channels, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("wavpack_decode");
        k_wavpack_decode<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, kSmemBytes, c.stream>>>(
            d_buf, d_blocks, n, channels, d_pcm, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, n, who));
    if (!sbframes::first_failure(status.data(), n, "WavPack block", table + 7, 8, sbwv::error_text, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return pcm_handle(blocks.take(d_pcm), samples, channels, rate, out);
}

}  // extern "C"
