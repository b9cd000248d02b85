// WavPack input: the blocks a raw .wv file or a Matroska A_WAVPACK4 track holds, decoded on the GPU into the interleaved
// int16 PCM that sb_load_pcm decodes from a WAV file.
// sb_wavpack_decode_blocks:
//   k_wavpack_decode   one thread per block: its metadata sub-blocks, then every sample through the entropy decoder and
//                      all decorrelation terms at once, as FFmpeg's decoder runs them, stored as the top 16 bits at the
//                      block's sample position and channel offset.  Each thread keeps its 16 terms' weights and histories
//                      in a column of shared memory; nothing is kept per block in global scratch, so every block goes in
//                      one launch.
// The per-block arithmetic is in sb_wavpack.cuh, shared with the CPU emulation of the tests.
#include "sb_internal.h"
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
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_wavpack_decode_blocks: library not initialised (call sb_init)");
    if (!buf || !table || !out) SB_FAIL(SB_EINVAL, "sb_wavpack_decode_blocks: NULL argument");
    if (channels < 1 || channels > 8) SB_FAIL(SB_EINVAL, "WavPack with %d channels is not supported (1 to 8)", channels);
    if (rate < 1 || nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_wavpack_decode_blocks: bad stream parameters");
    std::vector<sbwv::Block> blocks((size_t)n);
    int64_t samples = 0;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t* r = table + 8 * i;
        sbwv::Block& b = blocks[(size_t)i];
        b.offset = r[0]; b.size = r[1]; b.samples = (int32_t)r[2]; b.flags = (uint32_t)r[3]; b.crc = (uint32_t)r[4];
        b.sample = r[5]; b.channel = (int32_t)r[6];
        const int width = (b.flags & sbwv::kMono) ? 1 : 2;
        if (r[0] < 0 || r[1] < 0 || r[0] > nbytes - r[1] || r[2] < 1 || r[2] > sbwv::kMaxBlockSamples || r[5] < 0 ||
            r[6] < 0 || r[6] + width > channels)
            SB_FAIL(SB_EINVAL, "WavPack block %lld at byte offset %lld: block table entry out of range", (long long)i,
                    (long long)r[7]);
        samples = std::max(samples, r[5] + r[2]);
    }
    uint8_t* d_buf = nullptr;
    sbwv::Block* d_blocks = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    auto release = [&]() { pool_free(d_buf); pool_free(d_blocks); pool_free(d_status); };
    auto fail = [&](int code) { release(); pool_free(d_pcm); return code; };
    int rc = pool_alloc((void**)&d_buf, (size_t)nbytes + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_blocks, sizeof(sbwv::Block) * n + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)samples * channels + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_status, sizeof(int32_t) * n + 16);
    if (rc != SB_OK) return fail(rc);
    std::vector<int32_t> status((size_t)n);
    // the bit reader fetches 5 bytes at a time: zeros past the last block
    cudaError_t e = cudaMemsetAsync(d_buf + nbytes, 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_buf, buf, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_blocks, blocks.data(), sizeof(sbwv::Block) * n, cudaMemcpyHostToDevice,
                                              c.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_pcm, 0, sizeof(int16_t) * (size_t)samples * channels, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("wavpack_decode");
        k_wavpack_decode<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, kSmemBytes, c.stream>>>(
            d_buf, d_blocks, n, channels, d_pcm, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { fail(0); SB_FAIL(SB_ECUDA, "sb_wavpack_decode_blocks: %s", cudaGetErrorString(e)); }
    for (int64_t i = 0; i < n; ++i)
        if (status[(size_t)i] != sbwv::kOk) {
            fail(0);
            SB_FAIL(SB_EINVAL, "WavPack block %lld at byte offset %lld: %s", (long long)i, (long long)table[8 * i + 7],
                    sbwv::error_text(status[(size_t)i]));
        }
    release();
    return pcm_handle(d_pcm, samples, channels, rate, out);
}

}  // extern "C"
