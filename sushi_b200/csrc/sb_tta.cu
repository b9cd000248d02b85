// TTA input: the frames of a raw .tta file or a Matroska A_TTA1 track, decoded on the GPU into the interleaved int16
// PCM that sb_load_pcm decodes from a WAV file.
// sb_tta_decode_frames:
//   k_tta_decode   one thread per frame: every sample through the Rice code, the filter and the predictor, channel by
//                  channel, then the decorrelation and the top-16-bit store at the frame's sample position; then the
//                  frame's CRC-32.  Each thread keeps its channels' state in a column of shared memory, and its CTA
//                  shares one slice-by-4 CRC table there; nothing is kept per frame in global scratch, so every frame
//                  goes in one launch.
// The per-frame arithmetic is in sb_tta.cuh, shared with the CPU emulation of the tests.
#include "sb_internal.h"
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
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_tta_decode_frames: library not initialised (call sb_init)");
    if (!buf || !offsets || !file_offsets || !config || !out) SB_FAIL(SB_EINVAL, "sb_tta_decode_frames: NULL argument");
    sbtta::Config cfg;
    cfg.channels = config[0]; cfg.bits = config[1];
    const int32_t rate = config[2];
    cfg.frame_length = config[3]; cfg.last_length = config[4];
    if (cfg.channels < 1 || cfg.channels > sbtta::kMaxChannels)
        SB_FAIL(SB_EINVAL, "TTA with %d channels is not supported (1 to 8)", cfg.channels);
    if (cfg.bits != 16 && cfg.bits != 24) SB_FAIL(SB_EINVAL, "TTA with %d bits per sample is not supported (16 or 24)", cfg.bits);
    if (rate < 1 || rate > 0x7FFFFF || cfg.frame_length != (int32_t)(256ll * rate / 245) || cfg.frame_length < 1 ||
        cfg.last_length < 0 || cfg.last_length >= cfg.frame_length || nbytes < 1 || n < 1)
        SB_FAIL(SB_EINVAL, "sb_tta_decode_frames: bad stream parameters");
    std::vector<sbtta::Frame> frames((size_t)n);
    for (int64_t f = 0; f < n; ++f) {
        const int64_t end = f + 1 < n ? offsets[f + 1] : nbytes;
        if (offsets[f] < 0 || offsets[f] >= nbytes || end <= offsets[f] || end > nbytes)
            SB_FAIL(SB_EINVAL, "TTA frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    offsets[f] < 0 || offsets[f] >= nbytes ? "frame starts outside the buffer" : "empty frame");
        sbtta::Frame& d = frames[(size_t)f];
        d.offset = offsets[f]; d.size = end - offsets[f]; d.sample = f * (int64_t)cfg.frame_length;
        d.last = f + 1 == n; d.pad = 0;
    }
    const int64_t samples = (n - 1) * (int64_t)cfg.frame_length + (cfg.last_length ? cfg.last_length : cfg.frame_length);
    uint8_t* d_buf = nullptr;
    sbtta::Frame* d_frames = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    auto release = [&]() { pool_free(d_buf); pool_free(d_frames); pool_free(d_status); };
    auto fail = [&](int code) { release(); pool_free(d_pcm); return code; };
    int rc = pool_alloc((void**)&d_buf, (size_t)nbytes + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_frames, sizeof(sbtta::Frame) * n + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)samples * cfg.channels + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_status, sizeof(int32_t) * n + 16);
    if (rc != SB_OK) return fail(rc);
    std::vector<int32_t> status((size_t)n);
    const size_t smem = smem_bytes(cfg.channels);
    cudaError_t e = cudaFuncSetAttribute(k_tta_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_buf, buf, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_frames, frames.data(), sizeof(sbtta::Frame) * n, cudaMemcpyHostToDevice,
                                              c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("tta_decode");
        k_tta_decode<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, smem, c.stream>>>(d_buf, d_frames, n, cfg,
                                                                                                d_pcm, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { fail(0); SB_FAIL(SB_ECUDA, "sb_tta_decode_frames: %s", cudaGetErrorString(e)); }
    for (int64_t f = 0; f < n; ++f)
        if (status[(size_t)f] != sbtta::kOk) {
            fail(0);
            SB_FAIL(SB_EINVAL, "TTA frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    sbtta::error_text(status[(size_t)f]));
        }
    release();
    return pcm_handle(d_pcm, samples, cfg.channels, rate, out);
}

}  // extern "C"
