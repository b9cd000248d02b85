// ALAC input: the frames a container lists (MP4 samples, Matroska blocks) decoded on the GPU into the interleaved
// int16 PCM that sb_load_pcm decodes from a WAV file, then the loader's own kernel (k_decode_resample_pad, width 2).
// sb_alac_decode_frames:
//   k_alac_frames   upload the track's bytes; one thread per frame reads the first element's header for the frame's
//                   sample count; sample positions are the prefix sum, as for FLAC
//   k_alac_decode   one thread per frame walks its elements in bitstream order, Golomb residuals and LPC in place in an
//                   int32 scratch slice of its own, then unmixing and the shifted low bits, and writes the top 16 bits
//                   interleaved into an sb_pcm.  The scratch holds two channels (one element) per frame, and the
//                   frames go in launches that keep it under kScratchBytes
// The per-frame arithmetic is in sb_alac.cuh, shared with the CPU emulation of the tests.
#include "sb_internal.h"
#include "sb_alac.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

constexpr int64_t kScratchBytes = 256ll << 20;

__global__ void __launch_bounds__(256)
k_alac_frames(const uint8_t* __restrict__ buf, int64_t nbytes, const int64_t* __restrict__ offsets, int64_t n,
              sbalac::Config c, sbalac::Listed* __restrict__ out) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) out[f] = sbalac::first_element(buf, offsets[f], f + 1 < n ? offsets[f + 1] : nbytes, c);
}

__global__ void __launch_bounds__(64)
k_alac_decode(const uint8_t* __restrict__ buf, const sbalac::FrameDesc* __restrict__ frames,
              const sbalac::Listed* __restrict__ listed, int64_t first, int64_t count, sbalac::Config c,
              int32_t* __restrict__ scratch, int16_t* __restrict__ pcm, int32_t* __restrict__ status) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const int64_t f = first + k;
    const sbalac::FrameDesc d = frames[f];
    status[f] = sbalac::decode_frame(buf, d.offset, d.limit, c, listed[f].samples, scratch + k * 2 * c.frame_length,
                                     pcm + d.sample * c.channels);
}

}  // namespace

extern "C" {

int sb_alac_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                          const int32_t* config, sb_pcm** out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_alac_decode_frames: library not initialised (call sb_init)");
    if (!buf || !offsets || !file_offsets || !config || !out) SB_FAIL(SB_EINVAL, "sb_alac_decode_frames: NULL argument");
    sbalac::Config cfg;
    cfg.frame_length = config[0]; cfg.bit_depth = config[1]; cfg.pb = config[2]; cfg.mb = config[3];
    cfg.kb = config[4]; cfg.channels = config[5]; cfg.rate = config[6];
    if (cfg.bit_depth != 16 && cfg.bit_depth != 20 && cfg.bit_depth != 24 && cfg.bit_depth != 32)
        SB_FAIL(SB_EINVAL, "ALAC with %d bits per sample is not supported (16, 20, 24 or 32)", cfg.bit_depth);
    if (cfg.frame_length < 1 || cfg.frame_length > sbalac::kMaxFrameLength)
        SB_FAIL(SB_EINVAL, "ALAC frameLength %d is not supported (1 to %d)", cfg.frame_length, sbalac::kMaxFrameLength);
    if (cfg.channels < 1 || cfg.channels > 8) SB_FAIL(SB_EINVAL, "ALAC with %d channels is not supported (1 to 8)", cfg.channels);
    if (cfg.rate < 1 || cfg.pb < 0 || cfg.pb > 255 || cfg.mb < 0 || cfg.mb > 255 || cfg.kb < 0 || cfg.kb > 255 ||
        nbytes < 1 || n < 0)
        SB_FAIL(SB_EINVAL, "sb_alac_decode_frames: bad stream parameters");
    for (int64_t f = 0; f < n; ++f) {
        const int64_t end = f + 1 < n ? offsets[f + 1] : nbytes;
        if (offsets[f] < 0 || offsets[f] >= nbytes || end <= offsets[f])
            SB_FAIL(SB_EINVAL, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    offsets[f] < 0 || offsets[f] >= nbytes ? "frame starts outside the buffer" : "empty frame");
    }
    const int64_t slot = 2ll * cfg.frame_length;                        // int32 per frame in flight: one element
    const int64_t per_launch = std::max<int64_t>(1, std::min<int64_t>(n, kScratchBytes / (slot * 4)));
    uint8_t* d_buf = nullptr;
    int64_t* d_offsets = nullptr;
    sbalac::Listed* d_listed = nullptr;
    sbalac::FrameDesc* d_frames = nullptr;
    int32_t* d_scratch = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    auto release = [&]() {
        pool_free(d_buf); pool_free(d_offsets); pool_free(d_listed); pool_free(d_frames); pool_free(d_scratch);
        pool_free(d_status);
    };
    auto fail = [&](int code) { release(); pool_free(d_pcm); return code; };
    int rc = pool_alloc((void**)&d_buf, (size_t)nbytes + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_offsets, sizeof(int64_t) * n + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_listed, sizeof(sbalac::Listed) * n + 16);
    if (rc != SB_OK) return fail(rc);

    // every frame's sample count from its first element
    std::vector<sbalac::Listed> listed((size_t)n);
    // the reader fetches 5 bytes at a time: zeros past the last frame
    cudaError_t e = cudaMemsetAsync(d_buf + nbytes, 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_buf, buf, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_offsets, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        ProfScope ps("alac_frames");
        k_alac_frames<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d_buf, nbytes, d_offsets, n, cfg, d_listed);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(listed.data(), d_listed, sizeof(sbalac::Listed) * n, cudaMemcpyDeviceToHost,
                                              c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { fail(0); SB_FAIL(SB_ECUDA, "sb_alac_decode_frames: %s", cudaGetErrorString(e)); }
    int64_t samples = 0;
    std::vector<sbalac::FrameDesc> frames((size_t)n);
    for (int64_t f = 0; f < n; ++f) {
        const sbalac::Listed& l = listed[(size_t)f];
        if (l.code != sbalac::kOk) {
            fail(0);
            SB_FAIL(SB_EINVAL, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    sbalac::error_text(l.code));
        }
        frames[(size_t)f] = sbalac::FrameDesc{offsets[f], f + 1 < n ? offsets[f + 1] : nbytes, samples};
        samples += l.samples;
    }

    // every frame decoded, in launches that keep the scratch under kScratchBytes
    rc = pool_alloc((void**)&d_frames, sizeof(sbalac::FrameDesc) * n + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_scratch, sizeof(int32_t) * (size_t)(slot * per_launch) + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)samples * cfg.channels + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_status, sizeof(int32_t) * n + 16);
    if (rc != SB_OK) return fail(rc);
    std::vector<int32_t> status((size_t)n);
    e = cudaMemcpyAsync(d_frames, frames.data(), sizeof(sbalac::FrameDesc) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        const int64_t launches = (n + per_launch - 1) / per_launch;
        ProfScope ps("alac_decode", (int)launches);
        for (int64_t first = 0; first < n && e == cudaSuccess; first += per_launch) {
            const int64_t count = std::min(per_launch, n - first);
            k_alac_decode<<<(unsigned)((count + 63) / 64), 64, 0, c.stream>>>(d_buf, d_frames, d_listed, first, count,
                                                                              cfg, d_scratch, d_pcm, d_status);
            e = cudaGetLastError();
        }
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { fail(0); SB_FAIL(SB_ECUDA, "sb_alac_decode_frames: %s", cudaGetErrorString(e)); }
    for (int64_t f = 0; f < n; ++f)
        if (status[(size_t)f] != sbalac::kOk) {
            fail(0);
            SB_FAIL(SB_EINVAL, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    sbalac::error_text(status[(size_t)f]));
        }
    release();
    return pcm_handle(d_pcm, samples, cfg.channels, cfg.rate, out);
}

}  // extern "C"
