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
#include "sb_decode.h"
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
    const char* who = "sb_alac_decode_frames";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, buf && offsets && file_offsets && config && out));
    sbalac::Config cfg;
    char msg[256];
    if (!sbalac::parse_config(config, &cfg, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    if (nbytes < 1 || n < 0) SB_FAIL(SB_EINVAL, "sb_alac_decode_frames: bad stream parameters");
    if (!sbalac::check_offsets(offsets, file_offsets, n, nbytes, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    const int64_t slot = 2ll * cfg.frame_length;                        // int32 per frame in flight: one element
    const int64_t per_launch = std::max<int64_t>(1, std::min<int64_t>(n, kScratchBytes / (slot * 4)));
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    int64_t* d_offsets = nullptr;
    sbalac::Listed* d_listed = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, buf, nbytes, who));
    SB_TRY(blocks.alloc(&d_offsets, (size_t)n));
    SB_TRY(blocks.alloc(&d_listed, (size_t)n));

    // every frame's sample count from its first element
    std::vector<sbalac::Listed> listed((size_t)n);
    cudaError_t e = cudaMemcpyAsync(d_offsets, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        ProfScope ps("alac_frames");
        k_alac_frames<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d_buf, nbytes, d_offsets, n, cfg, d_listed);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, listed.data(), d_listed, n, who));
    int64_t samples = 0;
    std::vector<sbalac::FrameDesc> frames;
    if (!sbalac::frame_table(listed.data(), offsets, file_offsets, n, nbytes, frames, &samples, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);

    // every frame decoded, in launches that keep the scratch under kScratchBytes
    sbalac::FrameDesc* d_frames = nullptr;
    int32_t* d_scratch = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    SB_TRY(blocks.alloc(&d_frames, (size_t)n));
    SB_TRY(blocks.alloc(&d_scratch, (size_t)(slot * per_launch)));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)samples * cfg.channels));
    SB_TRY(blocks.alloc(&d_status, (size_t)n));
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
    SB_TRY(collect(e, status.data(), d_status, n, who));
    if (!sbframes::first_failure(status.data(), n, "ALAC frame", file_offsets, 1, sbalac::error_text, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return pcm_handle(blocks.take(d_pcm), samples, cfg.channels, cfg.rate, out);
}

}  // extern "C"
