// ALAC input: the frames a container lists (MP4 samples, Matroska blocks) decoded on the GPU into the interleaved
// int16 PCM that sb_load_pcm decodes from a WAV file, then the loader's own kernel (k_decode_resample_pad, width 2).
//   sb_alac_index_frames  upload the track's bytes; k_alac_frames, one thread per frame, reads the first element's
//                   header for the frame's sample count; sample positions are the prefix sum, as for FLAC
//   sb_alac_decode  k_alac_decode: one thread per frame walks its elements in bitstream order, Golomb residuals and LPC
//                   in place in an int32 scratch slice of its own, then unmixing and the shifted low bits, and writes
//                   the top 16 bits interleaved.  The scratch holds two channels (one element) per frame, and the
//                   frames go in launches that keep it under kScratchBytes
// Big-endian PCM (QuickTime `twos` / `in24`, ISO `ipcm`): sb_load_pcm_be, k_pcm_be writes the top 16 bits of each
// sample as little-endian int16, then k_decode_resample_pad.
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

// big-endian 16- or 24-bit samples -> the top 16 bits as int16
__global__ void __launch_bounds__(256)
k_pcm_be(const uint8_t* __restrict__ in, int64_t n, int width, int16_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint8_t* p = in + i * width;
        out[i] = (int16_t)(uint16_t)(((unsigned)p[0] << 8) | p[1]);
    }
}

}  // namespace

struct sb_alac {
    uint8_t* d_buf = nullptr;
    int64_t nbytes = 0;
    sbalac::Config cfg{};
    std::vector<sbalac::FrameDesc> frames;
    std::vector<sbalac::Listed> listed;
    std::vector<int64_t> where;        // file offset of each frame's MP4 sample or Matroska block (messages name it)
    int64_t samples = 0;
};

extern "C" {

int sb_alac_index_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                         const int32_t* config, sb_alac** out, int64_t* frames_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_alac_index_frames: library not initialised (call sb_init)");
    if (!buf || !offsets || !file_offsets || !config || !out || !frames_out)
        SB_FAIL(SB_EINVAL, "sb_alac_index_frames: NULL argument");
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
        SB_FAIL(SB_EINVAL, "sb_alac_index_frames: bad stream parameters");
    for (int64_t f = 0; f < n; ++f) {
        const int64_t end = f + 1 < n ? offsets[f + 1] : nbytes;
        if (offsets[f] < 0 || offsets[f] >= nbytes || end <= offsets[f])
            SB_FAIL(SB_EINVAL, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    offsets[f] < 0 || offsets[f] >= nbytes ? "frame starts outside the buffer" : "empty frame");
    }
    sb_alac* h = new (std::nothrow) sb_alac();
    if (!h) SB_FAIL(SB_ENOMEM, "sb_alac_index_frames: out of host memory");
    h->nbytes = nbytes; h->cfg = cfg;
    h->where.assign(file_offsets, file_offsets + n);
    auto fail = [&](int code) { sb_alac_destroy(h); return code; };
    if (pool_alloc((void**)&h->d_buf, (size_t)nbytes + 16) != SB_OK) return fail(SB_ENOMEM);
    int64_t* d_offsets = nullptr;
    sbalac::Listed* d_listed = nullptr;
    if (pool_alloc((void**)&d_offsets, sizeof(int64_t) * n + 16) != SB_OK) return fail(SB_ENOMEM);
    if (pool_alloc((void**)&d_listed, sizeof(sbalac::Listed) * n + 16) != SB_OK) { pool_free(d_offsets); return fail(SB_ENOMEM); }
    h->listed.resize((size_t)n);
    // the reader fetches 5 bytes at a time: zeros past the last frame
    cudaError_t e = cudaMemsetAsync(h->d_buf + nbytes, 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->d_buf, buf, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_offsets, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        ProfScope ps("alac_frames");
        k_alac_frames<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(h->d_buf, nbytes, d_offsets, n, cfg, d_listed);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->listed.data(), d_listed, sizeof(sbalac::Listed) * n,
                                              cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    pool_free(d_offsets); pool_free(d_listed);
    if (e != cudaSuccess) { sb_alac_destroy(h); SB_FAIL(SB_ECUDA, "sb_alac_index_frames: %s", cudaGetErrorString(e)); }
    int64_t sample = 0;
    h->frames.resize((size_t)n);
    for (int64_t f = 0; f < n; ++f) {
        const sbalac::Listed& l = h->listed[(size_t)f];
        if (l.code != sbalac::kOk) {
            sb::set_error("ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                          sbalac::error_text(l.code));
            sb_alac_destroy(h);
            return SB_EINVAL;
        }
        h->frames[(size_t)f] = sbalac::FrameDesc{offsets[f], f + 1 < n ? offsets[f + 1] : nbytes, sample};
        sample += l.samples;
    }
    h->samples = sample;
    *frames_out = sample;
    *out = h;
    return SB_OK;
}

int sb_alac_decode(sb_alac* h, int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_alac_decode: library not initialised (call sb_init)");
    if (!h || !out_f32) SB_FAIL(SB_EINVAL, "sb_alac_decode: NULL argument");
    const int64_t nf = (int64_t)h->frames.size();
    const sbalac::Config cfg = h->cfg;
    const int64_t slot = 2ll * cfg.frame_length;                        // int32 per frame in flight: one element
    const int64_t per_launch = std::max<int64_t>(1, std::min<int64_t>(nf, kScratchBytes / (slot * 4)));
    sbalac::FrameDesc* d_frames = nullptr;
    sbalac::Listed* d_listed = nullptr;
    int32_t* d_scratch = nullptr;
    int16_t* d_pcm = nullptr;
    int32_t* d_status = nullptr;
    int rc = pool_alloc((void**)&d_frames, sizeof(sbalac::FrameDesc) * nf + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_listed, sizeof(sbalac::Listed) * nf + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_scratch, sizeof(int32_t) * (size_t)(slot * per_launch) + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)h->samples * cfg.channels + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_status, sizeof(int32_t) * nf + 16);
    auto release = [&]() { pool_free(d_frames); pool_free(d_listed); pool_free(d_scratch); pool_free(d_pcm); pool_free(d_status); };
    if (rc != SB_OK) { release(); return rc; }
    std::vector<int32_t> status((size_t)nf);
    cudaError_t e = cudaMemcpyAsync(d_frames, h->frames.data(), sizeof(sbalac::FrameDesc) * nf, cudaMemcpyHostToDevice,
                                    c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_listed, h->listed.data(), sizeof(sbalac::Listed) * nf,
                                              cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && nf > 0) {
        const int64_t launches = (nf + per_launch - 1) / per_launch;
        ProfScope ps("alac_decode", (int)launches);
        for (int64_t first = 0; first < nf && e == cudaSuccess; first += per_launch) {
            const int64_t count = std::min(per_launch, nf - first);
            k_alac_decode<<<(unsigned)((count + 63) / 64), 64, 0, c.stream>>>(h->d_buf, d_frames, d_listed, first, count,
                                                                              cfg, d_scratch, d_pcm, d_status);
            e = cudaGetLastError();
        }
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost,
                                              c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { release(); SB_FAIL(SB_ECUDA, "sb_alac_decode: %s", cudaGetErrorString(e)); }
    for (int64_t f = 0; f < nf; ++f)
        if (status[(size_t)f] != sbalac::kOk) {
            release();
            SB_FAIL(SB_EINVAL, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)h->where[(size_t)f],
                    sbalac::error_text(status[(size_t)f]));
        }
    sb_stream* s = nullptr;
    rc = load_pcm_device(reinterpret_cast<const unsigned char*>(d_pcm), h->samples, cfg.channels, 2, cfg.rate,
                         sample_rate, padding, total_len, &s, "sb_alac_decode");
    e = cudaStreamSynchronize(c.stream);
    release();
    if (rc != SB_OK) return rc;
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_alac_decode: %s", cudaGetErrorString(e)); }
    *out_f32 = s;
    return SB_OK;
}

int sb_alac_destroy(sb_alac* h) {
    if (!h) return SB_OK;
    pool_free(h->d_buf);
    delete h;
    return SB_OK;
}

int sb_load_pcm_be(const void* pcm_host, int64_t frames, int channels, int sample_width, int framerate,
                   int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_load_pcm_be: library not initialised (call sb_init)");
    if (!pcm_host || !out_f32) SB_FAIL(SB_EINVAL, "sb_load_pcm_be: NULL argument");
    if (sample_width != 2 && sample_width != 3) SB_FAIL(SB_EINVAL, "Unsupported sample width: %d", sample_width);
    if (frames < 0 || channels < 1) SB_FAIL(SB_EINVAL, "sb_load_pcm_be: bad geometry");
    const int64_t n = frames * channels;
    unsigned char* d_in = nullptr;
    int16_t* d_pcm = nullptr;
    int rc = pool_alloc((void**)&d_in, (size_t)n * sample_width + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)n + 16);
    auto release = [&]() { pool_free(d_in); pool_free(d_pcm); };
    if (rc != SB_OK) { release(); return rc; }
    cudaError_t e = cudaMemcpyAsync(d_in, pcm_host, (size_t)n * sample_width, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        ProfScope ps("pcm_be");
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)c.sm_count * 16));
        k_pcm_be<<<grid, 256, 0, c.stream>>>(d_in, n, sample_width, d_pcm);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { release(); SB_FAIL(SB_ECUDA, "sb_load_pcm_be: %s", cudaGetErrorString(e)); }
    sb_stream* s = nullptr;
    rc = load_pcm_device(reinterpret_cast<const unsigned char*>(d_pcm), frames, channels, 2, framerate, sample_rate,
                         padding, total_len, &s, "sb_load_pcm_be");
    e = cudaStreamSynchronize(c.stream);                                  // pcm_host may be reused by the caller
    release();
    if (rc != SB_OK) return rc;
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_load_pcm_be: %s", cudaGetErrorString(e)); }
    *out_f32 = s;
    return SB_OK;
}

}  // extern "C"
