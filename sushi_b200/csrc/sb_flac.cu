// FLAC input: the file's frames decoded on the GPU into the interleaved int16 PCM that sb_load_pcm decodes from a WAV
// file, then the loader's own kernel (k_decode_resample_pad, width 2) from there on.
//   sb_flac_index   upload the file; k_flac_sync lists every byte position holding a sync code and a frame header
//                   that parses, agrees with STREAMINFO and passes its CRC-8 (false syncs included); the host chains
//                   the real frames from the first one by their coded frame / sample numbers
//   sb_flac_index_frames  the same for frames a container lists (Matroska blocks and laces): k_flac_frames, one thread
//                   per listed frame, checks the header at its offset; sample positions are the prefix sum of the
//                   block sizes, and errors name the file offset of the frame's block
//   sb_flac_decode  k_flac_decode: one thread per frame decodes its subframes in turn (a subframe starts where the
//                   previous one ends) and checks the frame's CRC-16 and end; k_flac_decorrelate: one CTA per frame
//                   undoes the stereo decorrelation and writes int16 (24-bit: the top 16 bits); then the loader
// The per-frame arithmetic is in sb_flac.cuh, shared with the CPU emulation of the tests.
#include "sb_internal.h"
#include "sb_flac.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

using sbflac::Candidate;
using sbflac::FrameDesc;

__global__ void __launch_bounds__(256)
k_flac_sync(const uint8_t* __restrict__ file, int64_t first, int64_t nbytes, int channels, int bits, int rate,
            Candidate* __restrict__ out, unsigned long long* __restrict__ count, int64_t cap) {
    const int64_t words = (nbytes + 3) >> 2;                       // the buffer is zero-padded past nbytes
    for (int64_t w = (first >> 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < words;
         w += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(file) + w);
        if (!(((v & 0xFF) == 0xFF) | (((v >> 8) & 0xFF) == 0xFF) | (((v >> 16) & 0xFF) == 0xFF) | ((v >> 24) == 0xFF)))
            continue;
        for (int k = 0; k < 4; ++k) {
            const int64_t i = 4 * w + k;
            if (i < first || i + 1 >= nbytes || ((v >> (8 * k)) & 0xFF) != 0xFF || (file[i + 1] & 0xFE) != 0xF8) continue;
            sbflac::Header h;
            if (sbflac::parse_header(file + i, nbytes - i, channels, bits, rate, &h) != sbflac::kOk) continue;
            const unsigned long long slot = atomicAdd(count, 1ull);
            if ((int64_t)slot < cap) {
                Candidate c; c.offset = i; c.number = h.number; c.block_size = h.block_size;
                c.assignment = (int16_t)h.assignment; c.variable = (int16_t)h.variable;
                out[slot] = c;
            }
        }
    }
}

// Frames listed by a container: one thread per frame parses the header at its listed offset, bounded by the next one
__global__ void __launch_bounds__(256)
k_flac_frames(const uint8_t* __restrict__ buf, int64_t nbytes, const int64_t* __restrict__ offsets, int64_t n,
              int channels, int bits, int rate, sbflac::ListedFrame* __restrict__ out) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) out[f] = sbflac::listed_frame(buf, nbytes, offsets, n, f, channels, bits, rate);
}

__global__ void __launch_bounds__(64)
k_flac_decode(const uint8_t* __restrict__ file, const FrameDesc* __restrict__ frames, int64_t n_frames, int channels,
              int bits, int rate, int32_t* __restrict__ planar, sbflac::FrameStatus* __restrict__ status) {
    __shared__ uint16_t s_crc[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = sbflac::crc16_entry(i);
    __syncthreads();
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const FrameDesc d = frames[f];
    sbflac::FrameStatus st;
    st.pad = 0;
    st.code = sbflac::decode_frame(file, d.offset, d.limit, channels, bits, rate, s_crc, planar + d.sample * channels,
                                   &st.end);
    status[f] = st;
}

__global__ void __launch_bounds__(256)
k_flac_decorrelate(const FrameDesc* __restrict__ frames, int64_t n_frames, int channels, int bits,
                   const int32_t* __restrict__ planar, int16_t* __restrict__ pcm) {
    for (int64_t f = blockIdx.x; f < n_frames; f += gridDim.x) {
        const FrameDesc d = frames[f];
        const int32_t* in = planar + d.sample * channels;
        for (int j = threadIdx.x; j < d.block_size; j += blockDim.x)
            sbflac::decorrelate(in, d.block_size, j, channels, d.assignment, bits, pcm + (d.sample + j) * channels);
    }
}

}  // namespace

struct sb_flac {
    uint8_t* d_file = nullptr;
    int64_t nbytes = 0;
    int channels = 0, bits = 0, framerate = 0;
    std::vector<FrameDesc> frames;
    std::vector<int64_t> where;        // sb_flac_index_frames: file offset of each frame's block (messages name it)
    int64_t samples = 0;
};

extern "C" {

int sb_flac_index(const void* file, int64_t nbytes, int64_t first_frame_offset, int channels, int bits,
                  int framerate, sb_flac** out, int64_t* frames_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_flac_index: library not initialised (call sb_init)");
    if (!file || !out || !frames_out) SB_FAIL(SB_EINVAL, "sb_flac_index: NULL argument");
    if (bits != 16 && bits != 24) SB_FAIL(SB_EINVAL, "FLAC with %d bits per sample is not supported (16 or 24)", bits);
    if (channels < 1 || channels > 8 || framerate < 1 || nbytes < 1 || first_frame_offset < 0 || first_frame_offset > nbytes)
        SB_FAIL(SB_EINVAL, "sb_flac_index: bad stream parameters");
    sb_flac* h = new (std::nothrow) sb_flac();
    if (!h) SB_FAIL(SB_ENOMEM, "sb_flac_index: out of host memory");
    h->nbytes = nbytes; h->channels = channels; h->bits = bits; h->framerate = framerate;
    const uint8_t* host = static_cast<const uint8_t*>(file);
    auto fail = [&](int code) { sb_flac_destroy(h); return code; };
    if (pool_alloc((void**)&h->d_file, (size_t)nbytes + 16) != SB_OK) return fail(SB_ENOMEM);
    cudaError_t e = cudaMemsetAsync(h->d_file + (nbytes & ~(int64_t)3), 0, 16, c.stream);      // zero tail for k_flac_sync
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->d_file, file, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e != cudaSuccess) { sb_flac_destroy(h); SB_FAIL(SB_ECUDA, "sb_flac_index: %s", cudaGetErrorString(e)); }

    // candidates: a frame has at least 9 bytes; real files hold one frame per few kB and false syncs are rarer still
    int64_t cap = nbytes / 256 + 4096;
    std::vector<Candidate> cand;
    for (int pass = 0; pass < 2; ++pass) {
        Candidate* d_cand = nullptr;
        unsigned long long* d_count = nullptr;
        if (pool_alloc((void**)&d_cand, sizeof(Candidate) * cap) != SB_OK) return fail(SB_ENOMEM);
        if (pool_alloc((void**)&d_count, sizeof(unsigned long long)) != SB_OK) { pool_free(d_cand); return fail(SB_ENOMEM); }
        unsigned long long count = 0;
        e = cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), c.stream);
        if (e == cudaSuccess) {
            ProfScope ps("flac_sync");
            const int64_t words = (nbytes + 3) / 4;
            const int grid = (int)std::min<int64_t>((words + 255) / 256, (int64_t)c.sm_count * 16);
            k_flac_sync<<<std::max(grid, 1), 256, 0, c.stream>>>(h->d_file, first_frame_offset, nbytes, channels, bits,
                                                                 framerate, d_cand, d_count, cap);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, c.stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        if (e == cudaSuccess && (int64_t)count <= cap) {
            cand.resize(count);
            e = cudaMemcpyAsync(cand.data(), d_cand, sizeof(Candidate) * count, cudaMemcpyDeviceToHost, c.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        }
        pool_free(d_cand); pool_free(d_count);
        if (e != cudaSuccess) { sb_flac_destroy(h); SB_FAIL(SB_ECUDA, "sb_flac_index: %s", cudaGetErrorString(e)); }
        if ((int64_t)count <= cap) break;
        cap = (int64_t)count;                                              // rescan with room for every candidate
    }
    char msg[256];
    int64_t sample = 0;
    if (!sbflac::chain(cand, first_frame_offset, nbytes, channels, bits, framerate, host + first_frame_offset, h->frames,
                       &sample, msg, sizeof(msg))) {
        sb::set_error("%s", msg);
        sb_flac_destroy(h);
        return SB_EINVAL;
    }
    h->samples = sample;
    *frames_out = sample;
    *out = h;
    return SB_OK;
}

int sb_flac_index_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                         int channels, int bits, int framerate, sb_flac** out, int64_t* frames_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_flac_index_frames: library not initialised (call sb_init)");
    if (!buf || !offsets || !file_offsets || !out || !frames_out) SB_FAIL(SB_EINVAL, "sb_flac_index_frames: NULL argument");
    if (bits != 16 && bits != 24) SB_FAIL(SB_EINVAL, "FLAC with %d bits per sample is not supported (16 or 24)", bits);
    if (channels < 1 || channels > 8 || framerate < 1 || nbytes < 1 || n < 0)
        SB_FAIL(SB_EINVAL, "sb_flac_index_frames: bad stream parameters");
    for (int64_t f = 0; f < n; ++f)
        if (offsets[f] < 0 || offsets[f] >= nbytes || (f > 0 && offsets[f] <= offsets[f - 1]))
            SB_FAIL(SB_EINVAL, "FLAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    offsets[f] < 0 || offsets[f] >= nbytes ? "frame starts outside the buffer" : "empty frame");
    sb_flac* h = new (std::nothrow) sb_flac();
    if (!h) SB_FAIL(SB_ENOMEM, "sb_flac_index_frames: out of host memory");
    h->nbytes = nbytes; h->channels = channels; h->bits = bits; h->framerate = framerate;
    h->where.assign(file_offsets, file_offsets + n);
    auto fail = [&](int code) { sb_flac_destroy(h); return code; };
    if (pool_alloc((void**)&h->d_file, (size_t)nbytes + 16) != SB_OK) return fail(SB_ENOMEM);
    int64_t* d_offsets = nullptr;
    sbflac::ListedFrame* d_listed = nullptr;
    if (pool_alloc((void**)&d_offsets, sizeof(int64_t) * n + 16) != SB_OK) return fail(SB_ENOMEM);
    if (pool_alloc((void**)&d_listed, sizeof(sbflac::ListedFrame) * n + 16) != SB_OK) { pool_free(d_offsets); return fail(SB_ENOMEM); }
    std::vector<sbflac::ListedFrame> listed((size_t)n);
    cudaError_t e = cudaMemsetAsync(h->d_file + (nbytes & ~(int64_t)3), 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->d_file, buf, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_offsets, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        ProfScope ps("flac_frames");
        k_flac_frames<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(h->d_file, nbytes, d_offsets, n, channels, bits,
                                                                         framerate, d_listed);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(listed.data(), d_listed, sizeof(sbflac::ListedFrame) * n,
                                              cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    pool_free(d_offsets); pool_free(d_listed);
    if (e != cudaSuccess) { sb_flac_destroy(h); SB_FAIL(SB_ECUDA, "sb_flac_index_frames: %s", cudaGetErrorString(e)); }
    char msg[256];
    int64_t sample = 0;
    if (!sbflac::list_frames(listed.data(), offsets, file_offsets, n, nbytes, h->frames, &sample, msg, sizeof(msg))) {
        sb::set_error("%s", msg);
        sb_flac_destroy(h);
        return SB_EINVAL;
    }
    h->samples = sample;
    *frames_out = sample;
    *out = h;
    return SB_OK;
}

int sb_flac_decode(sb_flac* h, int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_flac_decode: library not initialised (call sb_init)");
    if (!h || !out_f32) SB_FAIL(SB_EINVAL, "sb_flac_decode: NULL argument");
    const int64_t nf = (int64_t)h->frames.size();
    const int ch = h->channels;
    FrameDesc* d_frames = nullptr;
    int32_t* d_planar = nullptr;
    int16_t* d_pcm = nullptr;
    sbflac::FrameStatus* d_status = nullptr;
    int rc = pool_alloc((void**)&d_frames, sizeof(FrameDesc) * nf + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_planar, sizeof(int32_t) * (size_t)h->samples * ch + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)h->samples * ch + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_status, sizeof(sbflac::FrameStatus) * nf + 16);
    auto release = [&]() { pool_free(d_frames); pool_free(d_planar); pool_free(d_pcm); pool_free(d_status); };
    if (rc != SB_OK) { release(); return rc; }
    std::vector<sbflac::FrameStatus> status((size_t)nf);
    cudaError_t e = cudaMemcpyAsync(d_frames, h->frames.data(), sizeof(FrameDesc) * nf, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && nf > 0) {
        ProfScope ps("flac_decode");
        k_flac_decode<<<(unsigned)((nf + 63) / 64), 64, 0, c.stream>>>(h->d_file, d_frames, nf, ch, h->bits, h->framerate,
                                                                       d_planar, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, sizeof(sbflac::FrameStatus) * nf,
                                              cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { release(); SB_FAIL(SB_ECUDA, "sb_flac_decode: %s", cudaGetErrorString(e)); }
    // every frame must decode, pass its CRC-16 and end exactly where the next frame (or the file) does
    char msg[256];
    auto bytes_at = [&](int64_t off, uint8_t* buf) {
        if (off < h->nbytes) cudaMemcpy(buf, h->d_file + off, (size_t)std::min<int64_t>(16, h->nbytes - off), cudaMemcpyDeviceToHost);
    };
    if (!sbflac::check_frames(h->frames, status.data(), h->nbytes, ch, h->bits, h->framerate, bytes_at, msg, sizeof(msg),
                              h->where.empty() ? nullptr : h->where.data())) {
        release();
        SB_FAIL(SB_EINVAL, "%s", msg);
    }
    if (nf > 0) {
        ProfScope ps("flac_decorrelate");
        k_flac_decorrelate<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(nf, (int64_t)c.sm_count * 64)), 256, 0,
                             c.stream>>>(d_frames, nf, ch, h->bits, d_planar, d_pcm);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { release(); SB_FAIL(SB_ECUDA, "sb_flac_decode: %s", cudaGetErrorString(e)); }
    sb_stream* s = nullptr;
    rc = load_pcm_device(reinterpret_cast<const unsigned char*>(d_pcm), h->samples, ch, 2, h->framerate, sample_rate,
                         padding, total_len, &s, "sb_flac_decode");
    e = cudaStreamSynchronize(c.stream);
    release();
    if (rc != SB_OK) return rc;
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_flac_decode: %s", cudaGetErrorString(e)); }
    *out_f32 = s;
    return SB_OK;
}

int sb_flac_destroy(sb_flac* h) {
    if (!h) return SB_OK;
    pool_free(h->d_file);
    delete h;
    return SB_OK;
}

}  // extern "C"
