// Dolby TrueHD input: the stream's restart segments decoded on the GPU into the interleaved int16 PCM that sb_load_pcm
// decodes from a WAV file, then the loader's own kernel (k_decode_resample_pad, width 2) from there on.
//   sb_truehd_index   upload the stream; k_truehd_sync lists every byte position holding a major sync whose CRC passes
//                     (false syncs inside coded data included) and whether its decoded substreams open with restart
//                     headers; the host walks the AU lengths from the start, block by block, into restart segments
//                     (only a listed sync at an AU start begins one); k_truehd_decode gives one thread to each segment,
//                     which decodes its AUs in turn into int16 at AU index x samples per AU and returns its lossless
//                     check; the host joins the checks of neighbouring segments
//   sb_truehd_decode  the loader on the decoded PCM
// The per-AU arithmetic is in sb_truehd.cuh, shared with the CPU emulation of the tests.
#include "sb_internal.h"
#include "sb_truehd.cuh"
#include <algorithm>
#include <functional>
#include <new>
#include <vector>

using namespace sb;

namespace {

__global__ void __launch_bounds__(256)
k_truehd_sync(const uint8_t* __restrict__ buf, int64_t nbytes, sbthd::Format f, sbthd::Candidate* __restrict__ out,
              unsigned long long* __restrict__ count, int64_t cap) {
    const int64_t words = (nbytes + 3) >> 2;                       // the buffer is zero-padded past nbytes
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < words; w += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(buf) + w);
        if (!(((v & 0xFF) == 0xF8) | (((v >> 8) & 0xFF) == 0xF8) | (((v >> 16) & 0xFF) == 0xF8) | ((v >> 24) == 0xF8)))
            continue;
        for (int k = 0; k < 4; ++k) {
            const int64_t i = 4 * w + k - 4;                        // the AU starts 4 bytes before its major sync
            if (i < 0 || i + 36 > nbytes || ((v >> (8 * k)) & 0xFF) != 0xF8) continue;
            if (buf[i + 5] != 0x72 || buf[i + 6] != 0x6F || (buf[i + 7] & 0xFE) != 0xBA) continue;
            const sbthd::Candidate c = sbthd::candidate(buf, nbytes, i, f);
            if (c.code == sbthd::kBadSyncCrc) continue;
            const unsigned long long slot = atomicAdd(count, 1ull);
            if ((int64_t)slot < cap) out[slot] = c;
        }
    }
}

__global__ void __launch_bounds__(64)
k_truehd_decode(const uint8_t* __restrict__ buf, int64_t nbytes, const int64_t* __restrict__ blocks, int64_t n_blocks,
                sbthd::Format f, const sbthd::Segment* __restrict__ segs, int64_t n_segs, int16_t* __restrict__ pcm,
                sbthd::SegStatus* __restrict__ status) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_segs) return;
    sbthd::State st;                                                // per-thread decoder state, in local memory
    const sbthd::Segment g = segs[k];
    status[k] = sbthd::decode_segment(buf, nbytes, blocks, n_blocks, f, g, k == 0, st,
                                      pcm + g.first_au * f.spa * (int64_t)f.channels);
}

}  // namespace

struct sb_truehd {
    int16_t* d_pcm = nullptr;
    int64_t samples = 0;
    int channels = 0, rate = 0;
};

namespace sb {

// The body of sb_truehd_index on a stream already on the device: `host` and `d_buf` hold the same `nbytes` bytes (d_buf
// zero-padded to 16 bytes past nbytes & ~3 for k_truehd_sync); blocks start at offsets[0..n) (d_blocks: the same on
// the device); where(off) is the file offset messages give for stream byte `off`.  The caller keeps d_buf and d_blocks.
int truehd_index_device(const uint8_t* host, const uint8_t* d_buf, int64_t nbytes, const int64_t* offsets,
                        const int64_t* d_blocks, int64_t n, const std::function<int64_t(int64_t)>& where, int32_t* info,
                        sb_truehd** out, int64_t* frames_out) {
    Ctx& c = ctx();
    sbthd::Format f;
    char msg[256], fmsg[200];
    if (!sbthd::parse_format(host, nbytes, offsets[0], &f, fmsg, sizeof(fmsg))) {
        snprintf(msg, sizeof(msg), fmsg, (long long)where(offsets[0]));
        SB_FAIL(SB_EINVAL, "%s", msg);
    }
    sb_truehd* h = new (std::nothrow) sb_truehd();
    if (!h) SB_FAIL(SB_ENOMEM, "sb_truehd_index: out of host memory");
    h->channels = f.channels; h->rate = f.rate;
    auto fail = [&](int code) { sb_truehd_destroy(h); return code; };
    cudaError_t e = cudaSuccess;

    // candidates: a major sync opens every 1 to 128 AUs of at least a few dozen bytes
    int64_t cap = nbytes / 512 + 4096;
    std::vector<sbthd::Candidate> cand;
    for (int pass = 0; pass < 2; ++pass) {
        sbthd::Candidate* d_cand = nullptr;
        unsigned long long* d_count = nullptr;
        if (pool_alloc((void**)&d_cand, sizeof(sbthd::Candidate) * cap) != SB_OK) return fail(SB_ENOMEM);
        if (pool_alloc((void**)&d_count, sizeof(unsigned long long)) != SB_OK) { pool_free(d_cand); return fail(SB_ENOMEM); }
        unsigned long long count = 0;
        e = cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), c.stream);
        if (e == cudaSuccess) {
            ProfScope ps("truehd_sync");
            const int64_t words = (nbytes + 3) / 4;
            const int grid = (int)std::min<int64_t>((words + 255) / 256, (int64_t)c.sm_count * 16);
            k_truehd_sync<<<std::max(grid, 1), 256, 0, c.stream>>>(d_buf, nbytes, f, d_cand, d_count, cap);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, c.stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        if (e == cudaSuccess && (int64_t)count <= cap) {
            cand.resize(count);
            e = cudaMemcpyAsync(cand.data(), d_cand, sizeof(sbthd::Candidate) * count, cudaMemcpyDeviceToHost, c.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        }
        pool_free(d_cand); pool_free(d_count);
        if (e != cudaSuccess) { fail(0); SB_FAIL(SB_ECUDA, "sb_truehd_index: %s", cudaGetErrorString(e)); }
        if ((int64_t)count <= cap) break;
        cap = (int64_t)count;                                              // rescan with room for every candidate
    }
    std::sort(cand.begin(), cand.end(), [](const sbthd::Candidate& a, const sbthd::Candidate& b) { return a.offset < b.offset; });
    std::vector<sbthd::Segment> segs;
    int64_t n_au = 0;
    if (!sbthd::chain(host, nbytes, offsets, n, cand, where, segs, &n_au, msg, sizeof(msg))) {
        fail(0);
        SB_FAIL(SB_EINVAL, "%s", msg);
    }
    const int64_t ns = (int64_t)segs.size();
    sbthd::Segment* d_segs = nullptr;
    sbthd::SegStatus* d_status = nullptr;
    std::vector<sbthd::SegStatus> status((size_t)ns);
    int rc = pool_alloc((void**)&h->d_pcm, sizeof(int16_t) * (size_t)(n_au * f.spa * f.channels) + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_segs, sizeof(sbthd::Segment) * ns + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_status, sizeof(sbthd::SegStatus) * ns + 16);
    auto release = [&]() { pool_free(d_segs); pool_free(d_status); };
    if (rc != SB_OK) { release(); return fail(rc); }
    e = cudaMemcpyAsync(d_segs, segs.data(), sizeof(sbthd::Segment) * ns, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && ns > 0) {
        ProfScope ps("truehd_decode");
        k_truehd_decode<<<(unsigned)((ns + 63) / 64), 64, 0, c.stream>>>(d_buf, nbytes, d_blocks, n, f, d_segs, ns,
                                                                         h->d_pcm, d_status);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, sizeof(sbthd::SegStatus) * ns, cudaMemcpyDeviceToHost,
                                              c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    release();
    if (e != cudaSuccess) { fail(0); SB_FAIL(SB_ECUDA, "sb_truehd_index: %s", cudaGetErrorString(e)); }
    // messages name the failing AU by the offset of its block: walk the failing segment's AU lengths up to it
    auto where_au = [&](int64_t k, int64_t au) {
        int64_t off = segs[k].offset;
        for (int64_t a = segs[k].first_au; a < au; ++a) off += (int64_t)(((host[off] << 8) | host[off + 1]) & 0xFFF) * 2;
        return where(off);
    };
    const int64_t frames = sbthd::check_segments(segs, status.data(), f, where_au, msg, sizeof(msg));
    if (frames < 0) { sb_truehd_destroy(h); SB_FAIL(SB_EINVAL, "%s", msg); }
    h->samples = frames;
    info[0] = f.channels; info[1] = f.rate;
    *frames_out = frames;
    *out = h;
    return SB_OK;
}

}  // namespace sb

extern "C" {

int sb_truehd_index(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                    int32_t* info, sb_truehd** out, int64_t* frames_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_truehd_index: library not initialised (call sb_init)");
    if (!buf || !offsets || !file_offsets || !info || !out || !frames_out) SB_FAIL(SB_EINVAL, "sb_truehd_index: NULL argument");
    if (nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_truehd_index: empty stream");
    for (int64_t b = 0; b < n; ++b)
        if (offsets[b] < 0 || offsets[b] >= nbytes || (b > 0 && offsets[b] <= offsets[b - 1]))
            SB_FAIL(SB_EINVAL, "TrueHD block at byte offset %lld: %s", (long long)file_offsets[b],
                    offsets[b] < 0 || offsets[b] >= nbytes ? "block starts outside the buffer" : "empty block");
    const uint8_t* host = static_cast<const uint8_t*>(buf);
    // the file offset of the block holding buffer offset `off`
    auto where = [&](int64_t off) {
        const int64_t b = std::upper_bound(offsets, offsets + n, off) - offsets;
        return b > 0 && file_offsets[b - 1] >= 0 ? file_offsets[b - 1] : off;
    };
    uint8_t* d_buf = nullptr;
    int64_t* d_blocks = nullptr;
    auto release = [&]() { pool_free(d_buf); pool_free(d_blocks); };
    if (pool_alloc((void**)&d_buf, (size_t)nbytes + 16) != SB_OK || pool_alloc((void**)&d_blocks, sizeof(int64_t) * n + 16) != SB_OK) {
        release();
        SB_FAIL(SB_ENOMEM, "sb_truehd_index: out of device memory");
    }
    cudaError_t e = cudaMemsetAsync(d_buf + (nbytes & ~(int64_t)3), 0, 16, c.stream);      // zero tail for k_truehd_sync
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_buf, buf, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_blocks, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream);
    if (e != cudaSuccess) { release(); SB_FAIL(SB_ECUDA, "sb_truehd_index: %s", cudaGetErrorString(e)); }
    const int rc = truehd_index_device(host, d_buf, nbytes, offsets, d_blocks, n, where, info, out, frames_out);
    release();
    return rc;
}

int sb_truehd_decode(sb_truehd* h, int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_truehd_decode: library not initialised (call sb_init)");
    if (!h || !out_f32) SB_FAIL(SB_EINVAL, "sb_truehd_decode: NULL argument");
    sb_stream* s = nullptr;
    const int rc = load_pcm_device(reinterpret_cast<const unsigned char*>(h->d_pcm), h->samples, h->channels, 2, h->rate,
                                   sample_rate, padding, total_len, &s, "sb_truehd_decode");
    const cudaError_t e = cudaStreamSynchronize(c.stream);
    if (rc != SB_OK) return rc;
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_truehd_decode: %s", cudaGetErrorString(e)); }
    *out_f32 = s;
    return SB_OK;
}

int sb_truehd_destroy(sb_truehd* h) {
    if (!h) return SB_OK;
    pool_free(h->d_pcm);
    delete h;
    return SB_OK;
}

}  // extern "C"
