// Dolby TrueHD input: the stream's restart segments decoded on the GPU into the interleaved int16 PCM that sb_load_pcm
// decodes from a WAV file, then the loader's own kernel (k_decode_resample_pad, width 2) from there on.
//   sb_truehd_decode  upload the stream; k_truehd_sync lists every byte position holding a major sync whose CRC passes
//                     (false syncs inside coded data included) and whether its decoded substreams open with restart
//                     headers; the host walks the AU lengths from the start, block by block, into restart segments
//                     (only a listed sync at an AU start begins one); k_truehd_decode gives one thread to each segment,
//                     which decodes its AUs in turn into int16 at AU index x samples per AU and returns its lossless
//                     check; the host joins the checks of neighbouring segments
// The per-AU arithmetic is in sb_truehd.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
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

namespace sb {

// The body of sb_truehd_decode on a stream already on the device: `host` and `d_buf` hold the same `nbytes` bytes (d_buf
// followed by the zero bytes of sb_decode.h's contract, for k_truehd_sync); blocks start at offsets[0..n) (d_blocks: the same on
// the device); where(off) is the file offset messages give for stream byte `off`.  The caller keeps d_buf and d_blocks.
int truehd_index_device(const uint8_t* host, const uint8_t* d_buf, int64_t nbytes, const int64_t* offsets,
                        const int64_t* d_blocks, int64_t n, const std::function<int64_t(int64_t)>& where, sb_pcm** out) {
    Ctx& c = ctx();
    sbthd::Format f;
    char msg[256], fmsg[200];
    if (!sbthd::parse_format(host, nbytes, offsets[0], &f, fmsg, sizeof(fmsg))) {
        snprintf(msg, sizeof(msg), fmsg, (long long)where(offsets[0]));
        SB_FAIL(SB_EINVAL, "%s", msg);
    }
    const char* who = "sb_truehd_decode";       // a transport stream's payload comes through sb_ts_finish: same name

    // candidates: a major sync opens every 1 to 128 AUs of at least a few dozen bytes
    std::vector<sbthd::Candidate> cand;
    SB_TRY(scan_candidates(nbytes / 512 + 4096, "truehd_sync", who, [&](sbthd::Candidate* d_cand, unsigned long long* d_count, int64_t cap) {
        const int64_t words = (nbytes + 3) / 4;
        const int grid = (int)std::min<int64_t>((words + 255) / 256, (int64_t)c.sm_count * 16);
        k_truehd_sync<<<std::max(grid, 1), 256, 0, c.stream>>>(d_buf, nbytes, f, d_cand, d_count, cap);
    }, cand));
    std::sort(cand.begin(), cand.end(), [](const sbthd::Candidate& a, const sbthd::Candidate& b) { return a.offset < b.offset; });
    std::vector<sbthd::Segment> segs;
    int64_t n_au = 0;
    if (!sbthd::chain(host, nbytes, offsets, n, cand, where, segs, &n_au, msg, sizeof(msg))) SB_FAIL(SB_EINVAL, "%s", msg);
    const int64_t ns = (int64_t)segs.size();
    Blocks blocks;
    sbthd::Segment* d_segs = nullptr;
    sbthd::SegStatus* d_status = nullptr;
    int16_t* d_pcm = nullptr;
    std::vector<sbthd::SegStatus> status((size_t)ns);
    SB_TRY(blocks.alloc(&d_pcm, (size_t)(n_au * f.spa * f.channels)));
    SB_TRY(blocks.alloc(&d_segs, (size_t)ns));
    SB_TRY(blocks.alloc(&d_status, (size_t)ns));
    cudaError_t e = cudaMemcpyAsync(d_segs, segs.data(), sizeof(sbthd::Segment) * ns, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && ns > 0) {
        ProfScope ps("truehd_decode");
        k_truehd_decode<<<(unsigned)((ns + 63) / 64), 64, 0, c.stream>>>(d_buf, nbytes, d_blocks, n, f, d_segs, ns,
                                                                         d_pcm, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, ns, who));
    // messages name the failing AU by the offset of its block: walk the failing segment's AU lengths up to it
    auto where_au = [&](int64_t k, int64_t au) {
        int64_t off = segs[k].offset;
        for (int64_t a = segs[k].first_au; a < au; ++a) off += (int64_t)(((host[off] << 8) | host[off + 1]) & 0xFFF) * 2;
        return where(off);
    };
    const int64_t frames = sbthd::check_segments(segs, status.data(), f, where_au, msg, sizeof(msg));
    if (frames < 0) SB_FAIL(SB_EINVAL, "%s", msg);
    return pcm_handle(blocks.take(d_pcm), frames, f.channels, f.rate, out);
}

}  // namespace sb

extern "C" {

int sb_truehd_decode(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                     sb_pcm** out) {
    const char* who = "sb_truehd_decode";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, buf && offsets && file_offsets && out));
    if (nbytes < 1 || n < 1) SB_FAIL(SB_EINVAL, "sb_truehd_decode: empty stream");
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
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    int64_t* d_blocks = nullptr;
    int rc = upload_padded(blocks, &d_buf, buf, nbytes, who);
    if (rc == SB_OK) rc = blocks.alloc(&d_blocks, (size_t)n);
    if (rc == SB_ENOMEM) SB_FAIL(SB_ENOMEM, "sb_truehd_decode: out of device memory");
    SB_TRY(rc);
    SB_TRY(cuda_result(cudaMemcpyAsync(d_blocks, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream), who));
    return truehd_index_device(host, d_buf, nbytes, offsets, d_blocks, n, where, out);
}

}  // extern "C"
