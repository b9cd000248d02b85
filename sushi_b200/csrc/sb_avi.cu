// AVI input: one audio stream of the `movi` lists demuxed on the GPU, then loaded as PCM or decoded by the MP2 decoder
// of sb_mp2.cu, the host only reading the file in large chunks (DESIGN.md section 4).  Chunks have variable sizes and
// may straddle feeds: each feed is scanned from the chain position the previous one reached, a file offset that may lie
// past the bytes fed so far (the bytes before it are then not copied).
//   sb_avi_feed    the carried bytes and the chunk side by side on the device, then
//                    k_avi_mark     per 16 positions: the chunk headers there (sb_avi.cuh is_chunk); per-CTA counts
//                    k_scan_totals  one CTA: exclusive scan of the counts, the candidate total (sb_demux.cuh)
//                  (the candidate count comes back to size the tables and launches), then
//                    k_avi_cands    the candidates' positions, in order
//                    k_avi_link     one thread per candidate: its chunk's size and the candidate it links to (across
//                                   movi lists, too), or how the chain ends there
//                    k_chain_jump   log2(candidates) rounds of pointer jumping from the buffer's first position
//                                   (sb_demux.cuh)
//                    k_avi_sel      one thread per candidate on the chain: the chain's end (the next chain position, or
//                                   a refusal), the chosen stream's payload, per-CTA payload totals
//                    k_scan_totals  one CTA: their exclusive scan on top of the running totals
//                    k_avi_place    the payload's place in the elementary stream; the chunk table
//                    k_avi_copy     one warp per chunk: its payload into the elementary-stream buffer
//                  and returns; the running totals and the chain position come back before the next chunk is placed
//   sb_avi_finish  the carried bytes as the file's end (a last chunk may be cut), then the elementary stream:
//                    PCM  k_avi_pcm, the top 16 bits of each sample, as sb_pcm_from_le stores them
//                    MP2  sb::mp2_decode, messages naming the chunk that holds a frame's header
// The per-chunk rules are in sb_avi.cuh, shared with the CPU emulation of the tests.
#include "sb_demux.cuh"
#include "sb_avi.cuh"
#include <memory>
#include <new>

using namespace sb;

namespace {

constexpr int kPer = 16;                               // positions one k_avi_mark thread checks

struct Run { long long bytes, chunks, carry, need; };  // payload bytes and chunks so far; the chain position (file
                                                       // offset); the file offset the buffer must reach before the
                                                       // next scan (a chosen chunk's end), else 0
struct ChunkRec { int64_t file_off, es_off; };         // one chunk of the stream: its file offset, its payload's place
struct Sel { int64_t off, len, dst; };                 // one chain chunk's payload in the buffer (len 0: none kept)
                                                       // and its place in the elementary stream

// the chunk headers among positions [i0, i0 + kPer) below limit, as a bit mask
__device__ __forceinline__ unsigned chunk_mask(const uint8_t* __restrict__ buf, int64_t i0, int64_t limit, int64_t n) {
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
        const int64_t i = i0 + k;
        if (i < limit && sbavi::is_chunk(buf + i, n - i)) m |= 1u << k;
    }
    return m;
}

__global__ void __launch_bounds__(kThreads)
k_avi_mark(const uint8_t* __restrict__ buf, int64_t limit, int64_t n, long long* __restrict__ cta) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kPer;
    long long total;
    block_exclusive(__popc(chunk_mask(buf, i0, limit, n)), &total);
    if (threadIdx.x == 0) cta[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads)
k_avi_cands(const uint8_t* __restrict__ buf, int64_t limit, int64_t n, const long long* __restrict__ cta,
            int64_t* __restrict__ pos) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kPer;
    unsigned m = chunk_mask(buf, i0, limit, n);
    long long total;
    long long at = cta[blockIdx.x] + block_exclusive(__popc(m), &total);
    for (; m; m &= m - 1) pos[at++] = i0 + __ffs(m) - 1;
}

// node m is the sink every chain end links to; jump[] starts as the links
__global__ void __launch_bounds__(kThreads)
k_avi_link(const uint8_t* __restrict__ buf, int64_t n, int64_t limit, int at_end, int64_t base,
           const int64_t* __restrict__ ext, int64_t n_ext, uint32_t tag, const int64_t* __restrict__ pos, int64_t m,
           sbavi::Link* __restrict__ links, int32_t* __restrict__ jump, uint8_t* __restrict__ on, Run* __restrict__ run,
           unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) {
        run->carry = base + n;                          // unless the chain's end says otherwise (k_avi_sel)
        run->need = 0;
        jump[m] = (int32_t)m;
        on[m] = 0;
        if (m == 0 || pos[0] != 0) fail_at(err, base, sbavi::kNoChunk);
    }
    if (k >= m) return;
    const sbavi::Link l = sbavi::link(buf, pos[k], n, limit, at_end != 0, base, ext, n_ext, tag,
                                      [&](int64_t p) { return find_cand(pos, m, p) >= 0; });
    links[k] = l;
    jump[k] = (int32_t)(l.kind == sbavi::kLink ? find_cand(pos, m, l.next) : m);
    on[k] = k == 0 && pos[0] == 0;
}

// one thread per candidate: on the chain, the chosen stream's payload; the chain's end
__global__ void __launch_bounds__(kThreads)
k_avi_sel(const uint8_t* __restrict__ buf, int64_t n, int at_end, int64_t base, uint32_t tag, int64_t frame_bytes,
          const int64_t* __restrict__ pos, int64_t m, const sbavi::Link* __restrict__ links,
          const uint8_t* __restrict__ on, Sel* __restrict__ sel, long long* __restrict__ cta, Run* __restrict__ run,
          uint32_t* __restrict__ cut, unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Sel s{0, 0, 0};
    if (k < m && on[k]) {
        const int64_t q = pos[k];
        const sbavi::Link l = links[k];
        bool whole = true;
        if (l.kind == sbavi::kOverrun) { fail_at(err, base + q, sbavi::kPastList); whole = false; }
        else if (l.kind == sbavi::kBroken) fail_at(err, base + l.next, sbavi::kNoChunk);
        else if (l.kind == sbavi::kNext) run->carry = l.next == sbavi::kDone ? sbavi::kDone : base + l.next;
        else if (l.kind == sbavi::kPast) {
            whole = at_end != 0;                        // carried to the next feed, or cut by the file's end
            run->carry = at_end ? base + n : base + q;
            if (!at_end) run->need = base + q + 8 + l.size;
        }
        if (whole && sbavi::rd32(buf + q) == tag) {
            if (frame_bytes && l.size % frame_bytes) fail_at(err, base + q, sbavi::kPartialFrame);
            else {
                const int64_t len = min(l.size, n - q - 8);
                if (len < l.size) atomicOr(cut, 1u);
                if (len > 0) s = Sel{q + 8, len, 0};
            }
        }
    }
    if (k < m) sel[k] = s;
    long long tb, tp;
    block_exclusive(s.len, &tb);
    block_exclusive(s.len > 0, &tp);
    if (threadIdx.x == 0) { cta[2 * blockIdx.x] = tb; cta[2 * blockIdx.x + 1] = tp; }
}

__global__ void __launch_bounds__(kThreads)
k_avi_place(int64_t base, const int64_t* __restrict__ pos, int64_t m, Sel* __restrict__ sel,
            const long long* __restrict__ cta, ChunkRec* __restrict__ tab) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t len = k < m ? sel[k].len : 0;
    long long tb, tp;
    const long long eb = cta[2 * blockIdx.x] + block_exclusive(len, &tb);
    const long long ep = cta[2 * blockIdx.x + 1] + block_exclusive(len > 0, &tp);
    if (len <= 0) return;
    tab[ep] = ChunkRec{base + pos[k], eb};
    sel[k].dst = eb;
}

__global__ void __launch_bounds__(kThreads)
k_avi_copy(const uint8_t* __restrict__ buf, int64_t m, const Sel* __restrict__ sel, uint8_t* __restrict__ es) {
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= m) return;
    const Sel s = sel[k];
    for (int64_t b = threadIdx.x & 31; b < s.len; b += 32) es[s.dst + b] = buf[s.off + b];
}

// little-endian 16- or 24-bit samples -> the top 16 bits as int16
__global__ void __launch_bounds__(kThreads)
k_avi_pcm(const uint8_t* __restrict__ in, int64_t n, int width, int16_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint8_t* p = in + i * width + (width - 2);
        out[i] = (int16_t)(uint16_t)(p[0] | ((unsigned)p[1] << 8));
    }
}

}  // namespace

struct sb_avi : ChunkedDemux<Run> {
    uint32_t tag = 0;
    int codec = 0, channels = 0, width = 0, rate = 0;
    int64_t n_ext = 0;
    int64_t* d_ext = nullptr;
    uint8_t* d_buf[2] = {nullptr, nullptr}; int64_t buf_cap[2] = {0, 0};
    int cur = 0;                                        // the buffer the last chunk went to
    int64_t buf_len = 0, buf_off = 0;                   // its bytes, and the file offset of its first byte
    long long* d_cta = nullptr; int64_t cta_cap = 0;
    int64_t* d_pos = nullptr; int64_t pos_cap = 0;
    sbavi::Link* d_links = nullptr; int64_t links_cap = 0;
    int32_t* d_jump[2] = {nullptr, nullptr}; int64_t jump_cap[2] = {0, 0};
    uint8_t* d_on = nullptr; int64_t on_cap = 0;
    Sel* d_sel = nullptr; int64_t sel_cap = 0;
    uint8_t* d_es = nullptr; int64_t es_cap = 0;
    ChunkRec* d_tab = nullptr; int64_t tab_cap = 0;
    Run* d_run = nullptr;
    long long* d_count = nullptr;
    uint32_t* d_cut = nullptr;
    long long* h_count = nullptr;                       // pinned copy of *d_count; *h_run is that of *d_run

    ~sb_avi() {
        release_demux();
        pool_free(d_ext); pool_free(d_run); pool_free(d_count); pool_free(d_cut);
        if (h_count) cudaFreeHost(h_count);
    }
    void release_demux() {
        for (int b = 0; b < 2; ++b) { pool_free(d_buf[b]); pool_free(d_jump[b]); d_buf[b] = nullptr; d_jump[b] = nullptr;
                                      buf_cap[b] = jump_cap[b] = 0; }
        pool_free(d_cta); pool_free(d_pos); pool_free(d_links); pool_free(d_on); pool_free(d_sel); pool_free(d_es);
        pool_free(d_tab);
        d_cta = nullptr; d_pos = nullptr; d_links = nullptr; d_on = nullptr; d_sel = nullptr; d_es = nullptr;
        d_tab = nullptr;
        cta_cap = pos_cap = links_cap = on_cap = sel_cap = es_cap = tab_cap = 0;
    }
};

namespace {

// Scan buf[0, n) (file offset base): the chunk chain from position 0, the stream's payload appended.  `at_end`: the
// buffer ends the file.  Returns once the kernels are enqueued (the candidate count having come back first).
int scan_buffer(sb_avi* t, const uint8_t* buf, int64_t n, int64_t base, bool at_end, const char* who) {
    Ctx& c = ctx();
    const int64_t limit = at_end ? n : n - sbavi::kTail;
    const Run run = *t->h_run;
    const int64_t n_thr = (limit + kPer - 1) / kPer, n_cta = std::max<int64_t>(1, (n_thr + kThreads - 1) / kThreads);
    if (grow(&t->d_cta, &t->cta_cap, 0, 2 * n_cta + 2, c.stream) != SB_OK)
        SB_FAIL(SB_ENOMEM, "%s: out of device memory for a chunk of %lld bytes", who, (long long)n);
    cudaError_t e = cudaSuccess;
    {
        ProfScope ps("avi_mark", 2);
        k_avi_mark<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(buf, limit, n, t->d_cta);
        k_scan_totals<1><<<1, 1024, 0, c.stream>>>(t->d_cta, n_cta, nullptr, t->d_count);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->h_count, t->d_count, sizeof(long long), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    // chunk headers may lie two bytes apart (`ix00wb`), so the candidate table is sized by the count
    const int64_t m = *t->h_count;
    const int64_t m_cta = std::max<int64_t>(1, (m + kThreads - 1) / kThreads);
    int rc = grow(&t->d_pos, &t->pos_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) {
        ProfScope ps("avi_cands");
        k_avi_cands<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(buf, limit, n, t->d_cta, t->d_pos);
        e = cudaGetLastError();
    }
    if (rc == SB_OK) rc = grow(&t->d_links, &t->links_cap, 0, m + 1, c.stream);
    for (int b = 0; b < 2 && rc == SB_OK; ++b) rc = grow(&t->d_jump[b], &t->jump_cap[b], 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_on, &t->on_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_sel, &t->sel_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_cta, &t->cta_cap, 0, 2 * m_cta + 2, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_es, &t->es_cap, run.bytes, run.bytes + n, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_tab, &t->tab_cap, run.chunks, run.chunks + m + 1, c.stream);
    if (rc != SB_OK) SB_FAIL(rc, "%s: out of device memory for a chunk of %lld bytes", who, (long long)n);
    SB_TRY(cuda_result(e, who));
    const int64_t frame_bytes = t->codec == SB_AVI_PCM ? (int64_t)t->channels * t->width : 0;
    {
        ProfScope ps("avi_chain");
        k_avi_link<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, n, limit, at_end, base, t->d_ext, t->n_ext, t->tag,
                                                              t->d_pos, m, t->d_links, t->d_jump[0], t->d_on, t->d_run,
                                                              t->d_err);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = mark_chain(t->d_jump, t->d_on, m, "avi_chain", c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("avi_compact", 4);
        k_avi_sel<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, n, at_end, base, t->tag, frame_bytes, t->d_pos, m,
                                                             t->d_links, t->d_on, t->d_sel, t->d_cta, t->d_run, t->d_cut,
                                                             t->d_err);
        k_scan_totals<2><<<1, 1024, 0, c.stream>>>(t->d_cta, m_cta, reinterpret_cast<long long*>(t->d_run),
                                                  reinterpret_cast<long long*>(t->d_run));
        k_avi_place<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(base, t->d_pos, m, t->d_sel, t->d_cta, t->d_tab);
        k_avi_copy<<<(unsigned)((m * 32 + kThreads - 1) / kThreads + 1), kThreads, 0, c.stream>>>(buf, m, t->d_sel,
                                                                                                 t->d_es);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->h_run, t->d_run, sizeof(Run), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaEventRecord(t->done, c.stream);
    SB_TRY(cuda_result(e, who));
    t->pending = true;
    return SB_OK;
}

// The PCM of the elementary stream (run.bytes bytes of whole frames, a cut last frame dropped) as an sb_pcm
int pcm_out(sb_avi* t, const Run& run, sb_pcm** out, const char* who) {
    Ctx& c = ctx();
    const int64_t frames = run.bytes / ((int64_t)t->channels * t->width), n = frames * t->channels;
    int16_t* d_pcm = nullptr;
    SB_TRY(pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)n + 16));
    cudaError_t e = cudaSuccess;
    if (n > 0) {
        ProfScope ps("avi_pcm");
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads,
                                                                     (int64_t)c.sm_count * 16));
        k_avi_pcm<<<grid, kThreads, 0, c.stream>>>(t->d_es, n, t->width, d_pcm);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { pool_free(d_pcm); SB_FAIL(SB_ECUDA, "%s: %s", who, cudaGetErrorString(e)); }
    return pcm_handle(d_pcm, frames, t->channels, t->rate, out);
}

}  // namespace

extern "C" {

int sb_avi_open(int32_t stream_index, int32_t codec, const int32_t* config, const int64_t* movi_extents,
                int64_t n_extents, sb_avi** out) {
    const char* who = "sb_avi_open";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, out && config && (movi_extents || !n_extents)));
    if (stream_index < 0 || stream_index > 99)
        SB_FAIL(SB_EINVAL, "sb_avi_open: stream %d (chunk FOURCCs name streams 0 to 99)", stream_index);
    if (codec != SB_AVI_PCM && codec != SB_AVI_MP2) SB_FAIL(SB_EINVAL, "sb_avi_open: codec %d", codec);
    if (codec == SB_AVI_PCM && (config[0] < 1 || config[0] > 8 || (config[1] != 16 && config[1] != 24) ||
                                config[2] < 1))
        SB_FAIL(SB_EINVAL, "sb_avi_open: PCM of %d channels, %d bits at %d Hz (16 or 24 bits, 1 to 8 channels)",
                config[0], config[1], config[2]);
    if (n_extents < 0) SB_FAIL(SB_EINVAL, "sb_avi_open: %lld movi extents", (long long)n_extents);
    for (int64_t e = 0; e < n_extents; ++e)
        if (movi_extents[2 * e] >= movi_extents[2 * e + 1] || (e && movi_extents[2 * e] < movi_extents[2 * e - 1]))
            SB_FAIL(SB_EINVAL, "sb_avi_open: movi extent %lld is empty or out of order", (long long)e);
    std::unique_ptr<sb_avi> t(new (std::nothrow) sb_avi());
    if (!t) SB_FAIL(SB_ENOMEM, "sb_avi_open: out of host memory");
    t->tag = sbavi::audio_tag(stream_index);
    t->codec = codec;
    t->channels = config[0]; t->width = config[1] / 8; t->rate = config[2];
    t->n_ext = n_extents;
    SB_TRY(t->open(who));
    t->h_run->carry = n_extents ? movi_extents[0] : sbavi::kDone;
    SB_TRY(cuda_result(cudaMallocHost((void**)&t->h_count, sizeof(long long)), who));
    if (pool_alloc((void**)&t->d_run, sizeof(Run)) != SB_OK || pool_alloc((void**)&t->d_count, 16) != SB_OK ||
        pool_alloc((void**)&t->d_cut, 16) != SB_OK ||
        pool_alloc((void**)&t->d_ext, sizeof(int64_t) * (size_t)(2 * n_extents) + 16) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_avi_open: out of device memory");
    cudaError_t e = cudaMemsetAsync(t->d_run, 0, sizeof(Run), c.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(t->d_cut, 0, sizeof(uint32_t), c.stream);
    if (e == cudaSuccess && n_extents)
        e = cudaMemcpyAsync(t->d_ext, movi_extents, sizeof(int64_t) * (size_t)(2 * n_extents), cudaMemcpyHostToDevice,
                            c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    *out = t.release();
    return SB_OK;
}

int sb_avi_feed(sb_avi* t, const void* host_chunk, int64_t nbytes, int64_t file_offset) {
    const char* who = "sb_avi_feed";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && (host_chunk || !nbytes)));
    SB_TRY(t->feed_check(who, nbytes, file_offset, 1));
    if (!nbytes) return SB_OK;
    SB_TRY(t->settle(who));
    t->next_offset += nbytes;
    const int64_t at = t->h_run->carry;                 // the chain position
    if (at == sbavi::kDone || at >= file_offset + nbytes) {   // nothing of this chunk is read
        t->buf_len = 0;
        t->buf_off = file_offset + nbytes;
        return SB_OK;
    }
    // the bytes from the chain position: the tail of the last buffer, then this chunk (or this chunk's tail)
    const int64_t carry = at < file_offset ? t->buf_off + t->buf_len - at : 0;
    const int64_t skip = at > file_offset ? at - file_offset : 0, n = carry + nbytes - skip;
    const int nb = t->cur ^ 1;
    if (grow(&t->d_buf[nb], &t->buf_cap[nb], 0, n, c.stream) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_avi_feed: out of device memory for a chunk of %lld bytes", (long long)nbytes);
    cudaError_t e = cudaSuccess;
    if (carry) e = cudaMemcpyAsync(t->d_buf[nb], t->d_buf[t->cur] + (at - t->buf_off), (size_t)carry,
                                   cudaMemcpyDeviceToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->d_buf[nb] + carry, static_cast<const uint8_t*>(host_chunk) + skip,
                                              (size_t)(nbytes - skip), cudaMemcpyHostToDevice, c.stream);
    SB_TRY(cuda_result(e, who));
    t->cur = nb;
    t->buf_len = n;
    t->buf_off = at;
    // too short to read a chunk header, or short of the end of a chunk of the stream: all of it waits for more
    if (n <= sbavi::kTail || at + n < t->h_run->need)
        return cuda_result(cudaStreamSynchronize(c.stream), who);
    // scan_buffer waits for the candidate count, so the chunk has been copied when it returns
    return scan_buffer(t, t->d_buf[nb], n, t->buf_off, false, who);
}

int sb_avi_finish(sb_avi* t, int32_t* cut, sb_pcm** out) {
    const char* who = "sb_avi_finish";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && cut && out));
    SB_TRY(t->finish_check(who));
    ReleaseDemux<sb_avi> release_demux{t};
    SB_TRY(t->settle(who));
    // what the last feed left over, as the end of the file; a chain that stops short of the last movi list's end is a
    // file cut there
    bool short_chain = false;
    const int64_t at = t->h_run->carry;
    if (at != sbavi::kDone) {
        const int64_t rem = at >= t->buf_off ? t->buf_off + t->buf_len - at : 0;
        if (rem >= sbavi::kHeader) {
            SB_TRY(scan_buffer(t, t->d_buf[t->cur] + (at - t->buf_off), rem, at, true, who));
            SB_TRY(t->settle(who));
        }
        short_chain = t->h_run->carry != sbavi::kDone;
    }
    SB_TRY(t->check_failure(who, [](int) { return "AVI chunk"; }, sbavi::error_text));
    uint32_t was_cut = 0;
    SB_TRY(collect(cudaSuccess, &was_cut, t->d_cut, 1, who));
    const Run run = *t->h_run;
    if (run.chunks < 1 || run.bytes < 1) SB_FAIL(SB_EINVAL, "stream %c%c carries no audio chunk", (char)(t->tag & 0xFF),
                                                 (char)((t->tag >> 8) & 0xFF));
    if (t->codec == SB_AVI_PCM) {
        *cut = was_cut || short_chain;
        return pcm_out(t, run, out, who);
    }
    std::vector<uint8_t> host((size_t)run.bytes + 1);
    std::vector<ChunkRec> tab((size_t)run.chunks);
    // the elementary stream is put together on the device, so its zero tail (sb_decode.h) is written here
    cudaError_t e = cudaMemsetAsync(t->d_es + (run.bytes & ~(long long)3), 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(tab.data(), t->d_tab, sizeof(ChunkRec) * (size_t)run.chunks,
                                              cudaMemcpyDeviceToHost, c.stream);
    SB_TRY(collect(e, host.data(), t->d_es, run.bytes, who));
    // messages name the chunk holding a stream byte
    auto where = [&](int64_t b) { return file_offset_of(tab, b); };
    int32_t dropped = 0;
    SB_TRY(mp2_decode(host.data(), t->d_es, run.bytes, where, &dropped, out));
    *cut = was_cut || short_chain || dropped;
    return SB_OK;
}

int sb_avi_destroy(sb_avi* t) { return destroy_demux(t); }

}  // extern "C"
