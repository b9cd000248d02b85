// MPEG program stream input: one MPEG audio stream demuxed on the GPU and decoded by the MP2 decoder of sb_mp2.cu, the
// host only reading the file in large chunks (DESIGN.md section 4).  Packets have variable lengths and may straddle
// chunks: each chunk is scanned behind the bytes carried over from the one before, which start at the chain position
// the previous chunk reached.
//   sb_ps_feed     one chunk: the carried bytes and the chunk side by side on the device, then
//                    k_ps_mark      per 16 positions: the start codes there (00 00 01 xx, xx >= 0xB9); per-CTA counts
//                    k_scan_totals  one CTA: exclusive scan of the counts, the candidate total (sb_demux.cuh)
//                    k_ps_cands     the candidates' positions, in order
//                  (the candidate count comes back to size the launches), then
//                    k_ps_link      one thread per candidate: its packet's length and the candidate it links to (or how
//                                   the chain ends there)
//                    k_chain_jump   log2(candidates) rounds of pointer jumping from the chunk's first position: each
//                                   round, every candidate on the chain marks the one 2^r links on, and the links double
//                                   (sb_demux.cuh)
//                    k_ps_pes       one thread per candidate on the chain: the chain's end (the next chunk's carry, or a
//                                   refusal), the chosen stream's PES header, per-CTA payload totals
//                    k_scan_totals  one CTA: their exclusive scan on top of the running totals
//                    k_ps_place     the payload's place in the elementary stream; the PES table
//                    k_ps_copy      one warp per PES: its payload into the elementary-stream buffer
//                  and returns; the running totals and the carry position come back before the next chunk is placed
//   sb_ps_finish   the carried bytes as the file's end (a last PES may be cut), then the elementary stream through
//                  sb::mp2_decode, messages naming the PES that holds a frame's header
// The per-packet rules are in sb_ps.cuh, shared with the CPU emulation of the tests.
#include "sb_demux.cuh"
#include "sb_ps.cuh"
#include <memory>
#include <new>

using namespace sb;

namespace {

constexpr int kPer = 16;                               // positions one k_ps_mark thread checks

struct Run { long long bytes, pes, carry; };           // payload bytes and PES so far; where the last chunk's carry starts
struct PesRec { int64_t file_off, es_off; };           // one PES of the stream: its file offset, its payload's place
struct Sel { int64_t off, len, dst; };                 // one chain packet's payload in the buffer (len 0: none kept)
                                                       // and its place in the elementary stream

// the start codes among positions [i0, i0 + kPer) below limit, as a bit mask
__device__ __forceinline__ unsigned start_mask(const uint8_t* __restrict__ buf, int64_t i0, int64_t limit) {
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
        const int64_t i = i0 + k;
        if (i < limit && sbps::is_start(buf + i)) m |= 1u << k;
    }
    return m;
}

__global__ void __launch_bounds__(kThreads)
k_ps_mark(const uint8_t* __restrict__ buf, int64_t limit, long long* __restrict__ cta) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kPer;
    long long total;
    block_exclusive(__popc(start_mask(buf, i0, limit)), &total);
    if (threadIdx.x == 0) cta[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads)
k_ps_cands(const uint8_t* __restrict__ buf, int64_t limit, const long long* __restrict__ cta,
           int64_t* __restrict__ pos) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kPer;
    unsigned m = start_mask(buf, i0, limit);
    long long total;
    long long at = cta[blockIdx.x] + block_exclusive(__popc(m), &total);
    for (; m; m &= m - 1) pos[at++] = i0 + __ffs(m) - 1;
}

// node m is the sink every chain end links to; jump[] starts as the links
__global__ void __launch_bounds__(kThreads)
k_ps_link(const uint8_t* __restrict__ buf, int64_t n, int64_t limit, int at_end, int64_t file_off0,
          const int64_t* __restrict__ pos, int64_t m, sbps::Link* __restrict__ links, int32_t* __restrict__ jump,
          uint8_t* __restrict__ on, Run* __restrict__ run, unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) {
        run->carry = n;                                 // unless the chain's end says otherwise (k_ps_pes)
        jump[m] = (int32_t)m;
        on[m] = 0;
        if (m == 0 || pos[0] != 0) fail_at(err, file_off0, sbps::kNoStartCode);
    }
    if (k >= m) return;
    const sbps::Link l = sbps::link(buf, pos[k], n, limit, at_end != 0,
                                    [&](int64_t p) { return find_cand(pos, m, p) >= 0; });
    links[k] = l;
    jump[k] = (int32_t)(l.kind == sbps::kLink ? find_cand(pos, m, l.next) : m);
    on[k] = k == 0 && pos[0] == 0;
}

// one thread per candidate: on the chain, the chosen stream's PES payload; the chain's end
__global__ void __launch_bounds__(kThreads)
k_ps_pes(const uint8_t* __restrict__ buf, int64_t n, int at_end, int64_t file_off0, int stream_id,
         const int64_t* __restrict__ pos, int64_t m, const sbps::Link* __restrict__ links, const uint8_t* __restrict__ on,
         Sel* __restrict__ sel, long long* __restrict__ cta, Run* __restrict__ run, uint32_t* __restrict__ cut,
         unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Sel s{0, 0, 0};
    if (k < m && on[k]) {
        const int64_t q = pos[k];
        const sbps::Link l = links[k];
        bool whole = true;
        if (l.kind == sbps::kBadHeader) { fail_at(err, file_off0 + q, sbps::kBadPack); whole = false; }
        else if (l.kind == sbps::kBroken) { fail_at(err, file_off0 + l.next, sbps::kNoStartCode); run->carry = n; }
        else if (l.kind == sbps::kNext) run->carry = l.next;
        else if (l.kind == sbps::kPast) {
            whole = at_end != 0;                        // carried to the next chunk, or cut by the file's end
            run->carry = at_end ? n : q;
        }
        if (whole && buf[q + 3] == stream_id) {
            const sbps::Pes p = sbps::parse_pes(buf + q, n - q);
            if (p.code) fail_at(err, file_off0 + q, p.code);
            else {
                if (p.cut) atomicOr(cut, 1u);
                if (p.cut != 2) s = Sel{q + p.payload_off, p.payload_len, 0};
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
k_ps_place(int64_t file_off0, const int64_t* __restrict__ pos, int64_t m, Sel* __restrict__ sel,
           const long long* __restrict__ cta, PesRec* __restrict__ tab) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t len = k < m ? sel[k].len : 0;
    long long tb, tp;
    const long long eb = cta[2 * blockIdx.x] + block_exclusive(len, &tb);
    const long long ep = cta[2 * blockIdx.x + 1] + block_exclusive(len > 0, &tp);
    if (len <= 0) return;
    tab[ep] = PesRec{file_off0 + pos[k], eb};
    sel[k].dst = eb;
}

__global__ void __launch_bounds__(kThreads)
k_ps_copy(const uint8_t* __restrict__ buf, int64_t m, const Sel* __restrict__ sel, uint8_t* __restrict__ es) {
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= m) return;
    const Sel s = sel[k];
    for (int64_t b = threadIdx.x & 31; b < s.len; b += 32) es[s.dst + b] = buf[s.off + b];
}

}  // namespace

struct sb_ps : ChunkedDemux<Run> {
    int stream_id = 0;
    uint8_t* d_buf[2] = {nullptr, nullptr}; int64_t buf_cap[2] = {0, 0};
    int cur = 0;                                        // the buffer the last chunk went to
    int64_t buf_len = 0, buf_off = 0;                   // its bytes, and the file offset of its first byte
    long long* d_cta = nullptr; int64_t cta_cap = 0;
    int64_t* d_pos = nullptr; int64_t pos_cap = 0;
    sbps::Link* d_links = nullptr; int64_t links_cap = 0;
    int32_t* d_jump[2] = {nullptr, nullptr}; int64_t jump_cap[2] = {0, 0};
    uint8_t* d_on = nullptr; int64_t on_cap = 0;
    Sel* d_sel = nullptr; int64_t sel_cap = 0;
    uint8_t* d_es = nullptr; int64_t es_cap = 0;
    PesRec* d_tab = nullptr; int64_t tab_cap = 0;
    Run* d_run = nullptr;
    long long* d_count = nullptr;
    uint32_t* d_cut = nullptr;
    long long* h_count = nullptr;                       // pinned copy of *d_count; *h_run is that of *d_run

    ~sb_ps() {
        release_demux();
        pool_free(d_run); pool_free(d_count); pool_free(d_cut);
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

// Scan buf[0, n) of the current buffer (file offset base): the packet chain from position 0, the stream's payload
// appended.  `at_end`: the buffer ends the file.  Returns once the kernels are enqueued (the candidate count having
// come back first).
int scan_buffer(sb_ps* t, const uint8_t* buf, int64_t n, int64_t base, bool at_end, const char* who) {
    Ctx& c = ctx();
    const int64_t limit = at_end ? n - 3 : n - sbps::kTail;       // every candidate's 4 bytes lie inside
    const Run run = *t->h_run;
    const int64_t n_thr = (limit + kPer - 1) / kPer, n_cta = std::max<int64_t>(1, (n_thr + kThreads - 1) / kThreads);
    int rc = grow(&t->d_cta, &t->cta_cap, 0, 2 * n_cta + 2, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_pos, &t->pos_cap, 0, limit / 4 + 1, c.stream);
    if (rc != SB_OK) SB_FAIL(rc, "%s: out of device memory for a chunk of %lld bytes", who, (long long)n);
    cudaError_t e = cudaSuccess;
    {
        ProfScope ps("ps_mark", 3);
        k_ps_mark<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(buf, limit, t->d_cta);
        k_scan_totals<1><<<1, 1024, 0, c.stream>>>(t->d_cta, n_cta, nullptr, t->d_count);
        k_ps_cands<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(buf, limit, t->d_cta, t->d_pos);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->h_count, t->d_count, sizeof(long long), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    const int64_t m = *t->h_count;
    const int64_t m_cta = std::max<int64_t>(1, (m + kThreads - 1) / kThreads);
    rc = grow(&t->d_links, &t->links_cap, 0, m + 1, c.stream);
    for (int b = 0; b < 2 && rc == SB_OK; ++b) rc = grow(&t->d_jump[b], &t->jump_cap[b], 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_on, &t->on_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_sel, &t->sel_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_cta, &t->cta_cap, 0, 2 * m_cta + 2, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_es, &t->es_cap, run.bytes, run.bytes + n, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_tab, &t->tab_cap, run.pes, run.pes + m + 1, c.stream);
    if (rc != SB_OK) SB_FAIL(rc, "%s: out of device memory for a chunk of %lld bytes", who, (long long)n);
    {
        ProfScope ps("ps_chain");
        k_ps_link<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, n, limit, at_end, base, t->d_pos, m, t->d_links,
                                                             t->d_jump[0], t->d_on, t->d_run, t->d_err);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = mark_chain(t->d_jump, t->d_on, m, "ps_chain", c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("ps_compact", 4);
        k_ps_pes<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, n, at_end, base, t->stream_id, t->d_pos, m, t->d_links,
                                                            t->d_on, t->d_sel, t->d_cta, t->d_run, t->d_cut, t->d_err);
        k_scan_totals<2><<<1, 1024, 0, c.stream>>>(t->d_cta, m_cta, reinterpret_cast<long long*>(t->d_run),
                                                  reinterpret_cast<long long*>(t->d_run));
        k_ps_place<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(base, t->d_pos, m, t->d_sel, t->d_cta, t->d_tab);
        k_ps_copy<<<(unsigned)((m * 32 + kThreads - 1) / kThreads + 1), kThreads, 0, c.stream>>>(buf, m, t->d_sel, t->d_es);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->h_run, t->d_run, sizeof(Run), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaEventRecord(t->done, c.stream);
    SB_TRY(cuda_result(e, who));
    t->pending = true;
    return SB_OK;
}

}  // namespace

extern "C" {

int sb_ps_open(int32_t stream_id, int32_t substream_id, sb_ps** out) {
    const char* who = "sb_ps_open";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, out));
    if (stream_id < 0xC0 || stream_id > 0xDF)
        SB_FAIL(SB_EINVAL, "sb_ps_open: stream id 0x%x (MPEG audio streams, 0xC0 to 0xDF, are decoded)", stream_id);
    if (substream_id != -1) SB_FAIL(SB_EINVAL, "sb_ps_open: substream %d (MPEG audio streams have none)", substream_id);
    std::unique_ptr<sb_ps> t(new (std::nothrow) sb_ps());
    if (!t) SB_FAIL(SB_ENOMEM, "sb_ps_open: out of host memory");
    t->stream_id = stream_id;
    SB_TRY(t->open(who));
    SB_TRY(cuda_result(cudaMallocHost((void**)&t->h_count, sizeof(long long)), who));
    if (pool_alloc((void**)&t->d_run, sizeof(Run)) != SB_OK || pool_alloc((void**)&t->d_count, 16) != SB_OK ||
        pool_alloc((void**)&t->d_cut, 16) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_ps_open: out of device memory");
    cudaError_t e = cudaMemsetAsync(t->d_run, 0, sizeof(Run), c.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(t->d_cut, 0, sizeof(uint32_t), c.stream);
    SB_TRY(cuda_result(e, who));
    *out = t.release();
    return SB_OK;
}

int sb_ps_feed(sb_ps* t, const void* host_chunk, int64_t nbytes, int64_t file_offset) {
    const char* who = "sb_ps_feed";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && (host_chunk || !nbytes)));
    SB_TRY(t->feed_check(who, nbytes, file_offset, 1));
    if (!nbytes) return SB_OK;
    SB_TRY(t->settle(who));
    // the bytes from the chain position the last chunk reached, then this chunk, in the other buffer
    const int64_t carry_from = t->buf_len ? std::min<int64_t>(t->h_run->carry, t->buf_len) : 0;
    const int64_t carry = t->buf_len - carry_from, n = carry + nbytes;
    const int nb = t->cur ^ 1;
    if (grow(&t->d_buf[nb], &t->buf_cap[nb], 0, n, c.stream) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_ps_feed: out of device memory for a chunk of %lld bytes", (long long)nbytes);
    cudaError_t e = cudaSuccess;
    if (carry) e = cudaMemcpyAsync(t->d_buf[nb], t->d_buf[t->cur] + carry_from, (size_t)carry, cudaMemcpyDeviceToDevice,
                                   c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->d_buf[nb] + carry, host_chunk, (size_t)nbytes, cudaMemcpyHostToDevice,
                                              c.stream);
    SB_TRY(cuda_result(e, who));
    t->cur = nb;
    t->buf_len = n;
    t->buf_off = file_offset - carry;
    t->next_offset += nbytes;
    if (n <= sbps::kTail) {                             // too short to measure a packet: all of it waits for more
        t->h_run->carry = 0;
        return cuda_result(cudaStreamSynchronize(c.stream), who);
    }
    // scan_buffer waits for the candidate count, so the chunk has been copied when it returns
    return scan_buffer(t, t->d_buf[nb], n, t->buf_off, false, who);
}

int sb_ps_finish(sb_ps* t, int32_t* cut, sb_pcm** out) {
    const char* who = "sb_ps_finish";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && cut && out));
    SB_TRY(t->finish_check(who));
    ReleaseDemux<sb_ps> release_demux{t};
    SB_TRY(t->settle(who));
    // what the last chunk left over, as the end of the file; fewer than 4 bytes cannot start a packet (a file cut
    // inside a start code)
    const int64_t carry_from = t->buf_len ? std::min<int64_t>(t->h_run->carry, t->buf_len) : 0;
    if (t->buf_len - carry_from >= 4) {
        SB_TRY(scan_buffer(t, t->d_buf[t->cur] + carry_from, t->buf_len - carry_from, t->buf_off + carry_from, true, who));
        SB_TRY(t->settle(who));
    }
    SB_TRY(t->check_failure(who, [](int k) { return k == sbps::kBadPesHeader ? "PES packet" : "program stream packet"; },
                            sbps::error_text));
    uint32_t was_cut = 0;
    SB_TRY(collect(cudaSuccess, &was_cut, t->d_cut, 1, who));
    const Run run = *t->h_run;
    if (run.pes < 1 || run.bytes < 1) SB_FAIL(SB_EINVAL, "stream 0x%x carries no PES payload", t->stream_id);
    std::vector<uint8_t> host((size_t)run.bytes + 1);
    std::vector<PesRec> tab((size_t)run.pes);
    // the elementary stream is put together on the device, so its zero tail (sb_decode.h) is written here
    cudaError_t e = cudaMemsetAsync(t->d_es + (run.bytes & ~(long long)3), 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(tab.data(), t->d_tab, sizeof(PesRec) * (size_t)run.pes,
                                              cudaMemcpyDeviceToHost, c.stream);
    SB_TRY(collect(e, host.data(), t->d_es, run.bytes, who));
    // messages name the PES holding a stream byte
    auto where = [&](int64_t b) { return file_offset_of(tab, b); };
    int32_t dropped = 0;
    SB_TRY(mp2_decode(host.data(), t->d_es, run.bytes, where, &dropped, out));
    *cut = was_cut || dropped;
    return SB_OK;
}

int sb_ps_destroy(sb_ps* t) { return destroy_demux(t); }

}  // extern "C"
