// Ogg input: one Ogg FLAC stream demuxed on the GPU and decoded by the FLAC decoder of sb_flac.cu, the host only reading
// the file in large chunks (DESIGN.md section 4).  Pages have variable lengths and may straddle chunks: each chunk is
// scanned behind the bytes carried over from the one before, which start at the chain position the previous chunk
// reached.
//   sb_ogg_feed    one chunk: the carried bytes and the chunk side by side on the device, then
//                    k_ogg_mark     per 16 positions: the capture patterns there ("OggS"); per-CTA counts
//                    k_scan_totals  one CTA: exclusive scan of the counts, the candidate total (sb_demux.cuh)
//                    k_ogg_cands    the candidates' positions, in order
//                  (the candidate count comes back to size the launches), then
//                    k_ogg_link     one thread per candidate: its page's length and the candidate it links to (or how
//                                   the chain ends there)
//                    k_chain_jump   log2(candidates) rounds of pointer jumping from the chunk's first position
//                                   (sb_demux.cuh)
//                    k_ogg_crc      one warp per candidate on the chain: the page's CRC-32, 32 lane slices combined
//                    k_ogg_page     one thread per candidate on the chain: the chain's end (the next chunk's carry, or a
//                                   refusal), the first data page, the chosen stream's pages; per-CTA totals of pages,
//                                   body bytes and packet starts
//                    k_scan_totals  one CTA: their exclusive scan on top of the running totals
//                    k_ogg_place    a chained stream refused; each chosen page's body placed in the elementary stream,
//                                   its record and its packets' starts written
//                    k_ogg_copy     one warp per page: its body into the elementary-stream buffer
//                    k_ogg_check    one thread per chosen page: its sequence number and continuation flag against the
//                                   stream's page before it
//                  and returns; the running totals and the carry position come back before the next chunk is placed
//   sb_ogg_finish  the carried bytes as the file's end (a last page may be cut), then the packets after the headers,
//                  one FLAC frame each, through sb::flac_decode with the payload and the packet table left on the device;
//                  messages name the page holding the start of a frame's packet
// The per-page rules are in sb_ogg.cuh, shared with the CPU emulation of the tests.
#include "sb_demux.cuh"
#include "sb_ogg.cuh"
#include <climits>
#include <memory>
#include <new>

using namespace sb;

namespace {

constexpr int kPer = 16;                               // positions one k_ogg_mark thread checks

// the first three are scanned by k_scan_totals<3>: the chosen stream's pages, body bytes and packets so far.  carry:
// where the last chunk's carry starts; closed: where the stream's last complete packet ends; first_data: the file
// offset of the first page that does not begin a stream (LLONG_MAX before it)
struct Run { long long pages, bytes, packets, carry, closed, first_data; };
struct PageRec { int64_t file_off; uint32_t seq; int32_t flags; int32_t open; int32_t pad; };
// one candidate: its page's body in the buffer, and (k_ogg_place) its place in the elementary stream.  hdr 0: not a
// page of the chosen stream.  bos: a whole chain page that begins a stream
struct Sel { int64_t body_off, body, dst; int32_t hdr, starts, bos, pad; };

__device__ __forceinline__ unsigned capture_mask(const uint8_t* __restrict__ buf, int64_t i0, int64_t limit) {
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
        const int64_t i = i0 + k;
        if (i < limit && sbogg::is_capture(buf + i)) m |= 1u << k;
    }
    return m;
}

__global__ void __launch_bounds__(kThreads)
k_ogg_mark(const uint8_t* __restrict__ buf, int64_t limit, long long* __restrict__ cta) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kPer;
    long long total;
    block_exclusive(__popc(capture_mask(buf, i0, limit)), &total);
    if (threadIdx.x == 0) cta[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads)
k_ogg_cands(const uint8_t* __restrict__ buf, int64_t limit, const long long* __restrict__ cta,
            int64_t* __restrict__ pos) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kPer;
    unsigned m = capture_mask(buf, i0, limit);
    long long total;
    long long at = cta[blockIdx.x] + block_exclusive(__popc(m), &total);
    for (; m; m &= m - 1) pos[at++] = i0 + __ffs(m) - 1;
}

// node m is the sink every chain end links to; jump[] starts as the links
__global__ void __launch_bounds__(kThreads)
k_ogg_link(const uint8_t* __restrict__ buf, int64_t n, int64_t limit, int64_t file_off0, const int64_t* __restrict__ pos,
           int64_t m, sbogg::Link* __restrict__ links, int32_t* __restrict__ jump, uint8_t* __restrict__ on,
           Run* __restrict__ run, unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) {
        run->carry = n;                                 // unless the chain's end says otherwise (k_ogg_page)
        jump[m] = (int32_t)m;
        on[m] = 0;
        if (m == 0 || pos[0] != 0) fail_at(err, file_off0, sbogg::kNoCapture);
    }
    if (k >= m) return;
    const sbogg::Link l = sbogg::link(buf, pos[k], n, limit, [&](int64_t p) { return find_cand(pos, m, p) >= 0; });
    links[k] = l;
    jump[k] = (int32_t)(l.kind == sbogg::kLink ? find_cand(pos, m, l.next) : m);
    on[k] = k == 0 && pos[0] == 0;
}

__device__ __forceinline__ bool whole_page(const sbogg::Link& l) {
    return l.kind == sbogg::kLink || l.kind == sbogg::kNext || l.kind == sbogg::kBroken;
}

// one warp per candidate: a whole page on the chain has its CRC-32 checked.  Lane i takes the i-th of 32 slices; the
// slice CRCs are combined pairwise (sb_ogg.cuh crc_combine) in five rounds of shuffles.
__global__ void __launch_bounds__(kThreads)
k_ogg_crc(const uint8_t* __restrict__ buf, int64_t file_off0, const int64_t* __restrict__ pos, int64_t m,
          const sbogg::Link* __restrict__ links, const uint8_t* __restrict__ on, unsigned long long* __restrict__ err) {
    __shared__ uint32_t table[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) table[i] = sbogg::crc_entry(i);
    __syncthreads();
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (k >= m || !on[k]) return;
    const sbogg::Link l = links[k];
    if (!whole_page(l)) return;
    const int64_t q = pos[k], len = l.next - q;
    const uint8_t* page = buf + q;
    const int64_t slice = (len + 31) >> 5;
    const int64_t lo = min(len, lane * slice), hi = min(len, lo + slice);
    uint32_t c = sbogg::crc_range(page, lo, hi, table);
    int64_t span = hi - lo;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t c2 = __shfl_down_sync(0xFFFFFFFFu, c, o);
        const int64_t span2 = __shfl_down_sync(0xFFFFFFFFu, span, o);
        if ((lane & (2 * o - 1)) == 0) {
            c = sbogg::crc_combine(c, c2, span2);
            span += span2;
        }
    }
    if (lane == 0 && c != sbogg::stored_crc(page)) fail_at(err, file_off0 + q, sbogg::kBadCrc);
}

// one thread per candidate on the chain: the chain's end, the first data page, and the chosen stream's pages
__global__ void __launch_bounds__(kThreads)
k_ogg_page(const uint8_t* __restrict__ buf, int64_t n, int at_end, int64_t file_off0, uint32_t serial,
           const int64_t* __restrict__ pos, int64_t m, const sbogg::Link* __restrict__ links,
           const uint8_t* __restrict__ on, Sel* __restrict__ sel, long long* __restrict__ cta, Run* __restrict__ run,
           uint32_t* __restrict__ cut, unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Sel s{0, 0, 0, 0, 0, 0, 0};
    if (k < m && on[k]) {
        const int64_t q = pos[k];
        const sbogg::Link l = links[k];
        if (l.kind == sbogg::kBadHeader) fail_at(err, file_off0 + q, sbogg::kBadVersion);
        else if (l.kind == sbogg::kBroken) { fail_at(err, file_off0 + l.next, sbogg::kNoCapture); run->carry = n; }
        else if (l.kind == sbogg::kNext) {
            run->carry = l.next;
            if (at_end && l.next < n) atomicOr(cut, 1u);          // a file cut inside the next capture pattern
        } else if (l.kind == sbogg::kPast) {
            run->carry = at_end ? n : q;                          // carried to the next chunk, or cut by the file's end
            if (at_end) atomicOr(cut, 1u);
        }
        if (whole_page(l)) {
            const sbogg::Page p = sbogg::page_info(buf + q);
            if (p.flags & 2) s.bos = 1;
            else atomicMin(&run->first_data, (long long)(file_off0 + q));
            if (p.serial == serial) {
                s.hdr = p.hdr; s.body_off = q + p.hdr; s.body = p.body; s.starts = p.starts;
            }
        }
    }
    if (k < m) sel[k] = s;
    long long t0, t1, t2;
    block_exclusive(s.hdr > 0, &t0);
    block_exclusive(s.body, &t1);
    block_exclusive(s.starts, &t2);
    if (threadIdx.x == 0) { cta[3 * blockIdx.x] = t0; cta[3 * blockIdx.x + 1] = t1; cta[3 * blockIdx.x + 2] = t2; }
}

__global__ void __launch_bounds__(kThreads)
k_ogg_place(const uint8_t* __restrict__ buf, int64_t file_off0, const int64_t* __restrict__ pos, int64_t m,
            Sel* __restrict__ sel, const long long* __restrict__ cta, PageRec* __restrict__ tab,
            int64_t* __restrict__ pkt_es, int64_t* __restrict__ pkt_file, Run* __restrict__ run,
            unsigned long long* __restrict__ err) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Sel s{0, 0, 0, 0, 0, 0, 0};
    if (k < m) s = sel[k];
    long long t0, t1, t2;
    const long long ep = cta[3 * blockIdx.x] + block_exclusive(s.hdr > 0, &t0);
    const long long eb = cta[3 * blockIdx.x + 1] + block_exclusive(s.body, &t1);
    const long long ek = cta[3 * blockIdx.x + 2] + block_exclusive(s.starts, &t2);
    if (k >= m) return;
    const int64_t file_off = file_off0 + pos[k];
    if (s.bos && file_off > run->first_data) fail_at(err, file_off, sbogg::kChained);
    if (!s.hdr) return;
    const uint8_t* page = buf + pos[k];
    const sbogg::Page p = sbogg::page_info(page);
    tab[ep] = PageRec{file_off, p.seq, p.flags, p.open, 0};
    sel[k].dst = eb;
    sbogg::packet_starts(page, [&](int j, int64_t off) { pkt_es[ek + j] = eb + off; pkt_file[ek + j] = file_off; });
    if (p.closed >= 0) atomicMax(&run->closed, (long long)(eb + p.closed));
}

__global__ void __launch_bounds__(kThreads)
k_ogg_copy(const uint8_t* __restrict__ buf, int64_t m, const Sel* __restrict__ sel, uint8_t* __restrict__ es) {
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= m) return;
    const Sel s = sel[k];
    if (!s.hdr) return;
    for (int64_t b = threadIdx.x & 31; b < s.body; b += 32) es[s.dst + b] = buf[s.body_off + b];
}

// pages [first, run->pages) of the stream: page 0 begins the stream; every later one follows its predecessor
__global__ void __launch_bounds__(kThreads)
k_ogg_check(const PageRec* __restrict__ tab, int64_t first, const Run* __restrict__ run,
            unsigned long long* __restrict__ err) {
    const int64_t p = first + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= run->pages) return;
    const PageRec cur = tab[p];
    if (p == 0) {
        if (cur.flags & 1) fail_at(err, cur.file_off, sbogg::kBadContinuation);
        return;
    }
    const PageRec prev = tab[p - 1];
    if (cur.seq != prev.seq + 1u) fail_at(err, cur.file_off, sbogg::kSeqGap);
    else if ((cur.flags & 1) != prev.open) fail_at(err, cur.file_off, sbogg::kBadContinuation);
}

}  // namespace

struct sb_ogg : ChunkedDemux<Run> {
    uint32_t serial = 0;
    int channels = 0, bits = 0, rate = 0;
    int64_t header_packets = 0;
    uint8_t* d_buf[2] = {nullptr, nullptr}; int64_t buf_cap[2] = {0, 0};
    int cur = 0;                                        // the buffer the last chunk went to
    int64_t buf_len = 0, buf_off = 0;                   // its bytes, and the file offset of its first byte
    long long* d_cta = nullptr; int64_t cta_cap = 0;
    int64_t* d_pos = nullptr; int64_t pos_cap = 0;
    sbogg::Link* d_links = nullptr; int64_t links_cap = 0;
    int32_t* d_jump[2] = {nullptr, nullptr}; int64_t jump_cap[2] = {0, 0};
    uint8_t* d_on = nullptr; int64_t on_cap = 0;
    Sel* d_sel = nullptr; int64_t sel_cap = 0;
    uint8_t* d_es = nullptr; int64_t es_cap = 0;
    PageRec* d_tab = nullptr; int64_t tab_cap = 0;
    int64_t* d_pkt_es = nullptr; int64_t pkt_es_cap = 0;
    int64_t* d_pkt_file = nullptr; int64_t pkt_file_cap = 0;
    Run* d_run = nullptr;
    long long* d_count = nullptr;
    uint32_t* d_cut = nullptr;
    long long* h_count = nullptr;                       // pinned copy of *d_count; *h_run is that of *d_run
    bool short_tail = false;                            // the file ends inside a capture pattern

    ~sb_ogg() {
        release_demux();
        pool_free(d_run); pool_free(d_count); pool_free(d_cut);
        if (h_count) cudaFreeHost(h_count);
    }
    void release_demux() {
        for (int b = 0; b < 2; ++b) { pool_free(d_buf[b]); pool_free(d_jump[b]); d_buf[b] = nullptr; d_jump[b] = nullptr;
                                      buf_cap[b] = jump_cap[b] = 0; }
        pool_free(d_cta); pool_free(d_pos); pool_free(d_links); pool_free(d_on); pool_free(d_sel); pool_free(d_es);
        pool_free(d_tab); pool_free(d_pkt_es); pool_free(d_pkt_file);
        d_cta = nullptr; d_pos = nullptr; d_links = nullptr; d_on = nullptr; d_sel = nullptr; d_es = nullptr;
        d_tab = nullptr; d_pkt_es = nullptr; d_pkt_file = nullptr;
        cta_cap = pos_cap = links_cap = on_cap = sel_cap = es_cap = tab_cap = pkt_es_cap = pkt_file_cap = 0;
    }
};

namespace {

// Scan buf[0, n) of the current buffer (file offset base): the page chain from position 0, the stream's pages
// appended.  `at_end`: the buffer ends the file.  Returns once the kernels are enqueued (the candidate count having
// come back first).
int scan_buffer(sb_ogg* t, const uint8_t* buf, int64_t n, int64_t base, bool at_end, const char* who) {
    Ctx& c = ctx();
    const int64_t limit = n - 3;                                  // every candidate's 4 bytes lie inside
    const Run run = *t->h_run;
    const int64_t n_thr = (limit + kPer - 1) / kPer, n_cta = std::max<int64_t>(1, (n_thr + kThreads - 1) / kThreads);
    int rc = grow(&t->d_cta, &t->cta_cap, 0, 3 * n_cta + 3, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_pos, &t->pos_cap, 0, limit / 4 + 1, c.stream);
    if (rc != SB_OK) SB_FAIL(rc, "%s: out of device memory for a chunk of %lld bytes", who, (long long)n);
    cudaError_t e = cudaSuccess;
    {
        ProfScope ps("ogg_mark", 3);
        k_ogg_mark<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(buf, limit, t->d_cta);
        k_scan_totals<1><<<1, 1024, 0, c.stream>>>(t->d_cta, n_cta, nullptr, t->d_count);
        k_ogg_cands<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(buf, limit, t->d_cta, t->d_pos);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->h_count, t->d_count, sizeof(long long), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    const int64_t m = *t->h_count;
    const int64_t m_cta = std::max<int64_t>(1, (m + kThreads - 1) / kThreads);
    // the chunk's pages (sb_ogg.cuh max_pages); their packet starts are among their lacing values, which lie in the
    // chunk too, so there are fewer than n
    const int64_t max_pages = sbogg::max_pages(m, n);
    rc = grow(&t->d_links, &t->links_cap, 0, m + 1, c.stream);
    for (int b = 0; b < 2 && rc == SB_OK; ++b) rc = grow(&t->d_jump[b], &t->jump_cap[b], 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_on, &t->on_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_sel, &t->sel_cap, 0, m + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_cta, &t->cta_cap, 0, 3 * m_cta + 3, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_es, &t->es_cap, run.bytes, run.bytes + n, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_tab, &t->tab_cap, run.pages, run.pages + max_pages + 1, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_pkt_es, &t->pkt_es_cap, run.packets, run.packets + n + 1,
                               c.stream);
    if (rc == SB_OK) rc = grow(&t->d_pkt_file, &t->pkt_file_cap, run.packets,
                               run.packets + n + 1, c.stream);
    if (rc != SB_OK) SB_FAIL(rc, "%s: out of device memory for a chunk of %lld bytes", who, (long long)n);
    {
        ProfScope ps("ogg_chain");
        k_ogg_link<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, n, limit, base, t->d_pos, m, t->d_links,
                                                              t->d_jump[0], t->d_on, t->d_run, t->d_err);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = mark_chain(t->d_jump, t->d_on, m, "ogg_chain", c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("ogg_crc");
        k_ogg_crc<<<(unsigned)((m * 32 + kThreads - 1) / kThreads + 1), kThreads, 0, c.stream>>>(
            buf, base, t->d_pos, m, t->d_links, t->d_on, t->d_err);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("ogg_compact", 5);
        k_ogg_page<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, n, at_end, base, t->serial, t->d_pos, m, t->d_links,
                                                              t->d_on, t->d_sel, t->d_cta, t->d_run, t->d_cut, t->d_err);
        k_scan_totals<3><<<1, 1024, 0, c.stream>>>(t->d_cta, m_cta, reinterpret_cast<long long*>(t->d_run),
                                                  reinterpret_cast<long long*>(t->d_run));
        k_ogg_place<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(buf, base, t->d_pos, m, t->d_sel, t->d_cta, t->d_tab,
                                                               t->d_pkt_es, t->d_pkt_file, t->d_run, t->d_err);
        k_ogg_copy<<<(unsigned)((m * 32 + kThreads - 1) / kThreads + 1), kThreads, 0, c.stream>>>(buf, m, t->d_sel,
                                                                                                t->d_es);
        k_ogg_check<<<(unsigned)m_cta, kThreads, 0, c.stream>>>(t->d_tab, run.pages, t->d_run, t->d_err);
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

int sb_ogg_open(uint32_t serial, int32_t channels, int32_t bits, int32_t rate, int32_t header_packets, sb_ogg** out) {
    const char* who = "sb_ogg_open";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, out));
    if (bits != 16 && bits != 24) SB_FAIL(SB_EINVAL, "FLAC with %d bits per sample is not supported (16 or 24)", bits);
    if (channels < 1 || channels > 8 || rate < 1 || header_packets < 0)
        SB_FAIL(SB_EINVAL, "sb_ogg_open: bad stream parameters");
    std::unique_ptr<sb_ogg> t(new (std::nothrow) sb_ogg());
    if (!t) SB_FAIL(SB_ENOMEM, "sb_ogg_open: out of host memory");
    t->serial = serial; t->channels = channels; t->bits = bits; t->rate = rate; t->header_packets = header_packets;
    SB_TRY(t->open(who));
    SB_TRY(cuda_result(cudaMallocHost((void**)&t->h_count, sizeof(long long)), who));
    if (pool_alloc((void**)&t->d_run, sizeof(Run)) != SB_OK || pool_alloc((void**)&t->d_count, 16) != SB_OK ||
        pool_alloc((void**)&t->d_cut, 16) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_ogg_open: out of device memory");
    t->h_run->closed = 0;
    t->h_run->first_data = LLONG_MAX;
    cudaError_t e = cudaMemcpyAsync(t->d_run, t->h_run, sizeof(Run), cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(t->d_cut, 0, sizeof(uint32_t), c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    *out = t.release();
    return SB_OK;
}

int sb_ogg_feed(sb_ogg* t, const void* host_chunk, int64_t nbytes, int64_t file_offset) {
    const char* who = "sb_ogg_feed";
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
        SB_FAIL(SB_ENOMEM, "sb_ogg_feed: out of device memory for a chunk of %lld bytes", (long long)nbytes);
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
    if (n < sbogg::kHeader) {                           // too short to measure a page: all of it waits for more
        t->h_run->carry = 0;
        return cuda_result(cudaStreamSynchronize(c.stream), who);
    }
    // scan_buffer waits for the candidate count, so the chunk has been copied when it returns
    return scan_buffer(t, t->d_buf[nb], n, t->buf_off, false, who);
}

int sb_ogg_finish(sb_ogg* t, int32_t* cut, sb_pcm** out) {
    const char* who = "sb_ogg_finish";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && cut && out));
    SB_TRY(t->finish_check(who));
    ReleaseDemux<sb_ogg> release_demux{t};
    SB_TRY(t->settle(who));
    // what the last chunk left over, as the end of the file; fewer than 4 bytes cannot start a page (a file cut inside
    // a capture pattern)
    const int64_t carry_from = t->buf_len ? std::min<int64_t>(t->h_run->carry, t->buf_len) : 0;
    const int64_t left = t->buf_len - carry_from;
    if (left >= 4) {
        SB_TRY(scan_buffer(t, t->d_buf[t->cur] + carry_from, left, t->buf_off + carry_from, true, who));
        SB_TRY(t->settle(who));
    } else if (left > 0) {
        t->short_tail = true;
    }
    SB_TRY(t->check_failure(who, [](int) { return "Ogg page"; }, sbogg::error_text));
    uint32_t was_cut = 0;
    SB_TRY(collect(cudaSuccess, &was_cut, t->d_cut, 1, who));
    const Run run = *t->h_run;
    if (run.pages < 1) SB_FAIL(SB_EINVAL, "Ogg stream 0x%x has no pages", t->serial);
    // the packets that end before the stream's end: a last packet still open there is dropped
    std::vector<int64_t> pkt_es((size_t)run.packets), pkt_file((size_t)run.packets);
    cudaError_t e = cudaMemcpyAsync(pkt_es.data(), t->d_pkt_es, sizeof(int64_t) * (size_t)run.packets,
                                    cudaMemcpyDeviceToHost, c.stream);
    SB_TRY(collect(e, pkt_file.data(), t->d_pkt_file, run.packets, who));
    int64_t complete = run.packets;
    while (complete > 0 && pkt_es[(size_t)complete - 1] >= run.closed) --complete;
    const bool open_tail = complete < run.packets;
    // the mapping header and the metadata packets after it are not frames
    const int64_t skip = 1 + t->header_packets;
    if (complete < skip)
        SB_FAIL(SB_EINVAL, "Ogg stream 0x%x ends inside its header packets (%lld of %lld)", t->serial,
                (long long)complete, (long long)skip);
    const int64_t n = complete - skip;
    if (n < 1) SB_FAIL(SB_EINVAL, "Ogg stream 0x%x holds no FLAC frames", t->serial);
    // the zero tail sb_decode.h asks for, from the end of the last complete packet (the buffer has 16 bytes past its
    // capacity, grow)
    SB_TRY(cuda_result(cudaMemsetAsync(t->d_es + run.closed, 0, 16, c.stream), who));
    SB_TRY(flac_decode(t->d_es, run.closed, t->d_pkt_es + skip, pkt_es.data() + skip, pkt_file.data() + skip, n,
                       t->channels, t->bits, t->rate, out, who));
    *cut = was_cut || open_tail || t->short_tail;
    return SB_OK;
}

int sb_ogg_destroy(sb_ogg* t) { return destroy_demux(t); }

}  // extern "C"
