// MPEG transport stream input: one audio PID demuxed and decoded on the GPU, the host only reading the file in large
// chunks (DESIGN.md section 4).
//   sb_ts_feed     one chunk of whole packets: copied to the device, then
//                    k_ts_scan      one thread per packet: the sync byte of every packet, the header and adaptation
//                                   field of the PID's packets; per-CTA totals of the PID's payload bytes, packets and
//                                   PES starts
//                    k_scan_totals  one CTA: exclusive scan of the CTA totals on top of the running totals (sb_demux.cuh)
//                    k_ts_scatter   the PID's payload bytes appended to the elementary-stream buffer, its packets to the
//                                   packet table, its payload-unit starts to the PES table
//                    k_ts_cc        one thread per appended packet: the continuity counter against the packet before
//                                   (the last one of the previous chunk included)
//                  and returns once the chunk is copied; the running totals come back before the next chunk is placed
//   sb_ts_finish   k_pes_index (one thread per PES: header, PES_packet_length, BD-LPCM header or TrueHD routing), an
//                  exclusive scan of each PES's sample frames (or kept bytes), then k_bdlpcm_decode (a grid-stride loop
//                  over sample frames into interleaved int16) or k_ts_gather + the TrueHD decoder of sb_truehd.cu, into
//                  an sb_pcm
// The per-packet and per-PES rules are in sb_ts.cuh, shared with the CPU emulation of the tests.
#include "sb_demux.cuh"
#include "sb_ts.cuh"
#include <memory>
#include <new>

using namespace sb;

namespace {

struct Totals { long long bytes, packets, pes; };    // the PID's payload bytes, packets and PES starts

struct PktRec {                                      // one packet of the PID
    int64_t file_off;                                // byte offset of the packet (its arrival time stamp for BDAV)
    int64_t es_off;                                  // where its payload starts in the elementary-stream buffer
    int32_t len;
    uint8_t pusi, cc, disc, has_payload;
};
struct PesStart { int64_t es_off, pkt; };

__device__ __forceinline__ Totals packet_counts(const sbts::Packet& q) {
    Totals t;
    const bool mine = q.payload_len >= 0;
    t.bytes = mine ? q.payload_len : 0;
    t.packets = mine;
    t.pes = mine && q.pusi && q.payload_len > 0;
    return t;
}

__global__ void __launch_bounds__(kThreads)
k_ts_scan(const uint8_t* __restrict__ chunk, int64_t n_pk, int psize, int pid, int64_t file_off0,
          sbts::Packet* __restrict__ info, Totals* __restrict__ cta, unsigned long long* __restrict__ err) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    sbts::Packet q;
    q.payload_len = -1;                                // not the PID's
    if (i < n_pk) {
        const uint8_t* p = chunk + i * psize + (psize - sbts::kTsSize);
        int id;
        sbts::Packet r;
        const int code = sbts::parse_packet(p, pid, &id, &r);
        if (code) fail_at(err, file_off0 + i * psize, code);
        else if (id == pid) q = r;
        info[i] = q;
    }
    const Totals v = packet_counts(q);
    Totals total;
    block_exclusive(v.bytes, &total.bytes);
    block_exclusive(v.packets, &total.packets);
    block_exclusive(v.pes, &total.pes);
    if (threadIdx.x == 0) cta[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads)
k_ts_scatter(const uint8_t* __restrict__ chunk, int64_t n_pk, int psize, int64_t file_off0,
             const sbts::Packet* __restrict__ info, const Totals* __restrict__ cta, uint8_t* __restrict__ es,
             PktRec* __restrict__ tab, PesStart* __restrict__ pes) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    sbts::Packet q;
    q.payload_len = -1;
    if (i < n_pk) q = info[i];
    Totals total;
    const Totals v = packet_counts(q);
    Totals at;
    at.bytes = block_exclusive(v.bytes, &total.bytes);
    at.packets = block_exclusive(v.packets, &total.packets);
    at.pes = block_exclusive(v.pes, &total.pes);
    if (!v.packets) return;
    const Totals base = cta[blockIdx.x];
    at.bytes += base.bytes; at.packets += base.packets; at.pes += base.pes;
    PktRec r;
    r.file_off = file_off0 + i * psize;
    r.es_off = at.bytes;
    r.len = q.payload_len;
    r.pusi = q.pusi; r.cc = q.cc; r.disc = q.disc; r.has_payload = q.has_payload;
    tab[at.packets] = r;
    if (v.pes) pes[at.pes] = PesStart{at.bytes, at.packets};
    const uint8_t* src = chunk + i * psize + (psize - sbts::kTsSize) + q.payload_off;
    for (int b = 0; b < q.payload_len; ++b) es[at.bytes + b] = src[b];
}

__global__ void __launch_bounds__(kThreads)
k_ts_cc(const PktRec* __restrict__ tab, int64_t first, const Totals* __restrict__ run,
        unsigned long long* __restrict__ err) {
    const int64_t j = first + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= run->packets || j == 0) return;
    const PktRec a = tab[j - 1], b = tab[j];
    sbts::Packet q;
    q.cc = b.cc; q.disc = b.disc; q.has_payload = b.has_payload;
    if (!sbts::cc_ok(true, a.cc, q)) fail_at(err, b.file_off, sbts::kCcGap);
}

// one thread per PES: its span, header and (LPCM) sample frames or (TrueHD) kept bytes
__global__ void __launch_bounds__(kThreads)
k_pes_index(const uint8_t* __restrict__ es, int64_t es_total, const PesStart* __restrict__ pes, int64_t n_pes,
            const PktRec* __restrict__ tab, int codec, int64_t* __restrict__ off, int64_t* __restrict__ count,
            uint32_t* __restrict__ misc, unsigned long long* __restrict__ err) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_pes) return;
    const int64_t b = pes[s].es_off, e = s + 1 < n_pes ? pes[s + 1].es_off : es_total;
    const int64_t where = tab[pes[s].pkt].file_off;
    const sbts::Pes p = sbts::parse_pes(es, b, e, s + 1 == n_pes);
    off[s] = p.payload_off;
    count[s] = 0;
    if (p.code) { fail_at(err, where, p.code); return; }
    if (p.cut) atomicOr(&misc[1], 1u);
    if (p.cut == 2) return;                            // cut inside its header: dropped
    if (codec == SB_TS_MP2) {
        count[s] = p.payload_len;
        return;
    }
    if (codec == SB_TS_TRUEHD) {
        count[s] = p.ext_id == 0x76 ? 0 : p.payload_len;
        return;
    }
    // every PES against the first one's BD-LPCM header
    const sbts::Pes p0 = sbts::parse_pes(es, pes[0].es_off, n_pes > 1 ? pes[1].es_off : es_total, n_pes == 1);
    if (p0.code || p0.payload_len < 4) return;         // PES 0's own thread reports it
    const uint8_t* h0 = es + p0.payload_off;
    const uint32_t hdr0 = ((uint32_t)h0[0] << 24) | (h0[1] << 16) | (h0[2] << 8) | h0[3];
    sbts::Lpcm f;
    const int bad = sbts::parse_lpcm(hdr0, &f);
    if (bad) { if (s == 0) fail_at(err, where, bad); return; }
    if (s == 0) misc[0] = hdr0;
    if (p.payload_len < 4) {
        if (!p.cut) fail_at(err, where, sbts::kShortLpcm);
        return;
    }
    const uint8_t* h = es + p.payload_off;
    const uint32_t hdr = ((uint32_t)h[0] << 24) | (h[1] << 16) | (h[2] << 8) | h[3];
    if (sbts::lpcm_fields(hdr) != sbts::lpcm_fields(hdr0)) { fail_at(err, where, sbts::kLpcmChange); return; }
    off[s] = p.payload_off + 4;
    count[s] = sbts::lpcm_frames(p.payload_len, f);
}

__global__ void __launch_bounds__(kThreads)
k_bdlpcm_decode(const uint8_t* __restrict__ es, const int64_t* __restrict__ off, const int64_t* __restrict__ start,
                int64_t n_pes, int64_t frames, sbts::Lpcm f, int16_t* __restrict__ pcm) {
    const int64_t frame_bytes = (int64_t)f.src_channels * f.width;
    for (int64_t fr = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; fr < frames; fr += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = n_pes;                    // the last PES starting at or before fr
        while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (start[mid] <= fr) lo = mid; else hi = mid; }
        sbts::lpcm_frame(es + off[lo] + (fr - start[lo]) * frame_bytes, f, pcm + fr * f.channels);
    }
}

// the kept TrueHD payload of each PES, back to back (one CTA per PES)
__global__ void __launch_bounds__(kThreads)
k_ts_gather(const uint8_t* __restrict__ es, const int64_t* __restrict__ off, const int64_t* __restrict__ len,
            const int64_t* __restrict__ start, uint8_t* __restrict__ out) {
    const int64_t s = blockIdx.x;
    const uint8_t* src = es + off[s];
    uint8_t* dst = out + start[s];
    for (int64_t b = threadIdx.x; b < len[s]; b += blockDim.x) dst[b] = src[b];
}

}  // namespace

struct sb_ts : ChunkedDemux<Totals> {
    int psize = 188, pid = 0, codec = 0;
    uint8_t* d_chunk = nullptr; int64_t chunk_cap = 0;
    sbts::Packet* d_info = nullptr; int64_t info_cap = 0;
    Totals* d_cta = nullptr; int64_t cta_cap = 0;
    uint8_t* d_es = nullptr; int64_t es_cap = 0;
    PktRec* d_tab = nullptr; int64_t tab_cap = 0;
    PesStart* d_pes = nullptr; int64_t pes_cap = 0;
    Totals* d_run = nullptr;                            // after the last chunk; *h_run is its pinned copy
    cudaEvent_t copied = nullptr;

    ~sb_ts() {
        release_demux();
        pool_free(d_run);
        if (copied) cudaEventDestroy(copied);
    }
    void release_demux() {
        pool_free(d_chunk); pool_free(d_info); pool_free(d_cta); pool_free(d_es); pool_free(d_tab); pool_free(d_pes);
        d_chunk = nullptr; d_info = nullptr; d_cta = nullptr; d_es = nullptr; d_tab = nullptr; d_pes = nullptr;
        chunk_cap = info_cap = cta_cap = es_cap = tab_cap = pes_cap = 0;
    }
};

extern "C" {

int sb_ts_open(int packet_size, int32_t pid, int32_t codec, sb_ts** out) {
    const char* who = "sb_ts_open";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, out));
    if (packet_size != 188 && packet_size != 192) SB_FAIL(SB_EINVAL, "sb_ts_open: packet size %d (188 or 192)", packet_size);
    if (pid < 0 || pid > 0x1FFE) SB_FAIL(SB_EINVAL, "sb_ts_open: PID %d", pid);
    if (codec != SB_TS_PCM_BLURAY && codec != SB_TS_TRUEHD && codec != SB_TS_MP2) SB_FAIL(SB_EINVAL, "sb_ts_open: codec %d", codec);
    std::unique_ptr<sb_ts> t(new (std::nothrow) sb_ts());
    if (!t) SB_FAIL(SB_ENOMEM, "sb_ts_open: out of host memory");
    t->psize = packet_size; t->pid = pid; t->codec = codec;
    SB_TRY(t->open(who));
    SB_TRY(cuda_result(cudaEventCreateWithFlags(&t->copied, cudaEventDisableTiming), who));
    if (pool_alloc((void**)&t->d_run, sizeof(Totals)) != SB_OK) SB_FAIL(SB_ENOMEM, "sb_ts_open: out of device memory");
    SB_TRY(cuda_result(cudaMemsetAsync(t->d_run, 0, sizeof(Totals), c.stream), who));
    *out = t.release();
    return SB_OK;
}

int sb_ts_feed(sb_ts* t, const void* host_chunk, int64_t nbytes, int64_t file_offset) {
    const char* who = "sb_ts_feed";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && (host_chunk || !nbytes)));
    SB_TRY(t->feed_check(who, nbytes, file_offset, t->psize));
    if (!nbytes) return SB_OK;
    const int64_t n_pk = nbytes / t->psize, n_cta = (n_pk + kThreads - 1) / kThreads;
    // the totals after the previous chunk: they place this one
    SB_TRY(t->settle(who));
    const Totals run = *t->h_run;
    int rc = grow(&t->d_chunk, &t->chunk_cap, 0, nbytes, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_info, &t->info_cap, 0, n_pk, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_cta, &t->cta_cap, 0, n_cta, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_es, &t->es_cap, run.bytes, run.bytes + n_pk * sbts::kMaxPayload, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_tab, &t->tab_cap, run.packets, run.packets + n_pk, c.stream);
    if (rc == SB_OK) rc = grow(&t->d_pes, &t->pes_cap, run.pes, run.pes + n_pk, c.stream);
    if (rc != SB_OK) SB_FAIL(rc, "sb_ts_feed: out of device memory for a chunk of %lld bytes", (long long)nbytes);
    cudaError_t e = cudaMemcpyAsync(t->d_chunk, host_chunk, (size_t)nbytes, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaEventRecord(t->copied, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("ts_scan");
        k_ts_scan<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(t->d_chunk, n_pk, t->psize, t->pid, file_offset, t->d_info,
                                                              t->d_cta, t->d_err);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("ts_compact", 2);
        long long* run_d = reinterpret_cast<long long*>(t->d_run);
        k_scan_totals<3><<<1, 1024, 0, c.stream>>>(reinterpret_cast<long long*>(t->d_cta), n_cta, run_d, run_d);
        k_ts_scatter<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(t->d_chunk, n_pk, t->psize, file_offset, t->d_info,
                                                                 t->d_cta, t->d_es, t->d_tab, t->d_pes);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ProfScope ps("ts_scan");
        k_ts_cc<<<(unsigned)n_cta, kThreads, 0, c.stream>>>(t->d_tab, run.packets, t->d_run, t->d_err);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(t->h_run, t->d_run, sizeof(Totals), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaEventRecord(t->done, c.stream);
    SB_TRY(cuda_result(e, who));
    t->pending = true;
    t->next_offset += nbytes;
    // the caller may refill its buffer once the copy has run; the kernels go on behind it
    return cuda_result(cudaEventSynchronize(t->copied), who);
}

int sb_ts_finish(sb_ts* t, int32_t* cut, sb_pcm** out) {
    const char* who = "sb_ts_finish";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, t && cut && out));
    SB_TRY(t->finish_check(who));
    // the demultiplexer's buffers go when this returns, on whichever line: after truehd_index_device, whose `where`
    // reads t->d_tab when it words a message
    ReleaseDemux<sb_ts> release_demux{t};
    auto noun = [](int k) { return k <= sbts::kCcGap ? "transport stream packet" : "PES packet"; };
    SB_TRY(t->check_failure(who, noun, sbts::error_text));
    const Totals run = *t->h_run;
    if (run.pes < 1) SB_FAIL(SB_EINVAL, "PID %d carries no PES packet", t->pid);
    const int64_t n_pes = run.pes;
    Blocks blocks;
    int64_t* d_off = nullptr;
    int64_t* d_count = nullptr;
    uint32_t* d_misc = nullptr;
    if (blocks.alloc(&d_off, (size_t)n_pes) != SB_OK || blocks.alloc(&d_count, (size_t)n_pes) != SB_OK ||
        blocks.alloc(&d_misc, 4) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_ts_finish: out of device memory");
    uint32_t misc[2] = {0, 0};                          // the first BD-LPCM header, the cut flag
    cudaError_t e = cudaMemsetAsync(d_misc, 0, 16, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("pes_index");
        k_pes_index<<<(unsigned)((n_pes + kThreads - 1) / kThreads), kThreads, 0, c.stream>>>(
            t->d_es, run.bytes, t->d_pes, n_pes, t->d_tab, t->codec, d_off, d_count, d_misc, t->d_err);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, misc, d_misc, 2, who));
    SB_TRY(t->check_failure(who, noun, sbts::error_text));
    // per PES: the first sample frame (LPCM) or the first byte of the TrueHD stream (TrueHD)
    int64_t total = 0;
    SB_TRY(scan_i64(d_count, n_pes, &total, "pes_index", who));
    *cut = misc[1] ? 1 : 0;
    if (t->codec == SB_TS_PCM_BLURAY) {
        sbts::Lpcm f;
        if (sbts::parse_lpcm(misc[0], &f)) SB_FAIL(SB_EINVAL, "PID %d: no BD-LPCM header", t->pid);
        int16_t* d_pcm = nullptr;
        if (total > 0 && blocks.alloc(&d_pcm, (size_t)(total * f.channels)) != SB_OK)
            SB_FAIL(SB_ENOMEM, "sb_ts_finish: out of device memory for %lld sample frames", (long long)total);
        if (total > 0) {
            ProfScope ps("bdlpcm_decode");
            const int grid = (int)std::min<int64_t>((total + kThreads - 1) / kThreads, (int64_t)c.sm_count * 16);
            // the scan left each PES's first frame in d_count
            k_bdlpcm_decode<<<grid, kThreads, 0, c.stream>>>(t->d_es, d_off, d_count, n_pes, total, f, d_pcm);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        SB_TRY(cuda_result(e, who));
        return pcm_handle(blocks.take(d_pcm), total, f.channels, f.rate, out);
    }
    // TrueHD and MP2: the kept payloads back to back, then the decoder on them as one stream
    if (total < 1) SB_FAIL(SB_EINVAL, "PID %d carries no %s payload", t->pid, t->codec == SB_TS_MP2 ? "MP2" : "TrueHD");
    uint8_t* d_thd = nullptr;
    int64_t* d_len = nullptr;
    int64_t* d_block = nullptr;
    if (blocks.alloc(&d_thd, (size_t)total) != SB_OK || blocks.alloc(&d_len, (size_t)n_pes) != SB_OK ||
        blocks.alloc(&d_block, 2) != SB_OK)
        SB_FAIL(SB_ENOMEM, "sb_ts_finish: out of device memory for %lld bytes of TrueHD", (long long)total);
    std::vector<int64_t> start((size_t)n_pes), off((size_t)n_pes);
    std::vector<uint8_t> host((size_t)total + 1);
    // the lengths again (the scan replaced them by the starts): the difference of consecutive starts
    e = cudaMemcpyAsync(start.data(), d_count, sizeof(int64_t) * (size_t)n_pes, cudaMemcpyDeviceToHost, c.stream);
    SB_TRY(collect(e, off.data(), d_off, n_pes, who));
    std::vector<int64_t> len((size_t)n_pes);
    for (int64_t s = 0; s < n_pes; ++s) len[(size_t)s] = (s + 1 < n_pes ? start[(size_t)s + 1] : total) - start[(size_t)s];
    e = cudaMemcpyAsync(d_len, len.data(), sizeof(int64_t) * (size_t)n_pes, cudaMemcpyHostToDevice, c.stream);
    // the payload is put together on the device, so its zero tail (sb_decode.h) is written here
    if (e == cudaSuccess) e = cudaMemsetAsync(d_thd + (total & ~(int64_t)3), 0, 16, c.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_block, 0, 16, c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("ts_compact");
        k_ts_gather<<<(unsigned)n_pes, kThreads, 0, c.stream>>>(t->d_es, d_off, d_len, d_count, d_thd);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, host.data(), d_thd, total, who));
    // messages name the TS packet holding a TrueHD byte: its PES, its place in the PID's payload, then the packet table
    // (read back only when a message needs it)
    std::vector<PktRec> tab;
    auto where = [&](int64_t b) -> int64_t {
        int64_t s = std::upper_bound(start.begin(), start.end(), b) - start.begin() - 1;
        while (s > 0 && len[(size_t)s] == 0) --s;
        if (s < 0) return -1;
        const int64_t es = off[(size_t)s] + (b - start[(size_t)s]);
        if (tab.empty()) {
            tab.resize((size_t)run.packets);
            if (cudaMemcpy(tab.data(), t->d_tab, sizeof(PktRec) * (size_t)run.packets, cudaMemcpyDeviceToHost) != cudaSuccess)
                return -1;
        }
        return file_offset_of(tab, es);
    };
    if (t->codec == SB_TS_MP2) {
        int32_t dropped = 0;
        SB_TRY(mp2_decode(host.data(), d_thd, total, where, &dropped, out));
        *cut = *cut || dropped;
        return SB_OK;
    }
    const int64_t zero = 0;
    return truehd_index_device(host.data(), d_thd, total, &zero, d_block, 1, where, out);
}

int sb_ts_destroy(sb_ts* t) { return destroy_demux(t); }

}  // extern "C"
