// CPU build of the transport stream demuxer: sushi_b200/csrc/sb_ts.cuh compiled with g++, driven the way sb_ts.cu
// drives it (tests/test_kernel_emulation_ts.py).  The file is fed in chunks of whole packets; each packet is parsed as
// k_ts_scan parses it, the PID's packets are appended to the payload buffer and the packet table as k_ts_scatter
// appends them, the continuity counter is checked against the packet before as k_ts_cc checks it (across chunks), and
// sb_ts_finish's steps follow: k_pes_index per PES, the frame offsets, k_bdlpcm_decode per frame.  The first failure by
// byte offset wins, as the atomicMin of the kernels makes it.
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "sb_ts.cuh"

namespace {

struct Rec { int64_t file_off, es_off; sbts::Packet q; };

struct Demux {
    int psize, pid;
    std::vector<uint8_t> es;
    std::vector<Rec> tab;
    std::vector<int64_t> pes;                       // index into tab of each PES start
    uint64_t err = ~0ull;
    void fail(int64_t off, int code) { const uint64_t v = ((uint64_t)off << 8) | (unsigned)code; if (v < err) err = v; }

    void feed(const uint8_t* chunk, int64_t n, int64_t file_off) {
        const int64_t first = (int64_t)tab.size();
        for (int64_t i = 0; i < n / psize; ++i) {
            int id;
            sbts::Packet q;
            const int code = sbts::parse_packet(chunk + i * psize + psize - sbts::kTsSize, pid, &id, &q);
            if (code) { fail(file_off + i * psize, code); continue; }
            if (id != pid) continue;
            if (q.pusi && q.payload_len > 0) pes.push_back((int64_t)tab.size());
            tab.push_back(Rec{file_off + i * psize, (int64_t)es.size(), q});
            const uint8_t* src = chunk + i * psize + psize - sbts::kTsSize + q.payload_off;
            es.insert(es.end(), src, src + q.payload_len);
        }
        for (int64_t j = first > 0 ? first : 1; j < (int64_t)tab.size(); ++j)
            if (!sbts::cc_ok(true, tab[j - 1].q.cc, tab[j].q)) fail(tab[j].file_off, sbts::kCcGap);
    }
};

}  // namespace

extern "C" {

// Demux and decode PID `pid` of the file `buf` fed in chunks of `chunk` bytes (whole packets).  codec 0: BD-LPCM, pcm
// receives frames x channels int16 (at most cap frames; NULL: count only), info[0..3] = channels, rate, bits, cut flag;
// codec 1: TrueHD, pcm receives the kept payload bytes (at most cap).  Returns the frame (byte) count, or -1 with the
// message in msg.
int64_t emu_ts_decode(const uint8_t* buf, int64_t nbytes, int psize, int pid, int codec, int64_t chunk, void* out,
                      int64_t cap, int32_t* info, char* msg, int msg_len) {
    Demux d;
    d.psize = psize; d.pid = pid;
    const int64_t whole = nbytes - nbytes % psize;
    chunk -= chunk % psize;
    for (int64_t at = 0; at < whole; at += chunk) d.feed(buf + at, std::min(chunk, whole - at), at);
    auto refuse = [&](uint64_t e) {
        const int k = (int)(e & 0xFF);
        snprintf(msg, msg_len, "%s at byte offset %lld: %s", k <= sbts::kCcGap ? "transport stream packet" : "PES packet",
                 (long long)(e >> 8), sbts::error_text(k));
        return (int64_t)-1;
    };
    if (d.err != ~0ull) return refuse(d.err);
    const int64_t n = (int64_t)d.pes.size();
    if (n < 1) { snprintf(msg, msg_len, "PID %d carries no PES packet", pid); return -1; }
    std::vector<int64_t> off(n), count(n, 0);
    uint32_t hdr0 = 0;
    int cut = 0;
    sbts::Lpcm f{};
    for (int64_t s = 0; s < n; ++s) {
        const int64_t b = d.tab[d.pes[s]].es_off, e = s + 1 < n ? d.tab[d.pes[s + 1]].es_off : (int64_t)d.es.size();
        const int64_t where = d.tab[d.pes[s]].file_off;
        const sbts::Pes p = sbts::parse_pes(d.es.data(), b, e, s + 1 == n);
        off[s] = p.payload_off;
        if (p.code) { d.fail(where, p.code); continue; }
        cut |= p.cut;
        if (p.cut == 2) continue;
        if (codec == 1) { count[s] = p.ext_id == 0x76 ? 0 : p.payload_len; continue; }
        if (p.payload_len < 4) { if (!p.cut) d.fail(where, sbts::kShortLpcm); continue; }
        const uint8_t* h = d.es.data() + p.payload_off;
        const uint32_t hdr = ((uint32_t)h[0] << 24) | (h[1] << 16) | (h[2] << 8) | h[3];
        if (s == 0) {
            hdr0 = hdr;
            const int bad = sbts::parse_lpcm(hdr0, &f);
            if (bad) { d.fail(where, bad); break; }
        } else if (sbts::lpcm_fields(hdr) != sbts::lpcm_fields(hdr0)) { d.fail(where, sbts::kLpcmChange); continue; }
        off[s] = p.payload_off + 4;
        count[s] = sbts::lpcm_frames(p.payload_len, f);
    }
    if (d.err != ~0ull) return refuse(d.err);
    int64_t total = 0;
    std::vector<int64_t> start(n);
    for (int64_t s = 0; s < n; ++s) { start[s] = total; total += count[s]; }
    info[3] = cut ? 1 : 0;
    if (codec == 1) {
        if (out)
            for (int64_t s = 0; s < n; ++s)
                if (start[s] < cap) memcpy((uint8_t*)out + start[s], d.es.data() + off[s], (size_t)std::min(count[s], cap - start[s]));
        return total;
    }
    info[0] = f.channels; info[1] = f.rate; info[2] = f.bits;
    if (out) {
        const int64_t fb = (int64_t)f.src_channels * f.width;
        for (int64_t fr = 0; fr < std::min(total, cap); ++fr) {
            int64_t lo = 0, hi = n;
            while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (start[mid] <= fr) lo = mid; else hi = mid; }
            sbts::lpcm_frame(d.es.data() + off[lo] + (fr - start[lo]) * fb, f, (int16_t*)out + fr * f.channels);
        }
    }
    return total;
}

}  // extern "C"
