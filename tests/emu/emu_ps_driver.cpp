// CPU build of the program stream demuxer: sushi_b200/csrc/sb_ps.cuh compiled with g++, driven the way sb_ps.cu drives
// it (tests/test_ps_cases.py).  The file is fed in chunks; each buffer is the bytes carried from the chain position
// the previous chunk reached, then the chunk.  Per buffer: every start code below the limit (k_ps_mark / k_ps_cands),
// each candidate's link (k_ps_link), the chain marked by pointer jumping in rounds (k_ps_jump), then the chain's
// packets in order: its end (the next carry, or a refusal) and the chosen stream's PES payloads (k_ps_pes, k_ps_place,
// k_ps_copy).  The first failure by byte offset wins, as the atomicMin of the kernels makes it.
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "sb_ps.cuh"

namespace {

struct Demux {
    int stream_id;
    std::vector<uint8_t> es;
    std::vector<int64_t> pes_file;                   // file offset of each PES that carried payload
    uint64_t err = ~0ull;
    int cut = 0;
    void fail(int64_t off, int code) { const uint64_t v = ((uint64_t)off << 8) | (unsigned)code; if (v < err) err = v; }

    // buf[0, n) at file offset base; returns where the carry starts
    int64_t scan(const uint8_t* buf, int64_t n, int64_t base, bool at_end) {
        const int64_t limit = at_end ? n - 3 : n - sbps::kTail;
        std::vector<int64_t> pos;
        for (int64_t i = 0; i < limit; ++i)
            if (sbps::is_start(buf + i)) pos.push_back(i);
        const int64_t m = (int64_t)pos.size();
        auto find = [&](int64_t p) -> int64_t {
            auto it = std::lower_bound(pos.begin(), pos.end(), p);
            return it != pos.end() && *it == p ? it - pos.begin() : -1;
        };
        int64_t carry = n;
        if (m == 0 || pos[0] != 0) fail(base, sbps::kNoStartCode);
        std::vector<sbps::Link> links((size_t)m);
        std::vector<int64_t> jump((size_t)m + 1), next((size_t)m + 1);
        std::vector<uint8_t> on((size_t)m + 1, 0);
        for (int64_t k = 0; k < m; ++k) {
            links[k] = sbps::link(buf, pos[k], n, limit, at_end, [&](int64_t p) { return find(p) >= 0; });
            jump[k] = links[k].kind == sbps::kLink ? find(links[k].next) : m;
        }
        jump[m] = m;
        if (m) on[0] = pos[0] == 0;
        for (int r = 0; ((int64_t)1 << r) < m; ++r) {
            for (int64_t v = 0; v <= m; ++v) if (on[v]) on[jump[v]] = 1;
            for (int64_t v = 0; v <= m; ++v) next[v] = jump[jump[v]];
            jump.swap(next);
        }
        for (int64_t k = 0; k < m; ++k) {
            if (!on[k]) continue;
            const int64_t q = pos[k];
            const sbps::Link l = links[k];
            bool whole = true;
            if (l.kind == sbps::kBadHeader) { fail(base + q, sbps::kBadPack); whole = false; }
            else if (l.kind == sbps::kBroken) fail(base + l.next, sbps::kNoStartCode);
            else if (l.kind == sbps::kNext) carry = l.next;
            else if (l.kind == sbps::kPast) { whole = at_end; carry = at_end ? n : q; }
            if (!whole || buf[q + 3] != stream_id) continue;
            const sbps::Pes p = sbps::parse_pes(buf + q, n - q);
            if (p.code) { fail(base + q, p.code); continue; }
            if (p.cut) cut = 1;
            if (p.cut == 2 || p.payload_len <= 0) continue;
            pes_file.push_back(base + q);
            es.insert(es.end(), buf + q + p.payload_off, buf + q + p.payload_off + p.payload_len);
        }
        return carry;
    }
};

}  // namespace

extern "C" {

// Demux stream `stream_id` of the file buf[0, nbytes) fed in chunks of `chunk` bytes.  es (room for cap bytes)
// receives the elementary stream, pes (room for cap_pes) the file offset of each PES; info[0..1] = PES count, cut flag.
// Returns the byte count, or -1 with the message in msg.
int64_t emu_ps_demux(const uint8_t* buf, int64_t nbytes, int stream_id, int64_t chunk, uint8_t* es, int64_t cap,
                     int64_t* pes, int64_t cap_pes, int64_t* info, char* msg, int msg_len) {
    Demux d;
    d.stream_id = stream_id;
    std::vector<uint8_t> cur;
    int64_t cur_off = 0;
    for (int64_t at = 0; at < nbytes; at += chunk) {
        const int64_t n = std::min(chunk, nbytes - at);
        cur.insert(cur.end(), buf + at, buf + at + n);
        if ((int64_t)cur.size() <= sbps::kTail) continue;
        const int64_t carry = d.scan(cur.data(), (int64_t)cur.size(), cur_off, false);
        cur.erase(cur.begin(), cur.begin() + std::min<int64_t>(carry, (int64_t)cur.size()));
        cur_off += carry;
    }
    if (cur.size() >= 4) d.scan(cur.data(), (int64_t)cur.size(), cur_off, true);
    if (d.err != ~0ull) {
        const int k = (int)(d.err & 0xFF);
        snprintf(msg, msg_len, "%s at byte offset %lld: %s", k == sbps::kBadPesHeader ? "PES packet" : "program stream packet",
                 (long long)(d.err >> 8), sbps::error_text(k));
        return -1;
    }
    info[0] = (int64_t)d.pes_file.size();
    info[1] = d.cut;
    memcpy(es, d.es.data(), (size_t)std::min<int64_t>(cap, (int64_t)d.es.size()));
    memcpy(pes, d.pes_file.data(), sizeof(int64_t) * (size_t)std::min<int64_t>(cap_pes, (int64_t)d.pes_file.size()));
    return (int64_t)d.es.size();
}

}  // extern "C"
