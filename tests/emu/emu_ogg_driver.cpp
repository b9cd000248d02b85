// CPU build of the Ogg demuxer: sushi_b200/csrc/sb_ogg.cuh compiled with g++, driven the way sb_ogg.cu drives it
// (tests/test_ogg_cases.py).  The file is fed in chunks; each buffer is the bytes carried from the chain position the
// previous chunk reached, then the chunk.  Per buffer: every capture pattern below the limit (k_ogg_mark /
// k_ogg_cands), each candidate's link (k_ogg_link), the chain marked by pointer jumping in rounds (k_chain_jump), each
// chain page's CRC-32 from 32 slices combined as the lanes of k_ogg_crc combine them, then the chain's pages in order:
// its end (the next carry, or a refusal), the first data page, a chained stream, the chosen stream's pages placed,
// checked against the page before and their packet starts listed (k_ogg_page, k_ogg_place, k_ogg_copy, k_ogg_check).
// The first failure by byte offset wins, as the atomicMin of the kernels makes it.
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "sb_ogg.cuh"

namespace {

uint32_t g_table[256];

// the page's CRC as k_ogg_crc computes it: 32 slices, combined in five pairwise rounds
uint32_t warp_crc(const uint8_t* page, int64_t len) {
    uint32_t c[32];
    int64_t span[32];
    const int64_t slice = (len + 31) >> 5;
    for (int lane = 0; lane < 32; ++lane) {
        const int64_t lo = std::min(len, lane * slice), hi = std::min(len, lo + slice);
        c[lane] = sbogg::crc_range(page, lo, hi, g_table);
        span[lane] = hi - lo;
    }
    for (int o = 1; o < 32; o <<= 1)
        for (int lane = 0; lane + o < 32; lane += 2 * o) {
            c[lane] = sbogg::crc_combine(c[lane], c[lane + o], span[lane + o]);
            span[lane] += span[lane + o];
        }
    return c[0];
}

struct PageRec { int64_t file_off; uint32_t seq; int flags, open; };

struct Demux {
    uint32_t serial;
    std::vector<uint8_t> es;
    std::vector<int64_t> pkt_es, pkt_file;
    std::vector<PageRec> tab;
    int64_t closed = 0, first_data = LLONG_MAX;
    uint64_t err = ~0ull;
    int cut = 0;
    int table_overflow = 0;                          // a buffer held more pages or packets than the tables take
    void fail(int64_t off, int code) { const uint64_t v = ((uint64_t)off << 8) | (unsigned)code; if (v < err) err = v; }

    // buf[0, n) at file offset base; returns where the carry starts
    int64_t scan(const uint8_t* buf, int64_t n, int64_t base, bool at_end) {
        const int64_t limit = n - 3;
        std::vector<int64_t> pos;
        for (int64_t i = 0; i < limit; ++i)
            if (sbogg::is_capture(buf + i)) pos.push_back(i);
        const int64_t m = (int64_t)pos.size();
        auto find = [&](int64_t p) -> int64_t {
            auto it = std::lower_bound(pos.begin(), pos.end(), p);
            return it != pos.end() && *it == p ? it - pos.begin() : -1;
        };
        int64_t carry = n;
        if (m == 0 || pos[0] != 0) fail(base, sbogg::kNoCapture);
        std::vector<sbogg::Link> links((size_t)m);
        std::vector<int64_t> jump((size_t)m + 1), next((size_t)m + 1);
        std::vector<uint8_t> on((size_t)m + 1, 0);
        for (int64_t k = 0; k < m; ++k) {
            links[k] = sbogg::link(buf, pos[k], n, limit, [&](int64_t p) { return find(p) >= 0; });
            jump[k] = links[k].kind == sbogg::kLink ? find(links[k].next) : m;
        }
        jump[m] = m;
        if (m) on[0] = pos[0] == 0;
        for (int r = 0; ((int64_t)1 << r) < m; ++r) {
            for (int64_t v = 0; v <= m; ++v) if (on[v]) on[jump[v]] = 1;
            for (int64_t v = 0; v <= m; ++v) next[v] = jump[jump[v]];
            jump.swap(next);
        }
        std::vector<int64_t> chosen, bos;
        for (int64_t k = 0; k < m; ++k) {
            if (!on[k]) continue;
            const int64_t q = pos[k];
            const sbogg::Link l = links[k];
            if (l.kind == sbogg::kBadHeader) { fail(base + q, sbogg::kBadVersion); continue; }
            if (l.kind == sbogg::kBroken) { fail(base + l.next, sbogg::kNoCapture); carry = n; }
            else if (l.kind == sbogg::kNext) { carry = l.next; if (at_end && l.next < n) cut = 1; }
            else if (l.kind == sbogg::kPast) { carry = at_end ? n : q; if (at_end) cut = 1; continue; }
            if (warp_crc(buf + q, l.next - q) != sbogg::stored_crc(buf + q)) fail(base + q, sbogg::kBadCrc);
            const sbogg::Page p = sbogg::page_info(buf + q);
            if (p.flags & 2) bos.push_back(base + q);
            else first_data = std::min(first_data, base + q);
            if (p.serial == serial) chosen.push_back(q);
        }
        // the device's page and packet tables are sized by these bounds
        int64_t starts = 0;
        for (int64_t q : chosen) starts += sbogg::page_info(buf + q).starts;
        if ((int64_t)chosen.size() > sbogg::max_pages(m, n) || starts > n) table_overflow = 1;
        for (int64_t b : bos)
            if (b > first_data) fail(b, sbogg::kChained);
        for (int64_t q : chosen) {
            const sbogg::Page p = sbogg::page_info(buf + q);
            const int64_t eb = (int64_t)es.size();
            const PageRec cur{base + q, p.seq, p.flags, p.open};
            if (tab.empty()) {
                if (cur.flags & 1) fail(cur.file_off, sbogg::kBadContinuation);
            } else if (cur.seq != tab.back().seq + 1u) {
                fail(cur.file_off, sbogg::kSeqGap);
            } else if ((cur.flags & 1) != tab.back().open) {
                fail(cur.file_off, sbogg::kBadContinuation);
            }
            tab.push_back(cur);
            sbogg::packet_starts(buf + q, [&](int, int64_t off) { pkt_es.push_back(eb + off); pkt_file.push_back(base + q); });
            es.insert(es.end(), buf + q + p.hdr, buf + q + p.hdr + p.body);
            if (p.closed >= 0) closed = std::max(closed, eb + p.closed);
        }
        return carry;
    }
};

}  // namespace

extern "C" {

// the CRC of one page as the kernel computes it
uint32_t emu_ogg_crc(const uint8_t* page, int64_t len) {
    for (uint32_t i = 0; i < 256; ++i) g_table[i] = sbogg::crc_entry(i);
    return warp_crc(page, len);
}

// Demux the stream with serial number `serial` of the file buf[0, nbytes) fed in chunks of `chunk` bytes.  es (room
// for cap bytes) receives the pages' bodies; starts and files (room for cap_pkt each) each packet's start in es and
// the file offset of the page where it starts; info[0..2] = packets, the end of the last complete packet, cut flag.
// Returns the byte count, or -1 with the message in msg.
int64_t emu_ogg_demux(const uint8_t* buf, int64_t nbytes, uint32_t serial, int64_t chunk, uint8_t* es, int64_t cap,
                      int64_t* starts, int64_t* files, int64_t cap_pkt, int64_t* info, char* msg, int msg_len) {
    for (uint32_t i = 0; i < 256; ++i) g_table[i] = sbogg::crc_entry(i);
    Demux d;
    d.serial = serial;
    std::vector<uint8_t> cur;
    int64_t cur_off = 0;
    for (int64_t at = 0; at < nbytes; at += chunk) {
        const int64_t n = std::min(chunk, nbytes - at);
        cur.insert(cur.end(), buf + at, buf + at + n);
        if ((int64_t)cur.size() < sbogg::kHeader) continue;
        const int64_t carry = d.scan(cur.data(), (int64_t)cur.size(), cur_off, false);
        cur.erase(cur.begin(), cur.begin() + std::min<int64_t>(carry, (int64_t)cur.size()));
        cur_off += carry;
    }
    if (cur.size() >= 4) d.scan(cur.data(), (int64_t)cur.size(), cur_off, true);
    else if (!cur.empty()) d.cut = 1;
    if (d.table_overflow) {
        snprintf(msg, msg_len, "a buffer holds more pages or packet starts than sb_ogg.cu's tables are sized for");
        return -1;
    }
    if (d.err != ~0ull) {
        const int k = (int)(d.err & 0xFF);
        snprintf(msg, msg_len, "Ogg page at byte offset %lld: %s", (long long)(d.err >> 8), sbogg::error_text(k));
        return -1;
    }
    info[0] = (int64_t)d.pkt_es.size();
    info[1] = d.closed;
    info[2] = d.cut;
    memcpy(es, d.es.data(), (size_t)std::min<int64_t>(cap, (int64_t)d.es.size()));
    const size_t np = (size_t)std::min<int64_t>(cap_pkt, (int64_t)d.pkt_es.size());
    memcpy(starts, d.pkt_es.data(), sizeof(int64_t) * np);
    memcpy(files, d.pkt_file.data(), sizeof(int64_t) * np);
    return (int64_t)d.es.size();
}

}  // extern "C"
