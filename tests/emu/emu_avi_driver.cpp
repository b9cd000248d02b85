// CPU build of the AVI demuxer: sushi_b200/csrc/sb_avi.cuh compiled with g++, driven the way sb_avi.cu drives it
// (tests/test_kernel_emulation_avi.py).  The file is fed in chunks; each buffer holds the bytes from the chain position
// the previous one reached (a file offset, which may lie past the bytes fed so far: those are then skipped), then the
// chunk; a buffer short of the end of a chunk of the stream waits for more.  Per buffer: every chunk header below the limit (k_avi_mark / k_avi_cands), each candidate's link
// (k_avi_link), the chain marked by pointer jumping in rounds, then the chain's chunks in order: its end (the next
// chain position, or a refusal) and the chosen stream's payloads (k_avi_sel, k_avi_place, k_avi_copy).  The first
// failure by byte offset wins, as the atomicMin of the kernels makes it.
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "sb_avi.cuh"

namespace {

struct Demux {
    uint32_t tag;
    int64_t frame_bytes;                              // PCM: bytes of one sample frame; 0: any chunk size
    std::vector<int64_t> ext;
    std::vector<uint8_t> es;
    std::vector<int64_t> chunk_file;                  // file offset of each chunk that carried payload
    uint64_t err = ~0ull;
    int cut = 0;
    int64_t need = 0;                                 // the file offset the buffer must reach before the next scan
    void fail(int64_t off, int code) { const uint64_t v = ((uint64_t)off << 8) | (unsigned)code; if (v < err) err = v; }

    // buf[0, n) at file offset base; returns the chain position (a file offset) the next buffer starts at
    int64_t scan(const uint8_t* buf, int64_t n, int64_t base, bool at_end) {
        const int64_t limit = at_end ? n : n - sbavi::kTail;
        std::vector<int64_t> pos;
        for (int64_t i = 0; i < limit; ++i)
            if (sbavi::is_chunk(buf + i, n - i)) pos.push_back(i);
        const int64_t m = (int64_t)pos.size();
        auto find = [&](int64_t p) -> int64_t {
            auto it = std::lower_bound(pos.begin(), pos.end(), p);
            return it != pos.end() && *it == p ? it - pos.begin() : -1;
        };
        int64_t carry = base + n;
        need = 0;
        if (m == 0 || pos[0] != 0) fail(base, sbavi::kNoChunk);
        std::vector<sbavi::Link> links((size_t)m);
        std::vector<int64_t> jump((size_t)m + 1), next((size_t)m + 1);
        std::vector<uint8_t> on((size_t)m + 1, 0);
        const int64_t n_ext = (int64_t)ext.size() / 2;
        for (int64_t k = 0; k < m; ++k) {
            links[k] = sbavi::link(buf, pos[k], n, limit, at_end, base, ext.data(), n_ext, tag,
                                   [&](int64_t p) { return find(p) >= 0; });
            jump[k] = links[k].kind == sbavi::kLink ? find(links[k].next) : m;
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
            const sbavi::Link l = links[k];
            bool whole = true;
            if (l.kind == sbavi::kOverrun) { fail(base + q, sbavi::kPastList); continue; }
            if (l.kind == sbavi::kBroken) fail(base + l.next, sbavi::kNoChunk);
            else if (l.kind == sbavi::kNext) carry = l.next == sbavi::kDone ? sbavi::kDone : base + l.next;
            else if (l.kind == sbavi::kPast) {
                whole = at_end;
                carry = at_end ? base + n : base + q;
                if (!at_end) need = base + q + 8 + l.size;
            }
            if (!whole || sbavi::rd32(buf + q) != tag) continue;
            if (frame_bytes && l.size % frame_bytes) { fail(base + q, sbavi::kPartialFrame); continue; }
            const int64_t len = std::min<int64_t>(l.size, n - q - 8);
            if (len < l.size) cut = 1;
            if (len <= 0) continue;
            chunk_file.push_back(base + q);
            es.insert(es.end(), buf + q + 8, buf + q + 8 + len);
        }
        return carry;
    }
};

}  // namespace

extern "C" {

// Demux the chunks with FOURCC `tag` of the file buf[0, nbytes) fed in chunks of `chunk` bytes, ext[0, 2 n_ext) the
// movi extents; PCM chunks must hold whole frames of frame_bytes (0: any size).  es (room for cap bytes) receives the
// stream, offs (room for cap_offs) the file offset of each chunk; info[0..1] = chunk count, cut flag.  Returns the byte
// count, or -1 with the message in msg.
int64_t emu_avi_demux(const uint8_t* buf, int64_t nbytes, uint32_t tag, int64_t frame_bytes, const int64_t* ext,
                      int64_t n_ext, int64_t chunk, uint8_t* es, int64_t cap, int64_t* offs, int64_t cap_offs,
                      int64_t* info, char* msg, int msg_len) {
    Demux d;
    d.tag = tag;
    d.frame_bytes = frame_bytes;
    d.ext.assign(ext, ext + 2 * n_ext);
    std::vector<uint8_t> cur;
    int64_t cur_off = 0, carry = n_ext ? ext[0] : sbavi::kDone;
    for (int64_t at = 0; at < nbytes && carry != sbavi::kDone; at += chunk) {
        const int64_t n = std::min(chunk, nbytes - at);
        if (carry >= at) {                            // the bytes before the chain position are skipped
            cur.clear();
            if (carry < at + n) cur.insert(cur.end(), buf + carry, buf + at + n);
        } else {
            cur.erase(cur.begin(), cur.begin() + (carry - cur_off));
            cur.insert(cur.end(), buf + at, buf + at + n);
        }
        cur_off = carry;
        if ((int64_t)cur.size() <= sbavi::kTail || cur_off + (int64_t)cur.size() < d.need) continue;
        carry = d.scan(cur.data(), (int64_t)cur.size(), cur_off, false);
    }
    if (carry != sbavi::kDone) {
        const int64_t rem = nbytes - carry;
        if (rem >= sbavi::kHeader) {
            carry = d.scan(buf + carry, rem, carry, true);
            if (carry != sbavi::kDone) d.cut = 1;
        } else {
            d.cut = 1;
        }
    }
    if (d.err != ~0ull) {
        const int k = (int)(d.err & 0xFF);
        snprintf(msg, msg_len, "AVI chunk at byte offset %lld: %s", (long long)(d.err >> 8), sbavi::error_text(k));
        return -1;
    }
    info[0] = (int64_t)d.chunk_file.size();
    info[1] = d.cut;
    memcpy(es, d.es.data(), (size_t)std::min<int64_t>(cap, (int64_t)d.es.size()));
    memcpy(offs, d.chunk_file.data(), sizeof(int64_t) * (size_t)std::min<int64_t>(cap_offs, (int64_t)d.chunk_file.size()));
    return (int64_t)d.es.size();
}

}  // extern "C"
