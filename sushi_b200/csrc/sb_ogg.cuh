// Ogg page demuxing, written once for the GPU kernels of sb_ogg.cu and for the CPU (tests/emu/emu_ogg_driver.cpp
// compiles this header with g++).  Everything here is a __host__ __device__ function of plain integers and byte
// pointers: which bytes start a page, how long each page is, how one page links to the next on the chain, the page
// CRC-32 and how two CRCs of adjacent byte ranges combine, and where a page's packets start.
//
// An Ogg file is a chain of pages (RFC 3533): the capture pattern "OggS", version 0, the header type flags
// (1 continued packet, 2 first page of a stream, 4 last page), the 64-bit granule position, the stream serial number,
// the page sequence number, the CRC-32 and the segment count, 27 bytes in all, then that many lacing values and the
// body they measure.  A packet is the concatenation of lacing values of 255 up to and including the first one below
// 255; it may continue on the stream's next page.  FFmpeg's `ogg` demuxer finds pages by scanning for the capture
// pattern and drops pages whose CRC fails; here the chain is followed by length, and damage is refused (DESIGN.md
// section 2).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SBOGG_HD __host__ __device__ __forceinline__
#else
#define SBOGG_HD inline
#endif

namespace sbogg {

constexpr int kHeader = 27;                               // bytes of a page header before its lacing values
constexpr uint32_t kPoly = 0x04C11DB7u;                   // the CRC-32 polynomial, MSB first, initial value 0

enum {
    kOk = 0,
    kNoCapture, kBadVersion, kBadCrc, kChained,           // the chain (every page)
    kSeqGap, kBadContinuation,                            // the chosen stream's pages
};

SBOGG_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kNoCapture: return "no capture pattern where the page before it ends (a broken page header, a wrong lacing "
                            "value, or bytes between pages)";
    case kBadVersion: return "unsupported stream structure version (not 0)";
    case kBadCrc: return "page CRC-32 mismatch";
    case kChained: return "a new stream begins after the first data page (chained Ogg is not supported)";
    case kSeqGap: return "page sequence number does not follow the stream's previous page (a page is missing)";
    case kBadContinuation: return "continuation flag contradicts the stream's previous page (a packet is missing "
                                  "its start or its end)";
    default: return "unknown error";
    }
}

// How the page at a chain position ends (Link.kind)
enum {
    kLink = 0,       // the next page starts at .next, before the buffer's limit
    kNext,           // the page is whole; the next one starts at or after the limit (the next chunk measures it)
    kPast,           // the page runs past the bytes there are (carried to the next chunk; at the end: cut)
    kBroken,         // no capture pattern at .next
    kBadHeader,      // a version byte other than 0 at the position itself
};

SBOGG_HD bool is_capture(const uint8_t* p) { return p[0] == 'O' && p[1] == 'g' && p[2] == 'g' && p[3] == 'S'; }

SBOGG_HD uint32_t le32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// The length of the page at p (a capture pattern), `avail` bytes readable there: > 0 the length, 0 a bad version
// byte, -1 too few bytes to tell
SBOGG_HD int64_t page_length(const uint8_t* p, int64_t avail) {
    if (avail < 5) return -1;
    if (p[4] != 0) return 0;
    if (avail < kHeader) return -1;
    const int nsegs = p[26];
    if (avail < kHeader + nsegs) return -1;
    int64_t len = kHeader + nsegs;
    for (int i = 0; i < nsegs; ++i) len += p[kHeader + i];
    return len;
}

// The most pages a buffer of n bytes with m capture patterns holds, which sizes sb_ogg.cu's page table for it: every
// page is a candidate and takes at least its 27 header bytes (a page may have no segments)
SBOGG_HD int64_t max_pages(int64_t m, int64_t n) { return m < n / kHeader + 1 ? m : n / kHeader + 1; }

struct Link {
    int kind;
    int64_t next;        // kLink / kNext / kBroken: where the next page starts
};

// The page at buffer position q (a capture pattern, q < limit) of a buffer of n bytes, limit == n - 3.  is_cand(p):
// whether position p is a capture pattern the scan found.
template <class IsCand>
SBOGG_HD Link link(const uint8_t* buf, int64_t q, int64_t n, int64_t limit, IsCand is_cand) {
    Link r;
    r.next = -1;
    const int64_t len = page_length(buf + q, n - q);
    if (len == 0) { r.kind = kBadHeader; return r; }
    if (len < 0 || q + len > n) { r.kind = kPast; return r; }
    r.next = q + len;
    if (r.next >= limit) { r.kind = kNext; return r; }
    r.kind = is_cand(r.next) ? kLink : kBroken;
    return r;
}

// ---- the page CRC-32 ---------------------------------------------------------------------------------------------
// The CRC of a byte range with initial value 0 and no final XOR is M(x) x^32 mod P, so for adjacent ranges A, B:
// crc(A B) = crc(A) x^(8 |B|) + crc(B) mod P (zlib's crc32_combine, for this unreflected form).  A warp checks a page
// as 32 slices combined by that rule.

SBOGG_HD uint32_t crc_entry(uint32_t i) {
    uint32_t c = i << 24;
    for (int k = 0; k < 8; ++k) c = (c & 0x80000000u) ? (c << 1) ^ kPoly : c << 1;
    return c;
}

// a(x) b(x) mod P
SBOGG_HD uint32_t gf_mul(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int i = 31; i >= 0; --i) {
        r = (r & 0x80000000u) ? (r << 1) ^ kPoly : r << 1;
        if ((b >> i) & 1u) r ^= a;
    }
    return r;
}

// x^(8 n) mod P
SBOGG_HD uint32_t x_pow8(int64_t n) {
    uint32_t r = 1u, base = 0x100u;
    for (; n; n >>= 1) {
        if (n & 1) r = gf_mul(r, base);
        base = gf_mul(base, base);
    }
    return r;
}

SBOGG_HD uint32_t crc_combine(uint32_t a, uint32_t b, int64_t len_b) { return gf_mul(a, x_pow8(len_b)) ^ b; }

// The CRC of page bytes [lo, hi) (offsets in the page), the CRC field (bytes 22 to 25) read as zeros; table: crc_entry
template <class Table>
SBOGG_HD uint32_t crc_range(const uint8_t* page, int64_t lo, int64_t hi, const Table& table) {
    uint32_t c = 0;
    for (int64_t i = lo; i < hi; ++i) {
        const uint32_t b = (i >= 22 && i < 26) ? 0u : page[i];
        c = (c << 8) ^ table[(c >> 24) ^ b];
    }
    return c;
}

SBOGG_HD uint32_t stored_crc(const uint8_t* page) { return le32(page + 22); }

// ---- a page's packets ----------------------------------------------------------------------------------------------
struct Page {
    int flags;                 // 1 continued, 2 first of its stream (BOS), 4 last (EOS)
    uint32_t serial, seq;
    int hdr;                   // 27 + segment count: where the body starts
    int64_t body;              // body bytes
    int starts;                // packets that start on the page
    int open;                  // 1: a packet continues on the next page (the last lacing value is 255)
    int64_t closed;            // where in the body the last packet ending on the page ends, -1 if none does
};

SBOGG_HD Page page_info(const uint8_t* p) {
    Page r;
    r.flags = p[5];
    r.serial = le32(p + 14);
    r.seq = le32(p + 18);
    const int nsegs = p[26];
    r.hdr = kHeader + nsegs;
    r.body = 0; r.starts = 0; r.closed = -1;
    for (int i = 0; i < nsegs; ++i) {
        const int l = p[kHeader + i];
        if (i == 0 ? !(r.flags & 1) : p[kHeader + i - 1] < 255) ++r.starts;
        r.body += l;
        if (l < 255) r.closed = r.body;
    }
    // a page without segments leaves the packet that was open before it open
    r.open = nsegs > 0 ? p[kHeader + nsegs - 1] == 255 : (r.flags & 1);
    return r;
}

// where(k, off): the k-th packet starting on page p starts at body offset off
template <class Where>
SBOGG_HD void packet_starts(const uint8_t* p, Where where) {
    const int nsegs = p[26], flags = p[5];
    int64_t off = 0;
    int k = 0;
    for (int i = 0; i < nsegs; ++i) {
        if (i == 0 ? !(flags & 1) : p[kHeader + i - 1] < 255) where(k++, off);
        off += p[kHeader + i];
    }
}

}  // namespace sbogg
