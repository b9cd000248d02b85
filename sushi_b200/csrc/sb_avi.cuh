// AVI `movi` demuxing, written once for the GPU kernels of sb_avi.cu and for the CPU (tests/emu/emu_avi_driver.cpp
// compiles this header with g++).  Everything here is a __host__ __device__ function of plain integers and byte
// pointers: which bytes start a chunk, how one chunk links to the next on the chain, and where the chain crosses from
// one `movi` list to the next.
//
// The data of an AVI file lies in `LIST movi` lists: the one of `RIFF AVI ` and, in OpenDML files, one in each `RIFF
// AVIX` that follows.  Inside a list every chunk is a FOURCC, a 32-bit little-endian size and the payload, padded to an
// even length.  The FOURCCs met there are a stream's chunks `NNxx` (two decimal digits, the stream's index in the header,
// then `wb`, `dc`, `db`, `pc` or `tx`), OpenDML's standard index chunks `ix##`, `JUNK`, and `LIST rec ` grouping, whose
// first child follows its 12-byte header.  FFmpeg's `avi` demuxer finds chunks by scanning and resyncs past damage; here
// the chain is followed by size, and a link that does not land on a chunk header, or a size that runs past its `movi`
// list, is refused (DESIGN.md section 2).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SBAVI_HD __host__ __device__ __forceinline__
#else
#define SBAVI_HD inline
#endif

namespace sbavi {

// Bytes a chunk header needs at most (`LIST` size `rec `).  A chunk's last kTail bytes are left for the next one, where
// the chunk starting there can be read.
constexpr int kTail = 12;
// Bytes of a plain chunk header: a file's last chunk may be this short
constexpr int kHeader = 8;
// The chain has left the last `movi` list: every byte after it is ignored
constexpr int64_t kDone = INT64_MAX;

enum {
    kOk = 0,
    kNoChunk, kPastList,                                 // the chain
    kPartialFrame,                                       // the chosen stream's PCM chunks
};

SBAVI_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kNoChunk: return "no chunk header where the chunk before it ends (a broken FOURCC, a wrong size, or bytes "
                          "between chunks)";
    case kPastList: return "chunk size runs past its movi list";
    case kPartialFrame: return "PCM chunk is not a whole number of sample frames";
    default: return "unknown error";
    }
}

// How the chunk at a chain position ends (Link.kind)
enum {
    kLink = 0,       // the next chunk starts at .next, before the buffer's limit
    kNext,           // the next chunk starts at or after the limit (the next buffer reads it), or the chain is done
    kPast,           // a chunk of the chosen stream whose payload runs past the bytes there are (carried; at the end: cut)
    kBroken,         // no chunk header at .next
    kOverrun,        // the chunk's size runs past its movi list
};

SBAVI_HD bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

SBAVI_HD uint32_t rd32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

SBAVI_HD bool is_rec(const uint8_t* p) {
    return p[0] == 'L' && p[1] == 'I' && p[2] == 'S' && p[3] == 'T' && p[8] == 'r' && p[9] == 'e' && p[10] == 'c' &&
           p[11] == ' ';
}

// Whether a chunk header starts at p, `avail` bytes readable there
SBAVI_HD bool is_chunk(const uint8_t* p, int64_t avail) {
    if (avail < 8) return false;
    const uint8_t a = p[0], b = p[1], c = p[2], d = p[3];
    if (is_digit(a) && is_digit(b))
        return (c == 'w' && d == 'b') || (c == 'd' && (d == 'c' || d == 'b')) || (c == 'p' && d == 'c') ||
               (c == 't' && d == 'x');
    if (a == 'i' && b == 'x') return is_digit(c) && is_digit(d);
    if (a == 'J' && b == 'U' && c == 'N' && d == 'K') return true;
    return avail >= 12 && is_rec(p);
}

// The two ASCII digits of stream `index` followed by `wb`, as the 32-bit little-endian FOURCC
SBAVI_HD uint32_t audio_tag(int index) {
    return (uint32_t)('0' + index / 10) | ((uint32_t)('0' + index % 10) << 8) | ((uint32_t)'w' << 16) |
           ((uint32_t)'b' << 24);
}

// The extent [ext[2 e], ext[2 e + 1]) of file offsets holding `f`, of n (sorted, disjoint); -1 if none
SBAVI_HD int64_t extent_of(const int64_t* ext, int64_t n, int64_t f) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (ext[2 * mid + 1] <= f) lo = mid + 1; else hi = mid;
    }
    return lo < n && ext[2 * lo] <= f ? lo : -1;
}

struct Link {
    int kind;
    int64_t next;        // kLink / kNext / kBroken: where the next chunk starts (buffer position; kDone when done)
    int64_t size;        // the chunk's payload size (its header's)
};

// The chunk at buffer position q (a chunk header, q < limit) of a buffer of n bytes whose first byte is at file
// offset base.  ext[0, n_ext): the movi extents.  is_cand(p): whether position p holds a chunk header the scan found
// (p < limit).  `tag`: the chosen stream's FOURCC.  `at_end`: the buffer ends the file, limit == n.
template <class IsCand>
SBAVI_HD Link link(const uint8_t* buf, int64_t q, int64_t n, int64_t limit, bool at_end, int64_t base,
                   const int64_t* ext, int64_t n_ext, uint32_t tag, IsCand is_cand) {
    Link r;
    r.next = -1;
    const uint8_t* p = buf + q;
    const int64_t size = rd32(p + 4);
    r.size = size;
    const int64_t f = base + q;
    const int64_t e = extent_of(ext, n_ext, f);
    const int64_t end = e >= 0 ? ext[2 * e + 1] : f;
    if (e < 0 || f + 8 + size > end) { r.kind = kOverrun; return r; }
    int64_t nf = n - q >= 12 && is_rec(p) ? f + 12 : f + 8 + size + (size & 1);
    if (nf >= end) nf = e + 1 < n_ext ? ext[2 * e + 2] : kDone;
    if (rd32(p) == tag && q + 8 + size > n) { r.kind = kPast; return r; }
    if (nf == kDone) { r.kind = kNext; r.next = kDone; return r; }
    r.next = nf - base;
    if (r.next >= limit || (at_end && n - r.next < kTail && !is_chunk(buf + r.next, n - r.next))) {
        r.kind = kNext;     // a file may end inside a chunk header
        return r;
    }
    r.kind = is_cand(r.next) ? kLink : kBroken;
    return r;
}

}  // namespace sbavi
