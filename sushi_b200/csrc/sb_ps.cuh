// MPEG program stream demuxing, written once for the GPU kernels of sb_ps.cu and for the CPU (tests/emu/emu_ps_driver.cpp
// compiles this header with g++).  Everything here is a __host__ __device__ function of plain integers and byte
// pointers: which bytes start a packet, how long each packet is, how one packet links to the next on the chain, and the
// PES header in its MPEG-1 and MPEG-2 forms.
//
// A program stream is a chain of packets, each starting with a start code 00 00 01 xx (xx >= 0xB9) and giving its own
// length: the pack header (MPEG-1: 12 bytes; MPEG-2: 14 bytes and up to 7 stuffing bytes), the program end code (4
// bytes), and every other packet (system header, PSM, padding, private streams, PES) 6 bytes and its 16-bit length.
// FFmpeg's `mpeg` demuxer finds packets by scanning for start codes and resyncs past damage; here the chain is followed
// by length, and a link that does not land on a start code is refused (DESIGN.md section 2).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SBPS_HD __host__ __device__ __forceinline__
#else
#define SBPS_HD inline
#endif

namespace sbps {

// Bytes a packet's length needs at most (an MPEG-2 pack header's stuffing length is its 14th byte).  A chunk's last
// kTail bytes are left for the next one, where the packet starting there can be measured.
constexpr int kTail = 16;

enum {
    kOk = 0,
    kNoStartCode, kBadPack,                               // the chain (program stream packets)
    kBadPesHeader,                                        // the chosen stream's PES packets
};

SBPS_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kNoStartCode: return "no start code where the packet before it ends (broken start code, a wrong length, or "
                              "bytes between packets)";
    case kBadPack: return "invalid pack header (neither MPEG-1 nor MPEG-2)";
    case kBadPesHeader: return "invalid PES header";
    default: return "unknown error";
    }
}

// How the packet at a chain position ends (Link.kind)
enum {
    kLink = 0,       // the next packet starts at .next, before the chunk's limit
    kNext,           // the packet is whole; the next one starts at or after the limit (the next chunk measures it)
    kPast,           // the packet runs past the bytes there are (carried to the next chunk; at the end: cut)
    kBroken,         // no start code at .next
    kBadHeader,      // an invalid pack header at the position itself
};

SBPS_HD bool is_start(const uint8_t* p) { return p[0] == 0 && p[1] == 0 && p[2] == 1 && p[3] >= 0xB9; }

// The length of the packet at p (a start code), `avail` bytes readable there: > 0 the length, 0 an invalid pack
// header, -1 too few bytes to tell
SBPS_HD int64_t packet_length(const uint8_t* p, int64_t avail) {
    const int code = p[3];
    if (code == 0xB9) return 4;
    if (code == 0xBA) {
        if (avail < 5) return -1;
        if ((p[4] & 0xC0) == 0x40) return avail < 14 ? -1 : 14 + (p[13] & 7);
        if ((p[4] & 0xF0) == 0x20) return 12;
        return 0;
    }
    if (avail < 6) return -1;
    return 6 + (((int64_t)p[4] << 8) | p[5]);
}

struct Link {
    int kind;
    int64_t next;        // kLink / kNext / kBroken: where the next packet starts
};

// The packet at buffer position q (a start code, q < limit) of a buffer of n bytes.  is_cand(p): whether position p is
// a start code the scan found (p < limit).  `at_end`: the buffer ends the file, limit == n - 3.
template <class IsCand>
SBPS_HD Link link(const uint8_t* buf, int64_t q, int64_t n, int64_t limit, bool at_end, IsCand is_cand) {
    Link r;
    r.next = -1;
    const int64_t len = packet_length(buf + q, n - q);
    if (len == 0) { r.kind = kBadHeader; return r; }
    if (len < 0 || q + len > n) { r.kind = kPast; return r; }
    r.next = q + len;
    if (r.next >= limit || (at_end && n - r.next < 4)) { r.kind = kNext; return r; }   // a file may end inside a start code
    r.kind = is_cand(r.next) ? kLink : kBroken;
    return r;
}

// The payload of one PES packet of the chosen stream at h: `have` of its bytes present (fewer than its length only
// for the last packet of a cut file).  FFmpeg's mpegps_read_pes_header: 0xFF stuffing; an MPEG-1 STD buffer field;
// then an MPEG-1 PTS or PTS + DTS, an MPEG-2 header (flags, header length, the PTS and DTS it announces inside it), or
// MPEG-1's lone 0x0F.  Where FFmpeg skips a packet whose header it cannot read, the packet is refused.
struct Pes {
    int code;
    int64_t payload_off, payload_len;  // from h
    int cut;                           // 1: cut short, the bytes there are kept; 2: cut inside its header, dropped
};

SBPS_HD Pes parse_pes(const uint8_t* h, int64_t have) {
    Pes r;
    r.code = kOk; r.payload_off = r.payload_len = 0; r.cut = 0;
    if (have < 6) { r.cut = 2; return r; }
    const int64_t end = 6 + (((int64_t)h[4] << 8) | h[5]);
    const int64_t n = have < end ? have : end;
    if (have < end) r.cut = 1;
    int64_t at = 6;
    while (at < n && h[at] == 0xFF) ++at;
    if (at < n && (h[at] & 0xC0) == 0x40) at += 2;
    if (at >= n) {
        if (r.cut) r.cut = 2; else r.code = kBadPesHeader;
        return r;
    }
    const int c = h[at];
    if ((c & 0xE0) == 0x20) {
        at += (c & 0x10) ? 10 : 5;
    } else if ((c & 0xC0) == 0x80) {
        if (at + 3 > n) {
            if (r.cut) r.cut = 2; else r.code = kBadPesHeader;
            return r;
        }
        const int flags = h[at + 1], hlen = h[at + 2];
        const int need = (flags & 0x80) ? ((flags & 0x40) ? 10 : 5) : 0;
        if (hlen < need || at + 3 + hlen > end) { r.code = kBadPesHeader; return r; }
        at += 3 + hlen;
    } else if (c == 0x0F) {
        at += 1;
    } else {
        r.code = kBadPesHeader;
        return r;
    }
    if (at > end) { r.code = kBadPesHeader; return r; }
    if (at > n) { r.cut = 2; return r; }
    r.payload_off = at;
    r.payload_len = n - at;
    return r;
}

}  // namespace sbps
