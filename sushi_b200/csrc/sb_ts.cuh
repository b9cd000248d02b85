// MPEG transport stream demuxing and Blu-ray LPCM decoding, written once for the GPU kernels of sb_ts.cu and for the CPU
// (tests/emu/emu_ts_driver.cpp compiles this header with g++).  Everything here is a __host__ __device__ function of
// plain integers and byte pointers: the TS packet header and adaptation field, the continuity counter rule, the PES
// header (PES_packet_length, header length, PTS, PES extension 2's stream_id_extension), the BD-LPCM header and the
// sample conversion.
//
// The rules are FFmpeg's (libavformat/mpegts.c, libavcodec/pcm-bluray.c) where FFmpeg decodes; where FFmpeg resyncs,
// skips or only warns (lost sync, TEI, scrambling, CC gaps, a PES length mismatch, an LPCM header change) the packet
// or PES is refused instead (DESIGN.md section 2).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SBTS_HD __host__ __device__ __forceinline__
#else
#define SBTS_HD inline
#endif

namespace sbts {

constexpr int kTsSize = 188;          // a TS packet; BDAV packets carry a 4-byte arrival time stamp in front of it
constexpr int kMaxPayload = 184;

enum {
    kOk = 0,
    kLostSync, kTei, kScrambled, kBadAdaptation, kCcGap,                           // TS packets (k_ts_scan)
    kNoStartCode, kPesLength, kBadPesHeader, kBadStreamId,                        // PES packets (k_pes_index)
    kBadLpcmHeader, kLpcmChange, kShortLpcm, kLpcm20,
};

SBTS_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kLostSync: return "lost sync (no 0x47 sync byte)";
    case kTei: return "transport error indicator set";
    case kScrambled: return "scrambled packet";
    case kBadAdaptation: return "adaptation field length runs past the packet";
    case kCcGap: return "continuity counter gap";
    case kNoStartCode: return "PES packet without a start code";
    case kPesLength: return "PES_packet_length disagrees with the bytes the PID carries";
    case kBadPesHeader: return "invalid PES header";
    case kBadStreamId: return "PES stream id carries no audio";
    case kBadLpcmHeader: return "unsupported BD-LPCM header (channel assignment, sample rate or bits)";
    case kLpcmChange: return "BD-LPCM header changes the channel assignment, sample rate or bits of the first PES packet";
    case kShortLpcm: return "PES packet too short for its BD-LPCM header";
    case kLpcm20: return "20-bit BD-LPCM, which FFmpeg's pcm_bluray decoder does not decode either";
    default: return "unknown error";
    }
}

// What k_ts_scan keeps of one packet of the chosen PID.  payload_off counts from the sync byte.
struct Packet {
    int16_t payload_off, payload_len;
    uint8_t pusi, cc, disc, has_payload;
};

// The 188-byte packet at `p` (its sync byte).  *pid_out receives the PID (-1 when the sync byte is missing).  For a
// packet of `pid` the header and adaptation field are checked and *out filled; other PIDs are only sync-checked.
SBTS_HD int parse_packet(const uint8_t* p, int pid, int* pid_out, Packet* out) {
    *pid_out = -1;
    if (p[0] != 0x47) return kLostSync;
    const int id = ((p[1] & 0x1F) << 8) | p[2];
    *pid_out = id;
    if (id != pid) return kOk;
    if (p[1] & 0x80) return kTei;
    if (p[3] & 0xC0) return kScrambled;
    const int afc = (p[3] >> 4) & 3;
    int off = 4, disc = 0;
    if (afc & 2) {
        const int len = p[4];
        // adaptation field only: it fills the packet; with a payload: at most 182 bytes, leaving at least one
        if (len > (afc == 2 ? 183 : 182)) return kBadAdaptation;
        if (len > 0) disc = p[5] >> 7;
        off = 5 + len;
    }
    out->payload_off = (int16_t)off;
    out->payload_len = (int16_t)((afc & 1) ? kTsSize - off : 0);
    out->pusi = (uint8_t)((p[1] >> 6) & 1);
    out->cc = (uint8_t)(p[3] & 15);
    out->disc = (uint8_t)disc;
    out->has_payload = (uint8_t)(afc & 1);
    return kOk;
}

// FFmpeg's continuity rule: a packet with a payload advances the counter by one, one without repeats it; a
// discontinuity_indicator accepts any value; the PID's first packet starts the count.
SBTS_HD bool cc_ok(bool have_prev, int prev_cc, const Packet& q) {
    if (!have_prev || q.disc) return true;
    const int expect = q.has_payload ? ((prev_cc + 1) & 15) : prev_cc;
    return q.cc == expect;
}

// One PES packet: bytes [b, e) of the PID's payload, from its payload-unit-start packet up to the next one (or the
// end of the file).  `at_end`: the last PES, which a cut file leaves short.
struct Pes {
    int code;
    int64_t payload_off, payload_len;     // the PES payload (after the header), in the PID's payload bytes
    int stream_id, ext_id;                // ext_id: stream_id_extension, or -1
    int cut;                              // 1: the last PES, shorter than its PES_packet_length (kept, as FFmpeg does);
                                          // 2: the last PES, cut inside its header (dropped, as FFmpeg does)
};

SBTS_HD Pes parse_pes(const uint8_t* es, int64_t b, int64_t e, bool at_end) {
    Pes r;
    r.code = kOk; r.payload_off = r.payload_len = 0; r.stream_id = 0; r.ext_id = -1; r.cut = 0;
    const int64_t n = e - b;
    const uint8_t* h = es + b;
    if (n >= 3 && !(h[0] == 0 && h[1] == 0 && h[2] == 1)) { r.code = kNoStartCode; return r; }
    if (n < 6) {
        if (at_end) r.cut = 2;
        else r.code = kPesLength;
        return r;
    }
    r.stream_id = h[3];
    const int64_t len = (h[4] << 8) | h[5];
    if (len != 0 && n != len + 6) {
        if (!(at_end && n < len + 6)) { r.code = kPesLength; return r; }
        r.cut = 1;
    }
    // private_stream_1 (BD LPCM), extended_stream_id (TrueHD) and the audio / video ids carry a PES header
    const int sid = r.stream_id;
    if (!(sid == 0xBD || sid == 0xFD || (sid >= 0xC0 && sid <= 0xEF))) { r.code = kBadStreamId; return r; }
    if (n < 9) {
        if (r.cut) { r.cut = 2; return r; }
        r.code = kBadPesHeader; return r;
    }
    if ((h[6] & 0xC0) != 0x80) { r.code = kBadPesHeader; return r; }
    const int flags = h[7], hlen = h[8];
    if (9 + hlen > n) {
        if (r.cut) { r.cut = 2; return r; }
        r.code = kBadPesHeader; return r;
    }
    // the optional fields, in order, within the header; FFmpeg's walk to PES extension 2
    int at = 9;
    const int end = 9 + hlen;
    const int pts = flags >> 6;
    if (pts == 1) { r.code = kBadPesHeader; return r; }
    at += pts == 2 ? 5 : pts == 3 ? 10 : 0;
    if (pts >= 2 && at <= end && !(h[9] & 1)) { r.code = kBadPesHeader; return r; }     // PTS marker bit
    if (flags & 0x20) at += 6;                // ESCR
    if (flags & 0x10) at += 3;                // ES_rate
    if (flags & 0x08) at += 1;                // DSM trick mode
    if (flags & 0x04) at += 1;                // additional copy info
    if (flags & 0x02) at += 2;                // previous PES CRC
    if (at > end) { r.code = kBadPesHeader; return r; }
    if ((flags & 0x01) && at < end) {
        const int ext = h[at++];
        int skip = (ext >> 4) & 0xB;          // private data (16 bytes), sequence counter (2), P-STD buffer (2)
        skip += skip & 0x9;
        at += skip;
        if ((ext & 0x41) == 0x01 && at + 2 <= end && (h[at] & 0x7F) > 0 && (h[at + 1] & 0x80) == 0)
            r.ext_id = h[at + 1];
    }
    r.payload_off = b + end;
    r.payload_len = n - end;
    return r;
}

// The BD-LPCM header (the first 4 bytes of each PES payload), as FFmpeg's pcm_bluray decoder reads it.  The first 16
// bits (the payload size) are not read.
struct Lpcm {
    int channels, src_channels, rate, bits, width;   // width: bytes per coded sample (2, or 3 for 24 bits)
};

SBTS_HD uint32_t lpcm_fields(uint32_t header) { return header & 0xFFC0u; }   // channel assignment, rate, bits

// 0, or why the header is refused: kLpcm20 for 20-bit samples (FFmpeg's decoder refuses them), kBadLpcmHeader for a
// reserved channel assignment, sample rate or bits code
SBTS_HD int parse_lpcm(uint32_t header, Lpcm* out) {
    // channels of each channel assignment: 1 mono, 3 stereo, 4 3.0, 5 2.1, 6 3.1, 7 2.2, 8 3.2, 9 3.2+LFE, 10 3.4,
    // 11 3.4+LFE; coded with an even count, the last channel of an odd count being padding
    const int chans[16] = {0, 1, 0, 2, 3, 3, 4, 4, 5, 6, 7, 8, 0, 0, 0, 0};
    const int ch = chans[(header >> 12) & 15];
    const int rc = (header >> 8) & 15;
    const int rate = rc == 1 ? 48000 : rc == 4 ? 96000 : rc == 5 ? 192000 : 0;
    const int bc = (header >> 6) & 3;
    if (!ch || !rate || !bc) return kBadLpcmHeader;
    if (bc == 2) return kLpcm20;
    out->channels = ch;
    out->src_channels = (ch + 1) & ~1;
    out->rate = rate;
    out->bits = bc == 1 ? 16 : 24;
    out->width = bc == 1 ? 2 : 3;
    return kOk;
}

SBTS_HD int64_t lpcm_frames(int64_t payload_len, const Lpcm& f) {
    // whole sample frames after the header; leftover bytes are ignored, as FFmpeg ignores them
    return payload_len < 4 ? 0 : (payload_len - 4) / ((int64_t)f.src_channels * f.width);
}

// One sample frame at `src` into `dst`: big-endian samples, the top 16 bits kept, the padding channel skipped.
SBTS_HD void lpcm_frame(const uint8_t* src, const Lpcm& f, int16_t* dst) {
    for (int c = 0; c < f.channels; ++c)
        dst[c] = (int16_t)(uint16_t)((src[c * f.width] << 8) | src[c * f.width + 1]);
}

}  // namespace sbts
