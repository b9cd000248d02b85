// FLAC frame decoding, written once for the GPU kernels of sb_flac.cu and for the CPU (tests/emu/emu_flac_driver.cpp
// compiles this header with g++).  Everything here is a __host__ __device__ function of plain integers and byte
// pointers: the bit reader, the frame header parse with its CRC-8, the subframe decode (CONSTANT, VERBATIM, FIXED,
// LPC, Rice / Rice2 residuals with escape partitions, wasted bits), the channel decorrelation and the CRC-16.
//
// Widths: bit positions are 64-bit (a 1 GB file has 2^33 bits), coded sample numbers are 36 bits, and the LPC sum is
// accumulated in 64 bits (25-bit side samples x 15-bit coefficients x order 32 reach 2^45).
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <algorithm>
#include <vector>

#if defined(__CUDACC__)
#define SBF_HD __host__ __device__ __forceinline__
#else
#define SBF_HD inline
#endif

namespace sbflac {

// error codes of a frame (FrameStatus::code); flac_error_text names them
enum {
    kOk = 0,
    kBadSync, kBadHeader, kBadCrc8, kMismatch,            // header
    kBadSubframe, kBadResidual, kBadLpc, kOverrun,        // subframes
    kBadCrc16, kBadEnd, kTruncated,                        // frame end
};

SBF_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kBadSync: return "no frame sync code";
    case kBadHeader: return "invalid frame header";
    case kBadCrc8: return "frame header CRC-8 mismatch";
    case kMismatch: return "frame header disagrees with STREAMINFO";
    case kBadSubframe: return "invalid subframe header";
    case kBadResidual: return "invalid residual coding";
    case kBadLpc: return "invalid LPC precision or shift";
    case kOverrun: return "subframes run past the next frame";
    case kBadCrc16: return "frame CRC-16 mismatch";
    case kBadEnd: return "frame does not end where the next frame starts";
    case kTruncated: return "truncated frame";
    default: return "unknown error";
    }
}

// ---- CRCs ----------------------------------------------------------------------------------------------------------
// CRC-8 (polynomial x^8 + x^2 + x + 1) of a frame header: at most 16 bytes, bitwise
SBF_HD uint8_t crc8(const uint8_t* p, int n) {
    unsigned crc = 0;
    for (int i = 0; i < n; ++i) {
        crc ^= p[i];
        for (int b = 0; b < 8; ++b) crc = (crc & 0x80) ? ((crc << 1) ^ 0x07) & 0xFF : (crc << 1) & 0xFF;
    }
    return (uint8_t)crc;
}

// CRC-16 (polynomial x^16 + x^15 + x^2 + 1) of a whole frame, one table lookup per byte
SBF_HD uint16_t crc16_entry(int byte) {
    unsigned crc = (unsigned)byte << 8;
    for (int b = 0; b < 8; ++b) crc = (crc & 0x8000) ? ((crc << 1) ^ 0x8005) & 0xFFFF : (crc << 1) & 0xFFFF;
    return (uint16_t)crc;
}
SBF_HD uint16_t crc16(const uint16_t* table, const uint8_t* p, int64_t n) {
    unsigned crc = 0;
    for (int64_t i = 0; i < n; ++i) crc = ((crc << 8) ^ table[((crc >> 8) ^ p[i]) & 0xFF]) & 0xFFFF;
    return (uint16_t)crc;
}

// ---- frame header --------------------------------------------------------------------------------------------------
// What a frame header says, after it has been checked against STREAMINFO (channels, bits, rate)
struct Header {
    int64_t number;        // frame number (fixed blocking) or first sample number (variable blocking)
    int block_size;
    int assignment;        // 0..7 independent (assignment + 1 channels), 8 left/side, 9 side/right, 10 mid/side
    int variable;          // blocking strategy bit of the sync code
    int length;            // header bytes, CRC-8 included
};

SBF_HD int assignment_channels(int a) { return a < 8 ? a + 1 : 2; }
SBF_HD int code_rate(int c) {
    switch (c) {
    case 1: return 88200; case 2: return 176400; case 3: return 192000; case 4: return 8000; case 5: return 16000;
    case 6: return 22050; case 7: return 24000; case 8: return 32000; case 9: return 44100; case 10: return 48000;
    case 11: return 96000; default: return 0;
    }
}
SBF_HD int code_bits(int c) {
    switch (c) { case 1: return 8; case 2: return 12; case 4: return 16; case 5: return 20; case 6: return 24; case 7: return 32; default: return 0; }
}

// Parse the header at p[0..avail).  Returns kOk or an error code; `h` is valid on kOk.
SBF_HD int parse_header(const uint8_t* p, int64_t avail, int channels, int bits, int rate, Header* h) {
    if (avail < 6 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return kBadSync;
    h->variable = p[1] & 1;
    const int bs_code = p[2] >> 4, sr_code = p[2] & 15;
    const int assign = p[3] >> 4, ss_code = (p[3] >> 1) & 7;
    if (bs_code == 0 || sr_code == 15 || assign > 10 || ss_code == 3 || (p[3] & 1)) return kBadHeader;
    // UTF-8-style coded number: 1 to 7 bytes, at most 31 bits (frame number) or 36 bits (sample number)
    int at = 4;
    uint64_t v = p[at];
    int extra;
    if (!(v & 0x80)) extra = 0;
    else if ((v & 0xE0) == 0xC0) { extra = 1; v &= 0x1F; }
    else if ((v & 0xF0) == 0xE0) { extra = 2; v &= 0x0F; }
    else if ((v & 0xF8) == 0xF0) { extra = 3; v &= 0x07; }
    else if ((v & 0xFC) == 0xF8) { extra = 4; v &= 0x03; }
    else if ((v & 0xFE) == 0xFC) { extra = 5; v &= 0x01; }
    else if (v == 0xFE) { extra = 6; v = 0; }
    else return kBadHeader;
    if (extra == 6 && !h->variable) return kBadHeader;
    if (avail < at + 1 + extra + 4) return kBadSync;
    ++at;
    for (int i = 0; i < extra; ++i, ++at) {
        if ((p[at] & 0xC0) != 0x80) return kBadHeader;
        v = (v << 6) | (p[at] & 0x3F);
    }
    h->number = (int64_t)v;
    int bs;
    if (bs_code == 1) bs = 192;
    else if (bs_code <= 5) bs = 576 << (bs_code - 2);
    else if (bs_code == 6) bs = p[at++] + 1;
    else if (bs_code == 7) { bs = ((p[at] << 8) | p[at + 1]) + 1; at += 2; }
    else bs = 256 << (bs_code - 8);
    int sr = 0;
    if (sr_code == 12) sr = p[at++] * 1000;
    else if (sr_code == 13) { sr = (p[at] << 8) | p[at + 1]; at += 2; }
    else if (sr_code == 14) { sr = ((p[at] << 8) | p[at + 1]) * 10; at += 2; }
    if (crc8(p, at) != p[at]) return kBadCrc8;
    h->length = at + 1;
    h->block_size = bs;
    h->assignment = assign;
    // against STREAMINFO
    if (sr_code >= 1 && sr_code <= 11) sr = code_rate(sr_code);
    if (assignment_channels(assign) != channels) return kMismatch;
    if (ss_code != 0 && code_bits(ss_code) != bits) return kMismatch;
    if (sr_code != 0 && sr != rate) return kMismatch;
    return kOk;
}

// ---- bit reader ----------------------------------------------------------------------------------------------------
// MSB-first reader over p[0..limit) with a 64-bit cache.  Bytes past the limit read as zero; overrun() tells whether
// the bits consumed so far run past it (the cache itself may look ahead of the limit without harm)
struct BitReader {
    const uint8_t* p;
    int64_t next;          // next byte to load into the cache
    int64_t limit;         // bytes that may be read
    uint64_t cache;        // unread bits, left-aligned
    int bits;              // valid bits in cache

    SBF_HD void init(const uint8_t* base, int64_t byte_pos, int64_t limit_bytes) {
        p = base; next = byte_pos; limit = limit_bytes; cache = 0; bits = 0;
    }
    SBF_HD void refill() {
        while (bits <= 56) {
            const uint64_t b = next < limit ? p[next] : 0;
            ++next;
            cache |= b << (56 - bits);
            bits += 8;
        }
    }
    // absolute bit position of the next unread bit
    SBF_HD int64_t position() const { return next * 8 - bits; }
    SBF_HD bool overrun() const { return position() > limit * 8; }
    SBF_HD uint32_t read(int n) {                       // 0 <= n <= 32
        if (n == 0) return 0;
        if (bits < n) refill();
        const uint32_t v = (uint32_t)(cache >> (64 - n));
        cache <<= n; bits -= n;
        return v;
    }
    SBF_HD int32_t read_signed(int n) {                 // n-bit two's complement, 0 <= n <= 32
        if (n == 0) return 0;
        const uint32_t v = read(n);
        return n == 32 ? (int32_t)v : (int32_t)(v << (32 - n)) >> (32 - n);
    }
    // zero bits before the next one bit, which is consumed too; stops once past the limit (overrun() is then true)
    SBF_HD uint32_t unary() {
        uint32_t q = 0;
        for (;;) {
            if (bits == 0) refill();
            if (cache) {
#if defined(__CUDA_ARCH__)
                const int z = __clzll((long long)cache);
#else
                const int z = __builtin_clzll(cache);
#endif
                q += z; cache <<= z; cache <<= 1; bits -= z + 1;
                return q;
            }
            q += bits; bits = 0;
            if (overrun()) return q;
        }
    }
    SBF_HD void align() { const int r = bits & 7; cache <<= r; bits -= r; }
};

// ---- subframes -----------------------------------------------------------------------------------------------------
// Residual of a FIXED or LPC subframe into out[order .. n)
SBF_HD int residual(BitReader& br, int n, int order, int32_t* out) {
    const int method = (int)br.read(2);
    if (method > 1) return kBadResidual;
    const int pbits = method == 0 ? 4 : 5, escape = (1 << pbits) - 1;
    const int porder = (int)br.read(4);
    const int parts = 1 << porder;
    const int psize = n >> porder;
    if ((psize << porder) != n || psize < order) return kBadResidual;
    int i = order;
    for (int part = 0; part < parts; ++part) {
        const int end = (part + 1) * psize;
        const int k = (int)br.read(pbits);
        if (k == escape) {
            const int raw = (int)br.read(5);
            for (; i < end; ++i) out[i] = br.read_signed(raw);
        } else {
            for (; i < end; ++i) {
                const uint32_t q = br.unary();
                if (q > 64 && br.overrun()) return kOverrun;
                const uint32_t u = (q << k) | br.read(k);
                out[i] = (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
            }
        }
        if (br.overrun()) return kOverrun;
    }
    return kOk;
}

SBF_HD void restore_fixed(int32_t* x, int n, int order) {
    switch (order) {
    case 1: for (int i = 1; i < n; ++i) x[i] += x[i - 1]; break;
    case 2: for (int i = 2; i < n; ++i) x[i] += 2 * x[i - 1] - x[i - 2]; break;
    case 3: for (int i = 3; i < n; ++i) x[i] += 3 * x[i - 1] - 3 * x[i - 2] + x[i - 3]; break;
    case 4: for (int i = 4; i < n; ++i) x[i] += 4 * x[i - 1] - 6 * x[i - 2] + 4 * x[i - 3] - x[i - 4]; break;
    default: break;
    }
}

SBF_HD void restore_lpc(int32_t* x, int n, int order, const int32_t* coef, int shift) {
    for (int i = order; i < n; ++i) {
        int64_t sum = 0;
        for (int j = 0; j < order; ++j) sum += (int64_t)coef[j] * (int64_t)x[i - 1 - j];
        x[i] += (int32_t)(sum >> shift);
    }
}

// One subframe of n samples at `bps` bits (side channels carry one more) into out[0..n)
SBF_HD int subframe(BitReader& br, int n, int bps, int32_t* out) {
    if (br.read(1)) return kBadSubframe;                 // zero padding bit
    const int type = (int)br.read(6);
    int wasted = 0;
    if (br.read(1)) {
        wasted = (int)br.unary() + 1;
        if (br.overrun()) return kOverrun;
        if (wasted >= bps) return kBadSubframe;
    }
    const int sbps = bps - wasted;
    if (type == 0) {                                      // CONSTANT
        const int32_t v = br.read_signed(sbps);
        for (int i = 0; i < n; ++i) out[i] = v;
    } else if (type == 1) {                               // VERBATIM
        for (int i = 0; i < n; ++i) out[i] = br.read_signed(sbps);
    } else if (type >= 8 && type <= 12) {                 // FIXED, order 0..4
        const int order = type - 8;
        if (order > n) return kBadSubframe;
        for (int i = 0; i < order; ++i) out[i] = br.read_signed(sbps);
        const int rc = residual(br, n, order, out);
        if (rc != kOk) return rc;
        restore_fixed(out, n, order);
    } else if (type >= 32) {                              // LPC, order 1..32
        const int order = type - 31;
        if (order > n) return kBadSubframe;
        for (int i = 0; i < order; ++i) out[i] = br.read_signed(sbps);
        const int prec = (int)br.read(4) + 1;
        if (prec == 16) return kBadLpc;
        const int shift = br.read_signed(5);
        if (shift < 0) return kBadLpc;
        int32_t coef[32];
        for (int j = 0; j < order; ++j) coef[j] = br.read_signed(prec);
        const int rc = residual(br, n, order, out);
        if (rc != kOk) return rc;
        restore_lpc(out, n, order, coef, shift);
    } else {
        return kBadSubframe;
    }
    if (br.overrun()) return kOverrun;
    if (wasted)
        for (int i = 0; i < n; ++i) out[i] = (int32_t)((uint32_t)out[i] << wasted);
    return kOk;
}

// ---- one frame -----------------------------------------------------------------------------------------------------
// Decode the frame at file[offset]: every subframe, channel c into out[c * block_size ...], then the CRC-16.
// `limit` = the bytes the frame may occupy (the next frame's offset, or the file size for the last frame).
// end_out receives the byte offset just past the frame's CRC-16.
struct FrameStatus { int64_t end; int32_t code; int32_t pad; };

SBF_HD int decode_frame(const uint8_t* file, int64_t offset, int64_t limit, int channels, int bits, int rate,
                        const uint16_t* crc_table, int32_t* out, int64_t* end_out) {
    *end_out = offset;
    Header h;
    int rc = parse_header(file + offset, limit - offset, channels, bits, rate, &h);
    if (rc != kOk) return rc == kBadSync && limit - offset < 16 ? kTruncated : rc;
    BitReader br;
    br.init(file, offset + h.length, limit);
    for (int c = 0; c < channels; ++c) {
        const bool side = (h.assignment == 8 && c == 1) || (h.assignment == 9 && c == 0) || (h.assignment == 10 && c == 1);
        rc = subframe(br, h.block_size, bits + (side ? 1 : 0), out + (int64_t)c * h.block_size);
        if (rc != kOk) return rc;
    }
    br.align();
    const uint32_t stored = br.read(16);
    const int64_t end = br.position() / 8;
    *end_out = end;
    if (br.overrun()) return kOverrun;
    if (crc16(crc_table, file + offset, end - 2 - offset) != stored) return kBadCrc16;
    return kOk;
}

// Channel decorrelation of sample j of a frame whose channels sit at in[c * block_size + j]; 24-bit samples keep
// their top 16 bits (an arithmetic shift right by 8, what the WAV loader reads of a 24-bit sample)
SBF_HD void decorrelate(const int32_t* in, int block_size, int j, int channels, int assignment, int bits, int16_t* out) {
    const int sh = bits - 16;
    if (assignment < 8) {
        for (int c = 0; c < channels; ++c) out[c] = (int16_t)(in[(int64_t)c * block_size + j] >> sh);
        return;
    }
    const int32_t a = in[j], b = in[(int64_t)block_size + j];
    int32_t l, r;
    if (assignment == 8) { l = a; r = a - b; }                       // left, side
    else if (assignment == 9) { l = a + b; r = b; }                  // side, right
    else {                                                            // mid, side
        const int32_t mid = (int32_t)(((uint32_t)a << 1) | (uint32_t)(b & 1));
        l = (mid + b) >> 1; r = (mid - b) >> 1;
    }
    out[0] = (int16_t)(l >> sh); out[1] = (int16_t)(r >> sh);
}

// ---- the chain (host) ----------------------------------------------------------------------------------------------
// A position holding a sync code and a header that parses, agrees with STREAMINFO and passes its CRC-8
struct Candidate { int64_t offset; int64_t number; int32_t block_size; int16_t assignment; int16_t variable; };
// One frame of the chain: its bytes [offset, limit) and its samples [sample, sample + block_size)
struct FrameDesc { int64_t offset; int64_t limit; int64_t sample; int32_t block_size; int32_t assignment; };

// Why no frame starts at byte `offset`: the header there, reparsed from the at most 16 bytes at p
inline const char* no_frame_reason(const uint8_t* p, int64_t offset, int64_t nbytes, int channels, int bits, int rate) {
    if (offset >= nbytes) return "end of file";
    Header h;
    const int rc = parse_header(p, std::min<int64_t>(16, nbytes - offset), channels, bits, rate, &h);
    if (rc == kBadSync && nbytes - offset < 16) return error_text(kTruncated);
    return rc == kOk ? "frame number out of sequence" : error_text(rc);
}

// Frame 0 is the candidate at first_offset; frame k + 1 is the first later candidate with the next coded number (frame
// number k + 1, or sample number s + block size) and the same blocking strategy.  Each frame's limit is the next
// frame's offset (the file size for the last).  Returns false with a message when frame 0 is not there or is
// misnumbered; `first_bytes` are the (at most 16) bytes at first_offset.
inline bool chain(std::vector<Candidate>& cand, int64_t first_offset, int64_t nbytes, int channels, int bits, int rate,
                  const uint8_t* first_bytes, std::vector<FrameDesc>& frames, int64_t* samples, char* msg, size_t msg_len) {
    frames.clear();
    *samples = 0;
    if (first_offset == nbytes) return true;                               // no audio frames: an empty stream
    std::sort(cand.begin(), cand.end(), [](const Candidate& a, const Candidate& b) { return a.offset < b.offset; });
    size_t at = 0;
    while (at < cand.size() && cand[at].offset < first_offset) ++at;
    if (at == cand.size() || cand[at].offset != first_offset) {
        snprintf(msg, msg_len, "FLAC frame 0 at byte offset %lld: %s", (long long)first_offset,
                 no_frame_reason(first_bytes, first_offset, nbytes, channels, bits, rate));
        return false;
    }
    const int variable = cand[at].variable;
    int64_t sample = 0;
    for (;;) {
        const Candidate& cur = cand[at];
        const int64_t want = variable ? sample : (int64_t)frames.size();
        if (cur.number != want) {
            snprintf(msg, msg_len, "FLAC frame %lld at byte offset %lld: coded %s number %lld, expected %lld",
                     (long long)frames.size(), (long long)cur.offset, variable ? "sample" : "frame",
                     (long long)cur.number, (long long)want);
            return false;
        }
        FrameDesc d;
        d.offset = cur.offset; d.limit = nbytes; d.sample = sample; d.block_size = cur.block_size;
        d.assignment = cur.assignment;
        sample += cur.block_size;
        const int64_t next_number = variable ? sample : (int64_t)frames.size() + 1;
        size_t nx = at + 1;
        while (nx < cand.size() && !(cand[nx].number == next_number && cand[nx].variable == variable)) ++nx;
        if (nx < cand.size()) d.limit = cand[nx].offset;
        frames.push_back(d);
        if (nx == cand.size()) break;
        at = nx;
    }
    *samples = sample;
    return true;
}

// ---- frames listed by a container (host and k_flac_frames) -------------------------------------------------------
// In a Matroska track the frame boundaries are the block and lace boundaries: frame f occupies [offsets[f], limit),
// limit being the next listed offset (the buffer size for the last).  What one frame's header says, or why it is
// refused: the header must parse, agree with STREAMINFO and pass its CRC-8 right at its offset
struct ListedFrame { int32_t code; int32_t block_size; int32_t assignment; int32_t pad; };

SBF_HD ListedFrame listed_frame(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, int64_t n, int64_t f,
                                int channels, int bits, int rate) {
    ListedFrame r; r.code = kOk; r.block_size = 0; r.assignment = 0; r.pad = 0;
    const int64_t off = offsets[f], limit = f + 1 < n ? offsets[f + 1] : nbytes;
    if (off < 0 || limit > nbytes || limit < off) { r.code = kTruncated; return r; }
    Header h;
    const int rc = parse_header(buf + off, limit - off, channels, bits, rate, &h);
    if (rc != kOk) { r.code = rc == kBadSync && limit - off < 16 ? kTruncated : rc; return r; }
    r.block_size = h.block_size; r.assignment = h.assignment;
    return r;
}

// The frame table of listed frames: sample positions are the prefix sum of the header block sizes (a track cut from a
// longer stream starts at a coded number above 0, so the numbers are not required to run on).  `where` names each
// frame's block by its file offset in the message.  Returns false with a message.
inline bool list_frames(const ListedFrame* listed, const int64_t* offsets, const int64_t* where, int64_t n, int64_t nbytes,
                        std::vector<FrameDesc>& frames, int64_t* samples, char* msg, size_t msg_len) {
    frames.clear();
    int64_t sample = 0;
    for (int64_t f = 0; f < n; ++f) {
        if (listed[f].code != kOk) {
            snprintf(msg, msg_len, "FLAC frame %lld at byte offset %lld: %s", (long long)f, (long long)where[f],
                     error_text(listed[f].code));
            return false;
        }
        FrameDesc d;
        d.offset = offsets[f]; d.limit = f + 1 < n ? offsets[f + 1] : nbytes; d.sample = sample;
        d.block_size = listed[f].block_size; d.assignment = listed[f].assignment;
        frames.push_back(d);
        sample += listed[f].block_size;
    }
    *samples = sample;
    return true;
}

// Every frame must have decoded, passed its CRC-16 and ended exactly at its limit.  bytes_at(offset, buf16) fetches
// the (at most 16) bytes at an offset for the message about a missing frame.  `where` (NULL for a FLAC file) gives
// the file offset of each listed frame's block: messages then name it, and a frame must end exactly where its lace
// does.  Returns false with a message.
template <class BytesAt>
bool check_frames(const std::vector<FrameDesc>& frames, const FrameStatus* status, int64_t nbytes, int channels, int bits,
                  int rate, BytesAt bytes_at, char* msg, size_t msg_len, const int64_t* where = nullptr) {
    const int64_t nf = (int64_t)frames.size();
    for (int64_t f = 0; f < nf; ++f) {
        const FrameDesc& d = frames[f];
        const FrameStatus& st = status[f];
        const bool last = f == nf - 1;
        if (where) {
            if (st.code != kOk || st.end != d.limit) {
                snprintf(msg, msg_len, "FLAC frame %lld at byte offset %lld: %s", (long long)f, (long long)where[f],
                         st.code != kOk ? error_text(st.code) : "frame does not end where its lace ends");
                return false;
            }
            continue;
        }
        if (st.code != kOk) {
            snprintf(msg, msg_len, "FLAC frame %lld at byte offset %lld: %s", (long long)f, (long long)d.offset,
                     error_text(st.code == kOverrun && last ? kTruncated : st.code));
            return false;
        }
        if (st.end == d.limit) continue;
        if (last) {
            uint8_t buf[16] = {0};
            bytes_at(st.end, buf);
            snprintf(msg, msg_len, "FLAC frame %lld at byte offset %lld: %s", (long long)f + 1, (long long)st.end,
                     no_frame_reason(buf, st.end, nbytes, channels, bits, rate));
        } else {
            snprintf(msg, msg_len, "FLAC frame %lld at byte offset %lld: %s (it ends at byte %lld, the next frame starts "
                     "at byte %lld)", (long long)f, (long long)d.offset, error_text(kBadEnd), (long long)st.end,
                     (long long)d.limit);
        }
        return false;
    }
    return true;
}

}  // namespace sbflac
