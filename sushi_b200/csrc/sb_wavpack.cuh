// WavPack block decoding, written once for the GPU kernel of sb_wavpack.cu and for the CPU
// (tests/emu/emu_wavpack_driver.cpp compiles this header with g++).  Everything here is a __host__ __device__ function of
// plain integers and byte pointers: the metadata sub-blocks of one block (decorrelation terms, weights and sample
// history, entropy medians, ID_INT32_INFO, the custom rate, unknown sub-blocks skipped), the adaptive Golomb code with
// its three medians per channel, zero runs and the held one / zero, decorrelation terms 1-8, 17, 18 and the cross-channel
// terms -1, -2, -3, joint and false stereo, the header's shift, the block CRC and the top-16-bit store.  The arithmetic is
// FFmpeg's `wavpack` decoder's, operation for operation: 32-bit wrap-around for 16-bit streams, 64-bit weight products
// for wider ones.
//
// A block's sub-blocks are bytes [offset, offset + size) of the caller's buffer, which must hold at least 8 readable bytes
// past the last block.  Every sub-block header and every fixed-size field is checked against its sub-block before it is
// read; the bit reader fetches 5 bytes at a time and is checked after each code it reads (a Golomb tail of at most 24
// bits and its extra bit are read before the check), so no read reaches more than 8 bytes past a bitstream sub-block.
//
// The per-term state (value and delta, two weights, two 8-entry histories) lives in a Terms slice: 19 int32 per term,
// field f of term k at p[(k * 19 + f) * stride].  The kernel gives each thread a column of shared memory (stride = the
// block's thread count), so the per-sample loop over terms never touches local memory.
#pragma once
#include <stdint.h>
#include <algorithm>
#include <vector>

#include "sb_frames.h"

#if defined(__CUDACC__)
#define SBW_HD __host__ __device__ __forceinline__
#else
#define SBW_HD inline
#endif

namespace sbwv {

constexpr int kMaxTerms = 16;
constexpr int kTermWords = 19;                       // packed value / delta, weight A, weight B, 8 + 8 history
constexpr int kMaxBlockSamples = 150000;             // FFmpeg's WV_MAX_SAMPLES

// block header flags
constexpr uint32_t kMono = 0x4, kHybrid = 0x8, kJoint = 0x10, kFloat = 0x80, kInitial = 0x800, kFinal = 0x1000,
                   kFalseStereo = 0x40000000u, kDsd = 0x80000000u;

// metadata sub-block ids (id & 0x3f)
enum {
    kIdTerms = 2, kIdWeights = 3, kIdSamples = 4, kIdEntropy = 5, kIdInt32 = 9, kIdBitstream = 10, kIdWvx = 12,
    kIdChannels = 13, kIdRate = 0x27,
};

enum {
    kOk = 0,
    kUnsupported,        // flags: 1- or 4-byte samples, hybrid, float or DSD
    kSubblockOverrun,    // a metadata sub-block runs past its block
    kNoBitstream,        // samples but no ID_WV_BITSTREAM
    kMissingState,       // a bitstream without terms, weights, sample history or entropy medians
    kTooManyTerms,       // more than 16 decorrelation terms
    kBadTerm,            // a term other than 1-8, 17, 18 (or -1, -2, -3 in a stereo block)
    kBadWeights,         // weights before terms, more weights than terms, or a size that splits a weight pair
    kBadHistory,         // sample history before terms, or a size that does not end at a term's end
    kBadEntropy,         // entropy medians of the wrong size
    kBadInt32,           // ID_INT32_INFO of the wrong size, or a shift above 31
    kWideInt32,          // ID_INT32_INFO with sent bits: an extended-precision stream
    kWvx,                // ID_WVX_BITSTREAM: an extended-precision stream
    kBadRate,            // ID_SAMPLE_RATE of the wrong size
    kBadShift,           // the header's shift puts the sample above 32 bits
    kBitstream,          // the bitstream reads past its sub-block, or codes a residual of 2^25 or more
    kTooLarge,           // a 16-bit stereo sample pair of magnitude above 2^19
    kCrc,                // the block CRC disagrees
    kMonoNoTerms,        // a mono block without decorrelation terms, which FFmpeg decodes as silence
};

SBW_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kUnsupported: return "unsupported block flags (hybrid, float, DSD, or 1- or 4-byte samples)";
    case kSubblockOverrun: return "metadata sub-block runs past its block";
    case kNoBitstream: return "block with samples but no ID_WV_BITSTREAM";
    case kMissingState: return "bitstream without decorrelation terms, weights, samples or entropy medians";
    case kTooManyTerms: return "more than 16 decorrelation terms";
    case kBadTerm: return "invalid decorrelation term";
    case kBadWeights: return "invalid decorrelation weights";
    case kBadHistory: return "invalid decorrelation samples";
    case kBadEntropy: return "invalid entropy medians";
    case kBadInt32: return "invalid ID_INT32_INFO";
    case kWideInt32: return "ID_INT32_INFO with sent bits (extended precision) is not supported";
    case kWvx: return "ID_WVX_BITSTREAM (extended precision) is not supported";
    case kBadRate: return "invalid ID_SAMPLE_RATE";
    case kBadShift: return "shift above 31 bits";
    case kBitstream: return "bitstream reads past its sub-block";
    case kTooLarge: return "16-bit stereo sample too large";
    case kCrc: return "CRC mismatch";
    case kMonoNoTerms: return "mono block without decorrelation terms (FFmpeg decodes it as silence)";
    default: return "unknown error";
    }
}

// what the host hands k_wavpack_decode per block (sb_wavpack_decode_blocks' table row)
struct Block {
    int64_t offset, size;      // the block's sub-blocks: bytes [offset, offset + size) of the buffer
    int64_t sample;            // first sample of the block in the track
    uint32_t flags, crc;
    int32_t samples;           // block_samples
    int32_t channel;           // first output channel
};

#define SBW_EXP2_TABLE                                                                                                 \
    0x00, 0x01, 0x01, 0x02, 0x03, 0x03, 0x04, 0x05, 0x06, 0x06, 0x07, 0x08, 0x08, 0x09, 0x0a, 0x0b, 0x0b, 0x0c, 0x0d,  \
    0x0e, 0x0e, 0x0f, 0x10, 0x10, 0x11, 0x12, 0x13, 0x13, 0x14, 0x15, 0x16, 0x16, 0x17, 0x18, 0x19, 0x19, 0x1a, 0x1b,  \
    0x1c, 0x1d, 0x1d, 0x1e, 0x1f, 0x20, 0x20, 0x21, 0x22, 0x23, 0x24, 0x24, 0x25, 0x26, 0x27, 0x28, 0x28, 0x29, 0x2a,  \
    0x2b, 0x2c, 0x2c, 0x2d, 0x2e, 0x2f, 0x30, 0x30, 0x31, 0x32, 0x33, 0x34, 0x35, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,  \
    0x3a, 0x3b, 0x3c, 0x3d, 0x3e, 0x3f, 0x40, 0x41, 0x41, 0x42, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x48, 0x49, 0x4a,  \
    0x4b, 0x4c, 0x4d, 0x4e, 0x4f, 0x50, 0x51, 0x51, 0x52, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x5b, 0x5c,  \
    0x5d, 0x5e, 0x5e, 0x5f, 0x60, 0x61, 0x62, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x6b, 0x6c, 0x6d, 0x6e,  \
    0x6f, 0x70, 0x71, 0x72, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x7b, 0x7c, 0x7d, 0x7e, 0x7f, 0x80, 0x81,  \
    0x82, 0x83, 0x84, 0x85, 0x87, 0x88, 0x89, 0x8a, 0x8b, 0x8c, 0x8d, 0x8e, 0x8f, 0x90, 0x91, 0x92, 0x93, 0x95, 0x96,  \
    0x97, 0x98, 0x99, 0x9a, 0x9b, 0x9c, 0x9d, 0x9f, 0xa0, 0xa1, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa8, 0xa9, 0xaa, 0xab,  \
    0xac, 0xad, 0xaf, 0xb0, 0xb1, 0xb2, 0xb3, 0xb4, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xbc, 0xbd, 0xbe, 0xbf, 0xc0, 0xc2,  \
    0xc3, 0xc4, 0xc5, 0xc6, 0xc8, 0xc9, 0xca, 0xcb, 0xcd, 0xce, 0xcf, 0xd0, 0xd2, 0xd3, 0xd4, 0xd6, 0xd7, 0xd8, 0xd9,  \
    0xdb, 0xdc, 0xdd, 0xde, 0xe0, 0xe1, 0xe2, 0xe4, 0xe5, 0xe6, 0xe8, 0xe9, 0xea, 0xec, 0xed, 0xee, 0xf0, 0xf1, 0xf2,  \
    0xf4, 0xf5, 0xf6, 0xf8, 0xf9, 0xfa, 0xfc, 0xfd, 0xff

// round(256 * 2^(i / 256)) - 256: FFmpeg's wp_exp2_table
#if defined(__CUDACC__)
__constant__ uint8_t kExp2Device[256] = {SBW_EXP2_TABLE};
#endif
static const uint8_t kExp2Host[256] = {SBW_EXP2_TABLE};

SBW_HD int exp2_entry(int i) {
#if defined(__CUDA_ARCH__)
    return kExp2Device[i];
#else
    return kExp2Host[i];
#endif
}

// FFmpeg's wp_exp2: a stored 16-bit log back to a value (sample history, medians)
SBW_HD int32_t wp_exp2(int v) {
    v = (int16_t)v;
    const bool neg = v < 0;
    if (neg) v = -v;
    uint32_t res = (uint32_t)exp2_entry(v & 0xff) | 0x100u;
    v >>= 8;
    if (v > 31) return (int32_t)0x80000000u;
    res = v > 9 ? res << (v - 9) : res >> (9 - v);
    return neg ? (int32_t)(0u - res) : (int32_t)res;
}

SBW_HD int ctz64(uint64_t v) {
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)v) - 1;
#else
    return __builtin_ctzll(v);
#endif
}

SBW_HD int log2_floor(uint32_t v) {          // av_log2 (0 for 0)
#if defined(__CUDA_ARCH__)
    return v ? 31 - __clz((int)v) : 0;
#else
    return v ? 31 - __builtin_clz(v) : 0;
#endif
}

// LSB-first bit reader over bits [pos, end)
struct Bits {
    const uint8_t* p;
    int64_t pos, end;
    SBW_HD uint64_t peek() const {             // at least 33 valid bits, zeros above the 5 bytes fetched
        const uint8_t* q = p + (pos >> 3);
        const uint64_t v = (uint64_t)q[0] | ((uint64_t)q[1] << 8) | ((uint64_t)q[2] << 16) | ((uint64_t)q[3] << 24) |
                           ((uint64_t)q[4] << 32);
        return v >> (pos & 7);
    }
    SBW_HD uint32_t read(int n) {              // 0 <= n <= 32
        if (n == 0) return 0;
        const uint32_t v = (uint32_t)(peek() & (0xffffffffull >> (32 - n)));
        pos += n;
        return v;
    }
    SBW_HD int unary33() {                     // get_unary_0_33: ones up to a zero (consumed) or 33 ones
        const int ones = ctz64(~peek());
        if (ones >= 33) { pos += 33; return 33; }
        pos += ones + 1;
        return ones;
    }
    SBW_HD int64_t left() const { return end - pos; }
};

// the entropy decoder's state: three medians per channel, the zero-run count and the held one / zero
struct Entropy {
    int32_t med[2][3];
    int32_t zeroes;
    int one, zero;
};

SBW_HD uint32_t get_med(const int32_t* m, int n) { return (uint32_t)((m[n] >> 4) + 1); }
SBW_HD void dec_med(int32_t* m, int n) {
    m[n] = (int32_t)((uint32_t)m[n] - (uint32_t)((int32_t)((uint32_t)m[n] + (128u >> n) - 2) / (128 >> n)) * 2u);
}
SBW_HD void inc_med(int32_t* m, int n) {
    m[n] = (int32_t)((uint32_t)m[n] + (uint32_t)((int32_t)((uint32_t)m[n] + (128u >> n)) / (128 >> n)) * 5u);
}

// FFmpeg's get_tail: a value in [0, k] in the shortest prefix-free code
SBW_HD uint32_t get_tail(Bits& b, uint32_t k) {
    if (k < 1) return 0;
    const int p = log2_floor(k);
    const uint32_t e = (uint32_t)((1ull << (p + 1)) - k - 1);
    uint32_t res = b.read(p);
    if (res >= e) res = (res << 1) - e + b.read(1);
    return res;
}

// FFmpeg's wv_get_value for channel ch; false when the bitstream is exhausted or damaged
SBW_HD bool get_value(Bits& b, Entropy& e, int ch, int32_t* out) {
    int32_t* m = e.med[ch];
    *out = 0;
    if ((uint32_t)e.med[0][0] < 2u && (uint32_t)e.med[1][0] < 2u && !e.zero && !e.one) {
        if (e.zeroes) {
            if (--e.zeroes) return true;
        } else {
            int t = b.unary33();
            if (t >= 2) {
                if (t >= 32 || b.left() < t - 1) return false;
                t = (int)(b.read(t - 1) | (1u << (t - 1)));
            } else if (b.left() < 0) {
                return false;
            }
            e.zeroes = t;
            if (e.zeroes) {
                for (int c = 0; c < 2; ++c)
                    for (int i = 0; i < 3; ++i) e.med[c][i] = 0;
                return true;
            }
        }
    }
    int t;
    if (e.zero) {
        t = 0;
        e.zero = 0;
    } else {
        t = b.unary33();
        if (b.left() < 0) return false;
        if (t == 16) {
            const int t2 = b.unary33();
            if (t2 < 2) {
                if (b.left() < 0) return false;
                t += t2;
            } else {
                if (t2 >= 32 || b.left() < t2 - 1) return false;
                t += (int)(b.read(t2 - 1) | (1u << (t2 - 1)));
            }
        }
        if (e.one) {
            e.one = t & 1;
            t = (t >> 1) + 1;
        } else {
            e.one = t & 1;
            t >>= 1;
        }
        e.zero = !e.one;
    }
    uint32_t base, add;
    if (t == 0) {
        base = 0;
        add = get_med(m, 0) - 1;
        dec_med(m, 0);
    } else if (t == 1) {
        base = get_med(m, 0);
        add = get_med(m, 1) - 1;
        inc_med(m, 0);
        dec_med(m, 1);
    } else {
        base = get_med(m, 0) + get_med(m, 1) + get_med(m, 2) * (uint32_t)(t - 2);
        add = get_med(m, 2) - 1;
        inc_med(m, 0);
        inc_med(m, 1);
        if (t == 2) dec_med(m, 2);
        else inc_med(m, 2);
    }
    if (add >= 0x2000000u) return false;
    const uint32_t ret = base + get_tail(b, add);
    if (b.left() <= 0) return false;
    *out = b.read(1) ? (int32_t)~ret : (int32_t)ret;
    return true;
}

// the block's per-term state: field f of term k
struct Terms {
    int32_t* p;
    int stride;
    SBW_HD int32_t& at(int k, int f) const { return p[(k * kTermWords + f) * stride]; }
    SBW_HD int value(int k) const { return (int)(int8_t)(at(k, 0) & 0xff); }
    SBW_HD int delta(int k) const { return at(k, 0) >> 8; }
    SBW_HD int32_t& weight(int k, int side) const { return at(k, 1 + side); }
    SBW_HD int32_t& hist(int k, int side, int j) const { return at(k, 3 + 8 * side + j); }
};

SBW_HD int32_t apply_weight(int32_t w, int32_t a, bool wide) {
    if (wide) return (int32_t)(((int64_t)w * a + 512) >> 10);
    return (int32_t)((uint32_t)w * (uint32_t)a + 512u) >> 10;
}

SBW_HD void update_weight_clip(int32_t& w, int delta, int32_t s, int32_t in) {
    if (s && in) {
        if ((s ^ in) < 0) {
            w -= delta;
            if (w < -1024) w = -1024;
        } else {
            w += delta;
            if (w > 1024) w = 1024;
        }
    }
}

// FFmpeg's wv_get_value_integer (ID_INT32_INFO's zeros, ones or duplicates, then the header's shift), kept as the
// top 16 bits of FFmpeg's S32 sample for 3-byte streams and as FFmpeg's S16 sample for 2-byte ones
SBW_HD int16_t store(int32_t s, uint32_t and_mask, uint32_t or_mask, int ishift, int post_shift, bool wide) {
    const uint32_t bit = ((uint32_t)s & and_mask) | or_mask;
    const uint32_t v = ((((uint32_t)s + bit) << ishift) - bit) << post_shift;
    return wide ? (int16_t)(v >> 16) : (int16_t)v;
}

// One block: its sub-blocks, then block.samples samples (two channels unless mono) into out, the track's interleaved
// int16 PCM of `channels` channels.  ts holds the state of 16 terms.
SBW_HD int decode_block(const uint8_t* buf, const Block& blk, int channels, const Terms& ts, int16_t* out) {
    const uint32_t flags = blk.flags;
    const int bytes = (int)(flags & 3) + 1;
    if ((bytes != 2 && bytes != 3) || (flags & (kHybrid | kFloat | kDsd))) return kUnsupported;
    const bool wide = bytes == 3;                          // FFmpeg's S32P: 64-bit weight products
    const bool stereo = !(flags & kMono);
    const int stereo_in = (flags & kFalseStereo) ? 0 : (stereo ? 1 : 0);
    const int post_shift = (wide ? 8 : 0) + (int)((flags >> 13) & 0x1f);
    if (post_shift > 31) return kBadShift;

    int terms = 0;
    bool got_terms = false, got_weights = false, got_samples = false, got_entropy = false, got_bits = false;
    Entropy ent;
    for (int c = 0; c < 2; ++c)
        for (int i = 0; i < 3; ++i) ent.med[c][i] = 0;
    ent.zeroes = 0; ent.one = 0; ent.zero = 0;
    uint32_t and_mask = 0, or_mask = 0;
    int ishift = 0;
    Bits b; b.p = buf; b.pos = 0; b.end = 0;
    for (int k = 0; k < kMaxTerms; ++k)
        for (int f = 0; f < kTermWords; ++f) ts.at(k, f) = 0;

    int64_t pos = blk.offset;
    const int64_t end = blk.offset + blk.size;
    while (pos < end) {
        if (end - pos < 2) return kSubblockOverrun;
        const int id = buf[pos];
        int64_t words = buf[pos + 1];
        pos += 2;
        if (id & 0x80) {
            if (end - pos < 2) return kSubblockOverrun;
            words |= ((int64_t)buf[pos] | ((int64_t)buf[pos + 1] << 8)) << 8;
            pos += 2;
        }
        const int64_t ssize = words * 2;
        const int64_t size = ssize - ((id & 0x40) ? 1 : 0);
        if (size < 0 || end - pos < ssize) return kSubblockOverrun;
        const uint8_t* d = buf + pos;
        switch (id & 0x3f) {
        case kIdTerms:
            if (size > kMaxTerms) return kTooManyTerms;
            terms = (int)size;
            for (int i = 0; i < terms; ++i) {
                const int v = (d[i] & 0x1f) - 5;
                const bool ok = (v >= 1 && v <= 8) || v == 17 || v == 18 || (stereo_in && v >= -3 && v <= -1);
                if (!ok) return kBadTerm;
                ts.at(terms - i - 1, 0) = (v & 0xff) | ((d[i] >> 5) << 8);
            }
            got_terms = true;
            break;
        case kIdWeights: {
            const int64_t n = size >> stereo_in;
            if (!got_terms || n > terms || (n << stereo_in) != size) return kBadWeights;
            for (int i = 0; i < (int)n; ++i)
                for (int s = 0; s <= stereo_in; ++s) {
                    int32_t w = (int32_t)(int8_t)d[i * (stereo_in + 1) + s] * 8;
                    if (w > 0) w += (w + 64) >> 7;
                    ts.weight(terms - i - 1, s) = w;
                }
            got_weights = true;
            break;
        }
        case kIdSamples: {
            if (!got_terms) return kBadHistory;
            int64_t t = 0;
            auto le16 = [&](int64_t at) { return (int)d[at] | ((int)d[at + 1] << 8); };
            for (int i = terms - 1; i >= 0 && t < size; --i) {
                const int v = ts.value(i);
                const int64_t need = v > 8 ? 4 * (stereo_in + 1) : (v < 0 ? 4 : 2 * v * (stereo_in + 1));
                if (t + need > size) return kBadHistory;
                if (v > 8) {                                   // A[0], A[1], then B[0], B[1]
                    for (int s = 0; s <= stereo_in; ++s)
                        for (int j = 0; j < 2; ++j) ts.hist(i, s, j) = wp_exp2(le16(t + 4 * s + 2 * j));
                } else if (v < 0) {                            // A[0], B[0]
                    ts.hist(i, 0, 0) = wp_exp2(le16(t));
                    ts.hist(i, 1, 0) = wp_exp2(le16(t + 2));
                } else {                                       // A[j] (and B[j]) for j < v
                    for (int j = 0; j < v; ++j)
                        for (int s = 0; s <= stereo_in; ++s)
                            ts.hist(i, s, j) = wp_exp2(le16(t + 2 * (j * (stereo_in + 1) + s)));
                }
                t += need;
            }
            if (t != size) return kBadHistory;
            got_samples = true;
            break;
        }
        case kIdEntropy:
            if (size != 6 * (stereo_in + 1)) return kBadEntropy;
            for (int c = 0; c <= stereo_in; ++c)
                for (int i = 0; i < 3; ++i) ent.med[c][i] = wp_exp2(d[6 * c + 2 * i] | (d[6 * c + 2 * i + 1] << 8));
            got_entropy = true;
            break;
        case kIdInt32:
            if (size != 4) return kBadInt32;
            if (d[0]) return kWideInt32;
            if (d[1]) ishift = d[1];
            else if (d[2]) { and_mask = or_mask = 1; ishift = d[2]; }
            else if (d[3]) { and_mask = 1; ishift = d[3]; }
            if (ishift > 31) return kBadInt32;
            break;
        case kIdBitstream:
            b.pos = pos * 8;
            b.end = (pos + size) * 8;
            got_bits = true;
            break;
        case kIdWvx:
            return kWvx;
        case kIdRate:
            if (size != 3) return kBadRate;
            break;
        default:                                           // ID_CHANNEL_INFO, RIFF chunks, MD5, unknown: skipped
            break;
        }
        pos += ssize;
    }
    if (!got_bits) return kNoBitstream;
    if (!got_terms || !got_weights || !got_samples || !got_entropy) return kMissingState;
    if (!stereo_in && terms == 0) return kMonoNoTerms;

    uint32_t crc = 0xffffffffu;
    int hp = 0;                                            // history position of terms 1-8
    const int ch0 = blk.channel;
    for (int64_t n = 0; n < blk.samples; ++n) {
        int16_t* o = out + (blk.sample + n) * channels + ch0;
        if (stereo_in) {
            int32_t L, R;
            if (!get_value(b, ent, 0, &L) || !get_value(b, ent, 1, &R)) return kBitstream;
            for (int i = 0; i < terms; ++i) {
                const int t = ts.value(i);
                const int delta = ts.delta(i);
                int32_t& wA = ts.weight(i, 0);
                int32_t& wB = ts.weight(i, 1);
                if (t > 0) {
                    int32_t A, B;
                    int j;
                    if (t > 8) {
                        const int32_t a0 = ts.hist(i, 0, 0), a1 = ts.hist(i, 0, 1);
                        const int32_t b0 = ts.hist(i, 1, 0), b1 = ts.hist(i, 1, 1);
                        if (t & 1) {
                            A = (int32_t)(2u * (uint32_t)a0 - (uint32_t)a1);
                            B = (int32_t)(2u * (uint32_t)b0 - (uint32_t)b1);
                        } else {
                            A = (int32_t)(3u * (uint32_t)a0 - (uint32_t)a1) >> 1;
                            B = (int32_t)(3u * (uint32_t)b0 - (uint32_t)b1) >> 1;
                        }
                        ts.hist(i, 0, 1) = a0;
                        ts.hist(i, 1, 1) = b0;
                        j = 0;
                    } else {
                        A = ts.hist(i, 0, hp);
                        B = ts.hist(i, 1, hp);
                        j = (hp + t) & 7;
                    }
                    const int32_t L2 = (int32_t)((uint32_t)L + (uint32_t)apply_weight(wA, A, wide));
                    const int32_t R2 = (int32_t)((uint32_t)R + (uint32_t)apply_weight(wB, B, wide));
                    if (A && L) wA -= ((((L ^ A) >> 30) & 2) - 1) * delta;
                    if (B && R) wB -= ((((R ^ B) >> 30) & 2) - 1) * delta;
                    ts.hist(i, 0, j) = L = L2;
                    ts.hist(i, 1, j) = R = R2;
                } else if (t == -1) {
                    const int32_t a0 = ts.hist(i, 0, 0);
                    const int32_t L2 = (int32_t)((uint32_t)L + (uint32_t)apply_weight(wA, a0, wide));
                    update_weight_clip(wA, delta, a0, L);
                    L = L2;
                    const int32_t R2 = (int32_t)((uint32_t)R + (uint32_t)apply_weight(wB, L2, wide));
                    update_weight_clip(wB, delta, L2, R);
                    R = R2;
                    ts.hist(i, 0, 0) = R;
                } else {
                    const int32_t b0 = ts.hist(i, 1, 0);
                    int32_t R2 = (int32_t)((uint32_t)R + (uint32_t)apply_weight(wB, b0, wide));
                    update_weight_clip(wB, delta, b0, R);
                    R = R2;
                    if (t == -3) {
                        R2 = ts.hist(i, 0, 0);
                        ts.hist(i, 0, 0) = R;
                    }
                    const int32_t L2 = (int32_t)((uint32_t)L + (uint32_t)apply_weight(wA, R2, wide));
                    update_weight_clip(wA, delta, R2, L);
                    L = L2;
                    ts.hist(i, 1, 0) = L;
                }
            }
            if (!wide) {
                const int64_t al = L < 0 ? -(int64_t)L : L, ar = R < 0 ? -(int64_t)R : R;
                if (al + ar > (1 << 19)) return kTooLarge;
            }
            hp = (hp + 1) & 7;
            if (flags & kJoint) {
                R = (int32_t)((uint32_t)R - (uint32_t)(L >> 1));
                L = (int32_t)((uint32_t)L + (uint32_t)R);
            }
            crc = (crc * 3u + (uint32_t)L) * 3u + (uint32_t)R;
            o[0] = store(L, and_mask, or_mask, ishift, post_shift, wide);
            o[1] = store(R, and_mask, or_mask, ishift, post_shift, wide);
        } else {
            int32_t T;
            if (!get_value(b, ent, 0, &T)) return kBitstream;
            int32_t S = 0;
            for (int i = 0; i < terms; ++i) {
                const int t = ts.value(i);
                int32_t& wA = ts.weight(i, 0);
                int32_t A;
                int j;
                if (t > 8) {
                    const int32_t a0 = ts.hist(i, 0, 0), a1 = ts.hist(i, 0, 1);
                    A = (t & 1) ? (int32_t)(2u * (uint32_t)a0 - (uint32_t)a1)
                                : (int32_t)(3u * (uint32_t)a0 - (uint32_t)a1) >> 1;
                    ts.hist(i, 0, 1) = a0;
                    j = 0;
                } else {
                    A = ts.hist(i, 0, hp);
                    j = (hp + t) & 7;
                }
                S = (int32_t)((uint32_t)T + (uint32_t)apply_weight(wA, A, wide));
                if (A && T) wA -= ((((T ^ A) >> 30) & 2) - 1) * ts.delta(i);
                ts.hist(i, 0, j) = T = S;
            }
            hp = (hp + 1) & 7;
            crc = crc * 3u + (uint32_t)S;
            o[0] = store(S, and_mask, or_mask, ishift, post_shift, wide);
            if (stereo) o[1] = o[0];
        }
    }
    if (crc != blk.crc) return kCrc;
    return kOk;
}

// ---- host side: what sb_wavpack_decode_blocks does around the kernel; the CPU build of the tests runs the same ----

// The kernel's blocks from the caller's table (8 int64 per block: offset, size, samples, flags, crc, sample position,
// first channel, file offset): a block must lie inside the buffer, hold 1 to kMaxBlockSamples samples and write
// channels the track has.  *samples: where the last block ends.  Returns false with a message naming the row's file
// offset.
inline bool block_table(const int64_t* table, int64_t n, int64_t nbytes, int channels, std::vector<Block>& blocks,
                        int64_t* samples, char* msg, size_t msg_len) {
    blocks.resize((size_t)n);
    *samples = 0;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t* r = table + 8 * i;
        Block& b = blocks[(size_t)i];
        b.offset = r[0]; b.size = r[1]; b.samples = (int32_t)r[2]; b.flags = (uint32_t)r[3]; b.crc = (uint32_t)r[4];
        b.sample = r[5]; b.channel = (int32_t)r[6];
        const int width = (b.flags & kMono) ? 1 : 2;
        if (r[0] < 0 || r[1] < 0 || r[0] > nbytes - r[1] || r[2] < 1 || r[2] > kMaxBlockSamples || r[5] < 0 ||
            r[6] < 0 || r[6] + width > channels)
            return sbframes::refuse(msg, msg_len, "WavPack block", i, r[7], "block table entry out of range");
        *samples = std::max(*samples, r[5] + r[2]);
    }
    return true;
}

}  // namespace sbwv
