// MPEG-1/2 audio layer II (MP2) decoding, written once for the kernels of sb_mp2.cu and for the CPU
// (tests/emu/emu_mp2_driver.cpp compiles this header with g++).  The arithmetic is that of FFmpeg's fixed-point `mp2`
// decoder, the one `avcodec_find_decoder` returns for MP2, operation for operation: 23 fractional bits for the subband
// samples, a 16-bit window, 64-bit sums and the rounding remainder of every output carried into the next one.
//
// The decode splits where the data does:
//   frame table   the host walks the headers (frame_table): every frame's offset, size and header; the stream's layer,
//                 rate and channel count may not change, its bitrate may
//   unpack        one thread per frame: bit allocation, SCFSI, scalefactors, the grouped and plain samples and their
//                 requantisation (unpack_frame), the CRC-16 when the frame has one; 36 x 32 subband samples per
//                 channel into scratch
//   matrixing     one thread per time slot of a channel: FFmpeg's fixed-point 32-point DCT (dct32) in place, giving the
//                 32 values of the synthesis buffer that slot adds
//   window        one warp per time slot of a channel: the 512-tap window over the slot and the 15 before it
//                 (window_sum), exact in 64 bits.  FFmpeg's output of each sample is (remainder + sum) >> 24, and the
//                 new remainder the low 24 bits: so the remainder before any output is the running sum of every
//                 earlier window sum, modulo 2^24, in FFmpeg's emission order (frame, then channel, then slot, then
//                 the samples 0, 1, 31, 2, 30, ..., 15, 17, 16 of a slot).  An exclusive scan of the low 24 bits of the
//                 sums gives every remainder at once.
//
// The tables are the standard's (ISO/IEC 11172-3 annex B, ISO/IEC 13818-3 annex B): the bit-allocation tables, the
// quantiser classes, the scalefactors 2^(1 - i/3), the 512-tap synthesis window D[i] in units of 2^-16, and the DCT's
// butterfly constants 1 / (2 cos((2i + 1) pi / 2^(6 - j))) in units of 2^-32.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <vector>

#include "sb_frames.h"

#if defined(__CUDACC__)
#define SBM_HD __host__ __device__ __forceinline__
#define SBM_UNROLL _Pragma("unroll")
#define SBM_CONST __constant__
#else
#define SBM_HD inline
#define SBM_UNROLL
#define SBM_CONST
#endif
// A table in constant memory for the kernels and in host memory for the host, read as SBM_T(name) from either
#define SBM_TABLE(type, name, dims, ...) \
    SBM_CONST static const type name##_d dims = __VA_ARGS__; \
    static const type name##_h dims = __VA_ARGS__;
#if defined(__CUDA_ARCH__)
#define SBM_T(name) name##_d
#else
#define SBM_T(name) name##_h
#endif

namespace sbmp2 {

constexpr int kSb = 32;                  // subbands
constexpr int kSlots = 36;               // time slots per frame and channel
constexpr int kFrameSamples = kSb * kSlots;
constexpr int kOutShift = 24;            // FFmpeg's OUT_SHIFT: 16 window bits + 23 sample bits - 15
constexpr int kFracBits = 23;

// ---- tables ----

// kbit/s by [lsf][bitrate index] (layer II)
SBM_TABLE(int16_t, kBitrate, [2][15], {
    {0, 32, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, 384},
    {0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160},
})
SBM_TABLE(int32_t, kRate, [3], {44100, 48000, 32000})

// Quantiser classes: the levels of each, and the bits of one code (negative: three samples grouped in one code)
SBM_TABLE(int32_t, kSteps, [17], {3, 5, 7, 9, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 16383,
                                            32767, 65535})
SBM_TABLE(int8_t, kQuantBits, [17], {-5, -7, 3, -10, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16})

// The five bit-allocation tables: per subband, the allocation's bit count (nbal), then the quantiser class of each
// allocation 1 .. 2^nbal - 1 (11172-3 tables B.2a-d, 13818-3 table B.1).  A subband's entry takes 2^nbal bytes.
constexpr int kTables = 5;
SBM_TABLE(uint8_t, kSblimit, [kTables], {27, 30, 8, 12, 30})
#define SBM_A4 4, 0, 2, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16
#define SBM_B4 4, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 16
#define SBM_C3 3, 0, 1, 2, 3, 4, 5, 16
#define SBM_D2 2, 0, 1, 16
#define SBM_E4 4, 0, 1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15
#define SBM_F3 3, 0, 1, 3, 4, 5, 6, 7
#define SBM_G4 4, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14
#define SBM_H2 2, 0, 1, 3
// tables a and b: 3 subbands of A4, 8 of B4, 12 of C3, then D2 up to the limit (27, 30)
SBM_TABLE(uint8_t, kAllocAB, [], {
    SBM_A4, SBM_A4, SBM_A4,
    SBM_B4, SBM_B4, SBM_B4, SBM_B4, SBM_B4, SBM_B4, SBM_B4, SBM_B4,
    SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3, SBM_C3,
    SBM_D2, SBM_D2, SBM_D2, SBM_D2, SBM_D2, SBM_D2, SBM_D2,
})
// tables c and d: 2 subbands of E4, then F3 up to the limit (8, 12)
SBM_TABLE(uint8_t, kAllocCD, [], {
    SBM_E4, SBM_E4,
    SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3,
})
// MPEG-2 LSF: 4 subbands of G4, 7 of F3, 19 of H2
SBM_TABLE(uint8_t, kAllocLsf, [], {
    SBM_G4, SBM_G4, SBM_G4, SBM_G4,
    SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3, SBM_F3,
    SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2,
    SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2, SBM_H2,
})
#undef SBM_A4
#undef SBM_B4
#undef SBM_C3
#undef SBM_D2
#undef SBM_E4
#undef SBM_F3
#undef SBM_G4
#undef SBM_H2

SBM_HD const uint8_t* alloc_table(int table) {
    return table == 4 ? SBM_T(kAllocLsf) : table >= 2 ? SBM_T(kAllocCD) : SBM_T(kAllocAB);
}

// The synthesis window D[0..256] of 11172-3 table B.3, times 2^16 and rounded; D[512 - i] is -D[i] but where i is a
// multiple of 64 (window_at)
SBM_TABLE(int32_t, kWindow, [257], {
     0,    -1,    -1,    -1,    -1,    -1,    -1,    -2,    -2,    -2,    -2,    -3,    -3,    -4,    -4,    -5,
    -5,    -6,    -7,    -7,    -8,    -9,   -10,   -11,   -13,   -14,   -16,   -17,   -19,   -21,   -24,   -26,
   -29,   -31,   -35,   -38,   -41,   -45,   -49,   -53,   -58,   -63,   -68,   -73,   -79,   -85,   -91,   -97,
  -104,  -111,  -117,  -125,  -132,  -139,  -147,  -154,  -161,  -169,  -176,  -183,  -190,  -196,  -202,  -208,
   213,   218,   222,   225,   227,   228,   228,   227,   224,   221,   215,   208,   200,   189,   177,   163,
   146,   127,   106,    83,    57,    29,    -2,   -36,   -72,  -111,  -153,  -197,  -244,  -294,  -347,  -401,
  -459,  -519,  -581,  -645,  -711,  -779,  -848,  -919,  -991, -1064, -1137, -1210, -1283, -1356, -1428, -1498,
 -1567, -1634, -1698, -1759, -1817, -1870, -1919, -1962, -2001, -2032, -2057, -2075, -2085, -2087, -2080, -2063,
  2037,  2000,  1952,  1893,  1822,  1739,  1644,  1535,  1414,  1280,  1131,   970,   794,   605,   402,   185,
   -45,  -288,  -545,  -814, -1095, -1388, -1692, -2006, -2330, -2663, -3004, -3351, -3705, -4063, -4425, -4788,
 -5153, -5517, -5879, -6237, -6589, -6935, -7271, -7597, -7910, -8209, -8491, -8755, -8998, -9219, -9416, -9585,
 -9727, -9838, -9916, -9959, -9966, -9935, -9863, -9750, -9592, -9389, -9139, -8840, -8492, -8092, -7640, -7134,
  6574,  5959,  5288,  4561,  3776,  2935,  2037,  1082,    70,  -998, -2122, -3300, -4533, -5818, -7154, -8540,
 -9975,-11455,-12980,-14548,-16155,-17799,-19478,-21189,-22929,-24694,-26482,-28289,-30112,-31947,-33791,-35640,
-37489,-39336,-41176,-43006,-44821,-46617,-48390,-50137,-51853,-53534,-55178,-56778,-58333,-59838,-61289,-62684,
-64019,-65290,-66494,-67629,-68692,-69679,-70590,-71420,-72169,-72835,-73415,-73908,-74313,-74630,-74856,-74992,
 75038,
})

SBM_HD int32_t window_at(int i) {        // 0 <= i < 512
    if (i <= 256) return SBM_T(kWindow)[i];
    const int32_t v = SBM_T(kWindow)[512 - i];
    return (i & 63) ? -v : v;
}

// The DCT's butterfly constants round(2^32 / (2 cos((2i + 1) pi / 2^(6 - j))) / 2^s), s the butterfly's shift
// (tests/test_mp2_cases.py recomputes them): pass j = 0 (16 of them), 1 (8), 2 (4), 3 (2), and 1/sqrt(2) / 2
SBM_TABLE(int32_t, kCos0, [16], {
    1075036753, 1085490621, 1106914669, 1140405281, 1187781572, 1251843312, 1336817425, 1449139879,
    1598879467, 1802489638, 2088574387, 1255676567, 1593609622, 1104762768, 1829445839, 1367679739})
SBM_TABLE(int32_t, kCos1, [8], {
    1078937202, 1122057232, 1217503044, 1389039203, 1692549166, 1138893993, 1849463489, 1369329156})
SBM_TABLE(int32_t, kCos2, [4], {1094777670, 1291378312, 1932684223, 1375954754})
SBM_TABLE(int32_t, kCos3, [2], {1162209775, 1402911301})
constexpr int32_t kCos4 = 1518500250;

// the scalefactor multipliers: FFmpeg's scale_factor_mult (plain classes of 3 to 16 bits, [bits - 2][i % 3]) and
// scale_factor_mult2 (grouped classes of 3, 5 and 9 levels, [levels / 4][i % 3])
struct Scales {
    int32_t mult[15][3];
    int32_t mult2[3][3];
};

// 2^(1 - m/3) rounded to 23 fractional bits, m = 0, 1, 2
inline int32_t fixr_scale(int m, double by) {
    static const double kCube[3] = {1.0, 0.79370052598409973738, 0.62996052494743658238};
    return (int32_t)(kCube[m] * by * (1 << kFracBits) + 0.5);
}

inline Scales make_scales() {
    Scales s;
    for (int i = 0; i < 15; ++i) {
        const int n = i + 2;
        const int32_t norm = (int32_t)(((int64_t)1 << n) * ((int64_t)1 << kFracBits) / ((1 << n) - 1));
        for (int m = 0; m < 3; ++m) s.mult[i][m] = (int32_t)(((int64_t)norm * fixr_scale(m, 2.0)) >> kFracBits);
    }
    const double levels[3] = {4.0 / 3.0, 4.0 / 5.0, 4.0 / 9.0};
    for (int i = 0; i < 3; ++i)
        for (int m = 0; m < 3; ++m) s.mult2[i][m] = fixr_scale(m, levels[i]);
    return s;
}

// ---- header ----

enum {
    kOk = 0,
    kBitsPast,           // the frame's allocation, scalefactors and samples need more bits than it has
    kCrc,                // the CRC-16 over the header and the side information disagrees
};

SBM_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kBitsPast: return "the frame's samples run past its end";
    case kCrc: return "CRC-16 mismatch";
    default: return "unknown error";
    }
}

struct Header {
    int lsf, layer, rate, bitrate, padding, mode, mode_ext, channels, crc, emphasis, size, bitrate_index, rate_index;
};

// The fields of a 4-byte header h.  Returns NULL for a layer II header this decoder takes, else what it is not.
// FFmpeg's size is 144000 * kbit/s / rate + padding for layer II at both rate families.
inline const char* parse_header(uint32_t h, Header* o) {
    if ((h & 0xFFE00000u) != 0xFFE00000u) return "no frame sync";
    const int version = (h >> 19) & 3;
    if (version == 1) return "reserved MPEG version";
    if (version == 0) return "MPEG-2.5 (8 to 12 kHz), which is not decoded here";
    const int layer = 4 - (int)((h >> 17) & 3);
    if (layer == 4) return "reserved layer";
    if (layer != 2) return layer == 1 ? "layer I, which is not decoded here" : "layer III (MP3), which is not decoded here";
    o->layer = layer;
    o->lsf = version == 2;
    o->crc = !((h >> 16) & 1);
    o->bitrate_index = (h >> 12) & 15;
    if (o->bitrate_index == 15) return "reserved bitrate index";
    if (o->bitrate_index == 0) return "free-format bitrate, which is not decoded here";
    o->rate_index = (h >> 10) & 3;
    if (o->rate_index == 3) return "reserved sample-rate index";
    o->padding = (h >> 9) & 1;
    o->mode = (h >> 6) & 3;
    o->mode_ext = (h >> 4) & 3;
    o->emphasis = h & 3;
    if (o->emphasis == 2) return "reserved emphasis";
    o->channels = o->mode == 3 ? 1 : 2;
    o->rate = SBM_T(kRate)[o->rate_index] >> o->lsf;
    o->bitrate = SBM_T(kBitrate)[o->lsf][o->bitrate_index];
    o->size = o->bitrate * 144000 / o->rate + o->padding;
    return nullptr;
}

// FFmpeg's ff_mpa_l2_select_table
SBM_HD int select_table(int kbps, int channels, int rate, int lsf) {
    if (lsf) return 4;
    const int ch = kbps / channels;
    if ((rate == 48000 && ch >= 56) || (ch >= 56 && ch <= 80)) return 0;
    if (rate != 48000 && ch >= 96) return 1;
    if (rate != 32000 && ch <= 48) return 2;
    return 3;
}

// ---- per frame ----

// what the host hands the kernel per frame
struct Frame {
    int64_t offset;          // the frame's bytes, header included
    int32_t size;            // bytes present: the header's size, or what is left of a cut last frame
    uint32_t header;
    int32_t cut;             // 1 for a last frame cut short: FFmpeg decodes it with zeros for the missing bits
    int32_t pad;
};

// most-significant-bit-first reader over bytes [0, end) of p; zeros past `end`
struct Reader {
    const uint8_t* p;
    int64_t at, end;
    uint64_t cache;          // the next n bits, first in bit 63
    int n;
    int64_t pos;             // bits consumed
    SBM_HD uint32_t bits(int k) {                    // 1 <= k <= 16
        while (n < k) {
            const uint64_t b = at < end ? p[at] : 0;
            cache |= b << (56 - n);
            n += 8;
            ++at;
        }
        const uint32_t v = (uint32_t)(cache >> (64 - k));
        cache <<= k;
        n -= k;
        pos += k;
        return v;
    }
};

// CRC-16 (polynomial 0x8005, MSB first) of `count` bits of p starting at bit `from`, on top of `crc`
SBM_HD uint32_t crc16_bits(uint32_t crc, const uint8_t* p, int64_t from, int64_t count) {
    for (int64_t i = from; i < from + count; ++i) {
        const uint32_t bit = (p[i >> 3] >> (7 - (i & 7))) & 1u;
        const uint32_t top = (crc >> 15) & 1u;
        crc = (crc << 1) & 0xFFFFu;
        if (top ^ bit) crc ^= 0x8005u;
    }
    return crc;
}

// FFmpeg's l1_unscale: a plain code of n + 1 bits
SBM_HD int32_t unscale_plain(const Scales& s, int n, uint32_t mant, int sf) {
    const int shift = sf / 3 + n;
    const int64_t v = (int64_t)(int32_t)(mant - (1u << n) + 1u) * s.mult[n - 1][sf % 3];
    return (int32_t)((v + ((int64_t)1 << (shift - 1))) >> shift);
}

// FFmpeg's l2_unscale_group: one of three samples of a grouped code
SBM_HD int32_t unscale_group(const Scales& s, int steps, int mant, int sf) {
    const int shift = sf / 3;
    int32_t v = (int32_t)((uint32_t)(mant - (steps >> 1)) * (uint32_t)s.mult2[steps >> 2][sf % 3]);
    if (shift > 0) v = (v + (1 << (shift - 1))) >> shift;
    return v;
}

// Unpack frame f's subband samples: channel c's slot t at sb + ((c * n_frames + f) * kSlots + t) * kSb, subband
// order.  `buf` holds the stream; `end` the first byte the reader may not load.
SBM_HD int unpack_frame(const uint8_t* buf, int64_t end, const Frame& fr, int64_t f, int64_t n_frames, const Scales& sc,
                        int32_t* sb) {
    const uint32_t h = fr.header;
    const int lsf = ((h >> 19) & 1) ^ 1;
    const int protect = !((h >> 16) & 1);
    const int mode = (h >> 6) & 3, mode_ext = (h >> 4) & 3;
    const int channels = mode == 3 ? 1 : 2;
    const int rate = SBM_T(kRate)[(h >> 10) & 3] >> lsf;
    const int table = select_table(SBM_T(kBitrate)[lsf][(h >> 12) & 15], channels, rate, lsf);
    const int sblimit = SBM_T(kSblimit)[table];
    const uint8_t* at = alloc_table(table);
    int bound = mode == 1 ? (mode_ext + 1) * 4 : sblimit;
    if (bound > sblimit) bound = sblimit;

    Reader r;
    r.p = buf + fr.offset;
    r.at = 4;
    r.end = end - fr.offset < fr.size ? end - fr.offset : fr.size;
    r.cache = 0;
    r.n = 0;
    r.pos = 32;
    const uint32_t stored_crc = protect ? r.bits(16) : 0;

    uint8_t alloc[2][kSb], scfsi[2][kSb], sf[2][kSb][3];
    int j = 0;
    for (int i = 0; i < sblimit; ++i) {
        const int nbal = at[j];
        if (i < bound) {
            for (int c = 0; c < channels; ++c) alloc[c][i] = (uint8_t)r.bits(nbal);
        } else {
            alloc[0][i] = alloc[1][i] = (uint8_t)r.bits(nbal);
        }
        j += 1 << nbal;
    }
    for (int i = 0; i < sblimit; ++i)
        for (int c = 0; c < channels; ++c)
            if (alloc[c][i]) scfsi[c][i] = (uint8_t)r.bits(2);
    if (protect && !fr.cut) {
        // the header's last 16 bits, then the allocations and SCFSI
        uint32_t crc = crc16_bits(0xFFFFu, r.p, 16, 16);
        crc = crc16_bits(crc, r.p, 48, r.pos - 48);
        if (r.pos > (int64_t)fr.size * 8) return kBitsPast;
        if (crc != stored_crc) return kCrc;
    }
    for (int i = 0; i < sblimit; ++i)
        for (int c = 0; c < channels; ++c) {
            if (!alloc[c][i]) continue;
            uint8_t* s = sf[c][i];
            switch (scfsi[c][i]) {
            case 0: s[0] = (uint8_t)r.bits(6); s[1] = (uint8_t)r.bits(6); s[2] = (uint8_t)r.bits(6); break;
            case 1: s[0] = s[1] = (uint8_t)r.bits(6); s[2] = (uint8_t)r.bits(6); break;
            case 2: s[0] = s[1] = s[2] = (uint8_t)r.bits(6); break;
            default: s[0] = (uint8_t)r.bits(6); s[1] = s[2] = (uint8_t)r.bits(6); break;
            }
        }

    int32_t* out[2];
    for (int c = 0; c < channels; ++c) out[c] = sb + (c * n_frames + f) * (int64_t)kFrameSamples;
    for (int part = 0; part < 3; ++part)
        for (int g = 0; g < 4; ++g) {
            const int t0 = part * 12 + g * 3;
            j = 0;
            for (int i = 0; i < kSb; ++i) {
                if (i >= sblimit) {
                    for (int c = 0; c < channels; ++c)
                        for (int m = 0; m < 3; ++m) out[c][(t0 + m) * kSb + i] = 0;
                    continue;
                }
                const int nbal = at[j];
                const int shared = i >= bound;
                for (int c = 0; c < (shared ? 1 : channels); ++c) {
                    const int b = alloc[c][i];
                    int32_t v[2][3] = {{0, 0, 0}, {0, 0, 0}};
                    const int reach = shared ? channels : 1;            // channels the codes are scaled for
                    if (b) {
                        const int q = at[j + b];
                        const int bits = SBM_T(kQuantBits)[q];
                        if (bits < 0) {
                            const int steps = SBM_T(kSteps)[q];
                            uint32_t code = r.bits(-bits);
                            int mant[3];
                            mant[0] = (int)(code % (uint32_t)steps); code /= (uint32_t)steps;
                            mant[1] = (int)(code % (uint32_t)steps); code /= (uint32_t)steps;
                            mant[2] = (int)code;
                            for (int k = 0; k < reach; ++k)
                                for (int m = 0; m < 3; ++m)
                                    v[k][m] = unscale_group(sc, steps, mant[m], sf[shared ? k : c][i][part]);
                        } else {
                            for (int m = 0; m < 3; ++m) {
                                const uint32_t mant = r.bits(bits);
                                for (int k = 0; k < reach; ++k)
                                    v[k][m] = unscale_plain(sc, bits - 1, mant, sf[shared ? k : c][i][part]);
                            }
                        }
                    }
                    for (int k = 0; k < reach; ++k)
                        for (int m = 0; m < 3; ++m) out[shared ? k : c][(t0 + m) * kSb + i] = v[k][m];
                }
                j += 1 << nbal;
            }
        }
    if (r.pos > (int64_t)fr.size * 8 && !fr.cut) return kBitsPast;
    return kOk;
}

// FFmpeg's fixed-point dct32: 32 subband samples `in` to the 32 values `out` adds to the synthesis buffer (in and out
// may be the same).  Sums wrap in 32 bits; MULH3(x, c, s) is the top 32 bits of (s * x) * c.
SBM_HD int32_t mulh3(int32_t x, int32_t c, int s) {
    return (int32_t)(((int64_t)(int32_t)((uint32_t)x * (uint32_t)s) * c) >> 32);
}

SBM_HD void dct32(int32_t* out, const int32_t* in) {
    int32_t v[32];
#define SBM_ADD(a, b) (int32_t)((uint32_t)(a) + (uint32_t)(b))
#define SBM_SUB(a, b) (int32_t)((uint32_t)(a) - (uint32_t)(b))
#define BF0(a, b, c, s) { const int32_t x = in[a], y = in[b]; v[a] = SBM_ADD(x, y); v[b] = mulh3(SBM_SUB(x, y), c, 1 << (s)); }
#define BF(a, b, c, s) { const int32_t x = v[a], y = v[b]; v[a] = SBM_ADD(x, y); v[b] = mulh3(SBM_SUB(x, y), c, 1 << (s)); }
#define BF1(a, b, c, d) { BF(a, b, kCos4, 1); BF(c, d, -kCos4, 1); v[c] = SBM_ADD(v[c], v[d]); }
#define BF2(a, b, c, d) { BF(a, b, kCos4, 1); BF(c, d, -kCos4, 1); v[c] = SBM_ADD(v[c], v[d]); \
    v[a] = SBM_ADD(v[a], v[c]); v[c] = SBM_ADD(v[c], v[b]); v[b] = SBM_ADD(v[b], v[d]); }
    BF0(0, 31, SBM_T(kCos0)[0], 1); BF0(15, 16, SBM_T(kCos0)[15], 5);
    BF(0, 15, SBM_T(kCos1)[0], 1); BF(16, 31, -SBM_T(kCos1)[0], 1);
    BF0(7, 24, SBM_T(kCos0)[7], 1); BF0(8, 23, SBM_T(kCos0)[8], 1);
    BF(7, 8, SBM_T(kCos1)[7], 4); BF(23, 24, -SBM_T(kCos1)[7], 4);
    BF(0, 7, SBM_T(kCos2)[0], 1); BF(8, 15, -SBM_T(kCos2)[0], 1); BF(16, 23, SBM_T(kCos2)[0], 1); BF(24, 31, -SBM_T(kCos2)[0], 1);
    BF0(3, 28, SBM_T(kCos0)[3], 1); BF0(12, 19, SBM_T(kCos0)[12], 2);
    BF(3, 12, SBM_T(kCos1)[3], 1); BF(19, 28, -SBM_T(kCos1)[3], 1);
    BF0(4, 27, SBM_T(kCos0)[4], 1); BF0(11, 20, SBM_T(kCos0)[11], 2);
    BF(4, 11, SBM_T(kCos1)[4], 1); BF(20, 27, -SBM_T(kCos1)[4], 1);
    BF(3, 4, SBM_T(kCos2)[3], 3); BF(11, 12, -SBM_T(kCos2)[3], 3); BF(19, 20, SBM_T(kCos2)[3], 3); BF(27, 28, -SBM_T(kCos2)[3], 3);
    BF(0, 3, SBM_T(kCos3)[0], 1); BF(4, 7, -SBM_T(kCos3)[0], 1); BF(8, 11, SBM_T(kCos3)[0], 1); BF(12, 15, -SBM_T(kCos3)[0], 1);
    BF(16, 19, SBM_T(kCos3)[0], 1); BF(20, 23, -SBM_T(kCos3)[0], 1); BF(24, 27, SBM_T(kCos3)[0], 1); BF(28, 31, -SBM_T(kCos3)[0], 1);
    BF0(1, 30, SBM_T(kCos0)[1], 1); BF0(14, 17, SBM_T(kCos0)[14], 3);
    BF(1, 14, SBM_T(kCos1)[1], 1); BF(17, 30, -SBM_T(kCos1)[1], 1);
    BF0(6, 25, SBM_T(kCos0)[6], 1); BF0(9, 22, SBM_T(kCos0)[9], 1);
    BF(6, 9, SBM_T(kCos1)[6], 2); BF(22, 25, -SBM_T(kCos1)[6], 2);
    BF(1, 6, SBM_T(kCos2)[1], 1); BF(9, 14, -SBM_T(kCos2)[1], 1); BF(17, 22, SBM_T(kCos2)[1], 1); BF(25, 30, -SBM_T(kCos2)[1], 1);
    BF0(2, 29, SBM_T(kCos0)[2], 1); BF0(13, 18, SBM_T(kCos0)[13], 3);
    BF(2, 13, SBM_T(kCos1)[2], 1); BF(18, 29, -SBM_T(kCos1)[2], 1);
    BF0(5, 26, SBM_T(kCos0)[5], 1); BF0(10, 21, SBM_T(kCos0)[10], 1);
    BF(5, 10, SBM_T(kCos1)[5], 2); BF(21, 26, -SBM_T(kCos1)[5], 2);
    BF(2, 5, SBM_T(kCos2)[2], 1); BF(10, 13, -SBM_T(kCos2)[2], 1); BF(18, 21, SBM_T(kCos2)[2], 1); BF(26, 29, -SBM_T(kCos2)[2], 1);
    BF(1, 2, SBM_T(kCos3)[1], 2); BF(5, 6, -SBM_T(kCos3)[1], 2); BF(9, 10, SBM_T(kCos3)[1], 2); BF(13, 14, -SBM_T(kCos3)[1], 2);
    BF(17, 18, SBM_T(kCos3)[1], 2); BF(21, 22, -SBM_T(kCos3)[1], 2); BF(25, 26, SBM_T(kCos3)[1], 2); BF(29, 30, -SBM_T(kCos3)[1], 2);
    BF1(0, 1, 2, 3); BF2(4, 5, 6, 7); BF1(8, 9, 10, 11); BF2(12, 13, 14, 15);
    BF1(16, 17, 18, 19); BF2(20, 21, 22, 23); BF1(24, 25, 26, 27); BF2(28, 29, 30, 31);
    v[8] = SBM_ADD(v[8], v[12]); v[12] = SBM_ADD(v[12], v[10]); v[10] = SBM_ADD(v[10], v[14]);
    v[14] = SBM_ADD(v[14], v[9]); v[9] = SBM_ADD(v[9], v[13]); v[13] = SBM_ADD(v[13], v[11]);
    v[11] = SBM_ADD(v[11], v[15]);
    int32_t o[32];
    o[0] = v[0]; o[16] = v[1]; o[8] = v[2]; o[24] = v[3]; o[4] = v[4]; o[20] = v[5]; o[12] = v[6]; o[28] = v[7];
    o[2] = v[8]; o[18] = v[9]; o[10] = v[10]; o[26] = v[11]; o[6] = v[12]; o[22] = v[13]; o[14] = v[14]; o[30] = v[15];
    v[24] = SBM_ADD(v[24], v[28]); v[28] = SBM_ADD(v[28], v[26]); v[26] = SBM_ADD(v[26], v[30]);
    v[30] = SBM_ADD(v[30], v[25]); v[25] = SBM_ADD(v[25], v[29]); v[29] = SBM_ADD(v[29], v[27]);
    v[27] = SBM_ADD(v[27], v[31]);
    o[1] = SBM_ADD(v[16], v[24]); o[17] = SBM_ADD(v[17], v[25]); o[9] = SBM_ADD(v[18], v[26]);
    o[25] = SBM_ADD(v[19], v[27]); o[5] = SBM_ADD(v[20], v[28]); o[21] = SBM_ADD(v[21], v[29]);
    o[13] = SBM_ADD(v[22], v[30]); o[29] = SBM_ADD(v[23], v[31]); o[3] = SBM_ADD(v[24], v[20]);
    o[19] = SBM_ADD(v[25], v[21]); o[11] = SBM_ADD(v[26], v[22]); o[27] = SBM_ADD(v[27], v[23]);
    o[7] = SBM_ADD(v[28], v[18]); o[23] = SBM_ADD(v[29], v[19]); o[15] = SBM_ADD(v[30], v[17]); o[31] = v[31];
    SBM_UNROLL
    for (int i = 0; i < 32; ++i) out[i] = o[i];
#undef BF0
#undef BF
#undef BF1
#undef BF2
#undef SBM_ADD
#undef SBM_SUB
}

// The sample of a slot output in FFmpeg's emission order: 0, 1, 31, 2, 30, ..., 15, 17, 16
SBM_HD int emitted(int pos) {
    return pos == 0 ? 0 : pos == 31 ? 16 : (pos & 1) ? (pos + 1) >> 1 : 32 - (pos >> 1);
}

// The window sum of output sample n (0..31) of slot t of one channel, with no remainder: v(u) is the 32 synthesis
// values slot u added (the DCT output), zero before the first slot.  A = v(t - 2k), B = v(t - 2k - 1).
template <class Rows>
SBM_HD int64_t window_sum(const Rows& v, int64_t t, int n) {
    int64_t s = 0;
    SBM_UNROLL
    for (int k = 0; k < 8; ++k) {
        const int64_t ta = t - 2 * k, tb = ta - 1;
        const int32_t wa = window_at(n + 64 * k), wb = window_at(n + 32 + 64 * k);
        if (n == 0) {
            s += (int64_t)wa * v(ta, 16) - (int64_t)wb * v(tb, 16);
        } else if (n < 16) {
            s += (int64_t)wa * v(ta, 16 + n) - (int64_t)wb * v(tb, 16 - n);
        } else if (n == 16) {
            s -= (int64_t)wb * v(tb, 0);
        } else {
            s -= (int64_t)wa * v(ta, 48 - n) + (int64_t)wb * v(tb, n - 16);
        }
    }
    return s;
}

// the output sample for a window sum and the remainder before it
SBM_HD int16_t round_sample(uint32_t remainder, int64_t sum) {
    const int64_t x = ((int64_t)(remainder & ((1u << kOutShift) - 1)) + sum) >> kOutShift;
    return (int16_t)(x < -32768 ? -32768 : x > 32767 ? 32767 : x);
}

// ---- host side: the frame chain ----

// The stream parameters every frame shares
struct Stream {
    int32_t channels, rate, lsf;
    int64_t first;           // byte offset of the first frame header in the buffer
    int32_t skipped;         // 1 when bytes other than zeros precede it: that frame is not decoded
    int32_t cut;             // 1 when the stream ends inside a frame
};

// The frames of buf[0, nbytes) as FFmpeg's MPEG audio parser splits them and its decoder takes them: from the first
// position the parser takes for a header, header after header.  The parser hands the bytes before that header over
// with its frame, and the decoder, which skips only leading zeros, refuses that packet: so after other bytes the first
// frame is not decoded (s->skipped).  A last frame the stream cuts short (s->cut) is decoded with zeros for what is
// missing, as FFmpeg decodes it, when its header is whole, and dropped when not.  `where(b)` names the file offset of
// buffer byte b.  Returns false with a message for a header this decoder refuses, or a change of layer, rate or
// channel count.
template <class Where>
bool frame_table(const uint8_t* buf, int64_t nbytes, Where where, std::vector<Frame>& frames, Stream* s, char* msg,
                 size_t msg_len) {
    frames.clear();
    s->skipped = s->cut = 0;
    int64_t b = 0;
    Header h0{};
    // the first position whose four bytes FFmpeg's parser takes for a header: sync, no reserved version, layer,
    // bitrate or rate, and not free format.  If it is not layer II at 16 to 48 kHz, the stream is refused there.
    for (; b + 4 <= nbytes; ++b) {
        const uint32_t h = ((uint32_t)buf[b] << 24) | ((uint32_t)buf[b + 1] << 16) | ((uint32_t)buf[b + 2] << 8) | buf[b + 3];
        const int bi = (h >> 12) & 15;
        if ((h & 0xFFE00000u) != 0xFFE00000u || ((h >> 19) & 3) == 1 || ((h >> 17) & 3) == 0 || bi == 15 || bi == 0 ||
            ((h >> 10) & 3) == 3)
            continue;
        const char* why = parse_header(h, &h0);
        if (why) return sbframes::refuse(msg, msg_len, "MP2 frame", 0, where(b), why);
        break;
    }
    if (b + 4 > nbytes) {
        snprintf(msg, msg_len, "no MPEG audio layer II frame header in the stream");
        return false;
    }
    s->first = b;
    for (int64_t i = 0; i < b; ++i) s->skipped |= buf[i] != 0;
    s->channels = h0.channels;
    s->rate = h0.rate;
    s->lsf = h0.lsf;
    while (b < nbytes) {
        const int64_t f = (int64_t)frames.size();
        if (b + 4 > nbytes) { s->cut = 1; break; }
        const uint32_t h = ((uint32_t)buf[b] << 24) | ((uint32_t)buf[b + 1] << 16) | ((uint32_t)buf[b + 2] << 8) | buf[b + 3];
        Header t;
        const char* why = parse_header(h, &t);
        if (why) return sbframes::refuse(msg, msg_len, "MP2 frame", f, where(b), why);
        if (t.lsf != h0.lsf || t.rate != h0.rate)
            return sbframes::refuse(msg, msg_len, "MP2 frame", f, where(b), "the sample rate changes mid-stream");
        if (t.channels != h0.channels)
            return sbframes::refuse(msg, msg_len, "MP2 frame", f, where(b), "the channel count changes mid-stream");
        const int cut = b + t.size > nbytes;
        if (!(b == s->first && s->skipped)) frames.push_back(Frame{b, cut ? (int32_t)(nbytes - b) : t.size, h, cut, 0});
        if (cut) { s->cut = 1; break; }
        b += t.size;
    }
    if (frames.empty()) {
        snprintf(msg, msg_len, "MP2 frame 0 at byte offset %lld: the stream ends inside it", (long long)where(s->first));
        return false;
    }
    return true;
}

}  // namespace sbmp2
