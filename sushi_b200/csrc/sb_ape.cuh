// Monkey's Audio (APE, file version 3990) frame decoding, written once for the kernels of sb_ape.cu and for the CPU
// (tests/emu/emu_ape_driver.cpp compiles this header with g++).  Everything here is a __host__ __device__ function of
// plain integers and byte pointers; the arithmetic is FFmpeg's `ape` decoder's, operation for operation:
//   the packet as FFmpeg's demuxer cuts it, read through the decoder's 32-bit word byte-swap, from its `skip` byte on;
//   the frame header: CRC word, optional flags word, one ignored byte;
//   the 3990 range decoder with its adaptive sum (ksum) and the overflow escape;
//   the NN filters: int16 weights and saturated int16 history, the dot product in 32-bit wrap-around, sign-based
//     adaptation with adapt values that halve 1, 2 and 8 samples back;
//   the 3950 predictor (stage A per channel, stage B fed by the other channel's filtered output) in FFmpeg's 64-bit
//     layout with 32-bit predictions (its default mode);
//   the decorrelation, the CRC-32 of the little-endian output bytes and the top-16-bit store.
//
// A frame decodes in four stages (sb_ape.cu runs one kernel per stage, the emulation one loop):
//   entropy    entropy_frame: the frame's residuals into the int32 scratch at scratch[(sample + i) * channels + ch];
//   NN         one filter cascade per (frame, coded channel): NnFilter's lane_step on each of 32 lanes' taps, their
//              partial dot products summed, then finish on the sum;
//   predictor  predictor_frame: the predictor, the decorrelation, the output int32 back into the scratch and the
//              top 16 bits into the PCM;
//   CRC        crc_bytes over 32 slices of the frame's samples, joined by crc_combine, then check_crc.
// Each stage leaves a status per frame; a later stage skips a frame whose status is not kOk.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <vector>

#include "sb_frames.h"

#if defined(__CUDACC__)
#define SBA_HD __host__ __device__ __forceinline__
#else
#define SBA_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define SBA_UNROLL _Pragma("unroll")
#else
#define SBA_UNROLL
#endif

namespace sbape {

constexpr int kVersion = 3990;
constexpr int kLevels = 3;                        // NN filters per channel at most
constexpr int kRing = 2048;                       // NN history ring (a power of two above the longest filter)

enum {
    kOk = 0,
    kShort,             // fewer than 6 bytes left for the CRC or the flags word
    kFlags,             // flags outside mono silence, stereo silence and pseudo-stereo
    kRange,             // the range decoder reads past the frame
    kSymbol,            // an overflow symbol past 65535
    kCrc,               // the frame CRC disagrees
    kInterim,           // a 24-bit stereo sample past +-2^23: FFmpeg leaves its default (32-bit) predictor there
};

SBA_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kShort: return "invalid frame header (fewer than 6 bytes left for the CRC or the flags)";
    case kFlags: return "invalid frame flags";
    case kRange: return "range decoder runs past the frame";
    case kSymbol: return "range decoder symbol out of range";
    case kCrc: return "CRC mismatch";
    case kInterim: return "24-bit sample outside 24 bits (where FFmpeg leaves its default predictor)";
    default: return "unknown error";
    }
}

// what a frame turned out to be, from its flags (entropy stage); the later stages follow it
enum { kSilence = 0, kMono = 1, kStereo = 2 };

// FFmpeg's ape_filter_orders / ape_filter_fracbits, by compression level / 1000 - 1
SBA_HD int filter_order(int fset, int l) {
    const int t[5][3] = {{0, 0, 0}, {16, 0, 0}, {64, 0, 0}, {32, 256, 0}, {16, 256, 1280}};
    return t[fset][l];
}
SBA_HD int filter_frac(int fset, int l) {
    const int t[5][3] = {{0, 0, 0}, {11, 0, 0}, {11, 0, 0}, {10, 13, 0}, {11, 13, 15}};
    return t[fset][l];
}

// the stream parameters every frame shares (sb_ape_decode_frames' config)
struct Config {
    int32_t channels;        // 1 or 2
    int32_t bits;            // 16 or 24
    int32_t fset;            // compression level / 1000 - 1
    int32_t blocks;          // blocks per frame
    int32_t final_blocks;    // blocks of the last frame
};

// one frame as FFmpeg's demuxer hands it over: bytes [start, start + size) of the buffer, byte-swapped in 32-bit words;
// the frame begins `skip` bytes in; bytes past `whole` (the size rounded down to 4) read as zeros
struct Frame {
    int64_t start, size, whole;
    int64_t sample;          // first block of the frame in the stream
    int32_t skip, blocks;
};

// byte i of the frame's swapped packet
SBA_HD uint32_t byte_at(const uint8_t* buf, const Frame& f, int64_t i) {
    return i < f.whole ? buf[f.start + (i ^ 3)] : 0u;
}

SBA_HD int sign_neg(int64_t x) { return (x < 0) - (x > 0); }     // FFmpeg's APESIGN

// ---- entropy ----

struct RangeDecoder {
    const uint8_t* buf;
    const Frame* f;
    int64_t pos;
    uint32_t low, range, help, buffer;
    bool error;

    SBA_HD void normalize() {
        while (range <= (1u << 23)) {
            buffer <<= 8;
            if (pos < f->size) buffer += byte_at(buf, *f, pos);
            else error = true;
            ++pos;
            low = (low << 8) | ((buffer >> 1) & 0xFF);
            range <<= 8;
        }
    }
    SBA_HD uint32_t culfreq(uint32_t total) {
        normalize();
        help = range / total;
        return low / help;
    }
    SBA_HD uint32_t culshift(int shift) {
        normalize();
        help = range >> shift;
        return low / help;
    }
    SBA_HD void update(uint32_t width, uint32_t start) {
        low -= help * start;
        range = help * width;
    }
};

// One residual.  ksum: the channel's adaptive sum, which sets the pivot.  (FFmpeg also keeps a Rice parameter k
// beside it, but in version 3990 k feeds only its own update and no output, so it is not kept here.)  counts: FFmpeg's
// counts_3980 (cumulative frequencies of the overflow symbols 0 to 20).
SBA_HD int32_t decode_value(RangeDecoder& rc, uint32_t& ksum, const uint16_t* counts, bool& bad_symbol) {
    uint32_t pivot = ksum >> 5;
    if (pivot == 0) pivot = 1;
    const uint32_t cf = rc.culshift(16);
    uint32_t overflow;
    if (cf > 65492) {
        overflow = cf - 65535 + 63;
        rc.update(1, cf);
        if (cf > 65535) bad_symbol = true;
    } else {
        uint32_t s = 0;
        while (counts[s + 1] <= cf) ++s;
        rc.update(counts[s + 1] - counts[s], counts[s]);
        overflow = s;
    }
    if (overflow == 63) {
        uint32_t hi = rc.culshift(16);
        rc.update(1, hi);
        uint32_t lo = rc.culshift(16);
        rc.update(1, lo);
        overflow = (hi << 16) | lo;
    }
    uint32_t base;
    if (pivot < 0x10000) {
        base = rc.culfreq(pivot);
        rc.update(1, base);
    } else {
        uint32_t hi = pivot;
        int bbits = 0;
        while (hi & ~0xFFFFu) {
            hi >>= 1;
            ++bbits;
        }
        const uint32_t bh = rc.culfreq(hi + 1);
        rc.update(1, bh);
        const uint32_t bl = rc.culfreq(1u << bbits);
        rc.update(1, bl);
        base = (bh << bbits) + bl;
    }
    base += overflow * pivot;
    ksum += ((base + 1) / 2) - ((ksum + 16) >> 5);
    return (int32_t)(((base >> 1) ^ ((base & 1) - 1)) + 1);
}

// The frame's header and residuals: scratch + (f.sample * channels) receives them interleaved by the stream's
// channels (Y then X; a mono-coded frame of a stereo stream fills channel 0 only).  *kind: kSilence, kMono or kStereo;
// *crc: the header's CRC (top bit cleared).
SBA_HD int entropy_frame(const uint8_t* buf, const Frame& f, const Config& c, int32_t* scratch, int32_t* kind,
                         uint32_t* crc) {
    int64_t pos = f.skip;
    *kind = kSilence;
    if (f.size - pos < 6) return kShort;
    uint32_t w = 0;
    for (int i = 0; i < 4; ++i) w = (w << 8) | byte_at(buf, f, pos++);
    uint32_t flags = 0;
    if (w & 0x80000000u) {
        w &= 0x7FFFFFFFu;
        if (f.size - pos < 6) return kShort;
        for (int i = 0; i < 4; ++i) flags = (flags << 8) | byte_at(buf, f, pos++);
    }
    *crc = w;
    if (flags & ~7u) return kFlags;
    ++pos;                                                  // the first byte of the range coder is ignored
    RangeDecoder rc;
    rc.buf = buf;
    rc.f = &f;
    rc.buffer = byte_at(buf, f, pos++);
    rc.pos = pos;
    rc.low = rc.buffer >> 1;
    rc.range = 1u << 7;
    rc.help = 0;
    rc.error = false;
    const bool mono = c.channels == 1 || (flags & 4);
    if (mono ? (flags & 3) != 0 : (flags & 3) == 3) return kOk;     // silence: FFmpeg decodes nothing
    *kind = mono ? kMono : kStereo;
    const int coded = mono ? 1 : 2;
    const uint16_t counts[22] = {0,     19578, 36160, 48417, 56323, 60899, 63265, 64435, 64971, 65232, 65351,
                                 65416, 65447, 65466, 65476, 65482, 65485, 65488, 65490, 65491, 65492, 65493};
    uint32_t ksum[2] = {16u << 10, 16u << 10};
    bool bad = false;
    int32_t* out = scratch + f.sample * c.channels;
    // a frame that reads past its end is refused, so its decode stops there (a damaged block count cannot keep the
    // thread decoding past the frame's bytes)
    for (int32_t i = 0; i < f.blocks && !rc.error; ++i)
        for (int ch = 0; ch < coded; ++ch) out[(int64_t)i * c.channels + ch] = decode_value(rc, ksum[ch], counts, bad);
    if (rc.error) return kRange;
    if (bad) return kSymbol;
    return kOk;
}

// ---- NN filters ----

// One filter's state shared by the lanes: its history ring of saturated outputs and the adapt value each output set
// (before halving), both kRing int16; and the running average of |output|.  Lane l holds taps l, l + 32, l + 64, ...
// of the filter's weights (tap i pairs with the output `order - i` samples back).
struct NnShared {
    int16_t* hist;
    int16_t* adapt;
};

// Lane `lane`'s share of step t: its partial dot product of the weights with the last `order` outputs, and its weights
// adapted by `sign` (APESIGN of the step's input) times their adapt values.  T: taps per lane, ceil(order / 32).
template <int T>
SBA_HD uint32_t lane_step(int32_t (&w)[T], int lane, int order, const NnShared& s, int64_t t, int sign) {
    uint32_t dot = 0;
    SBA_UNROLL
    for (int k = 0; k < T; ++k) {
        const int i = k * 32 + lane;
        if (i < order) {
            const int age = order - i;
            const int at = (int)((t - age) & (kRing - 1));
            const int32_t h = s.hist[at];
            const int shift = (age >= 2) + (age >= 3) + (age >= 9);
            const int32_t a = (int32_t)s.adapt[at] >> shift;
            dot += (uint32_t)(w[k] * h);
            w[k] = (int16_t)(w[k] + sign * a);
        }
    }
    return dot;
}

// The rest of step t once the lanes' dot products are summed: the filter's output, and the history and adapt value it
// leaves (to be stored at ring position t & (kRing - 1)).
SBA_HD int32_t finish(uint32_t dot, int frac, int32_t in, int32_t& avg, int16_t& hist, int16_t& adapt) {
    const int32_t res = (int32_t)(((int64_t)(int32_t)dot + (1ll << (frac - 1))) >> frac);
    const int32_t out = (int32_t)((uint32_t)res + (uint32_t)in);
    hist = (int16_t)(out > 32767 ? 32767 : out < -32768 ? -32768 : out);
    const uint32_t absres = out < 0 ? 0u - (uint32_t)out : (uint32_t)out;
    if (absres)
        adapt = (int16_t)(sign_neg(out) *
                          (8 << ((absres > (int64_t)avg * 3) + (absres > (uint32_t)(avg + avg / 3)))));
    else
        adapt = 0;
    avg += (int32_t)(absres - (uint32_t)avg) / 16;
    return out;
}

// ---- predictor ----

struct Predictor {
    int64_t dA[2][4], aA[2][4], dB[2][5], aB[2][5];
    int64_t cA[2][4], cB[2][5];
    int64_t lastA[2], filterA[2], filterB[2];

    SBA_HD void init() {
        const int64_t c0[4] = {360, 317, -109, 98};
        for (int f = 0; f < 2; ++f) {
            for (int i = 0; i < 4; ++i) { dA[f][i] = aA[f][i] = 0; cA[f][i] = c0[i]; }
            for (int i = 0; i < 5; ++i) dB[f][i] = aB[f][i] = cB[f][i] = 0;
            lastA[f] = filterA[f] = filterB[f] = 0;
        }
    }
    // FFmpeg's predictor_update_filter for channel f (0: Y, 1: X) in its default (32-bit prediction) mode
    SBA_HD int32_t stereo(int f, int32_t decoded) {
        SBA_UNROLL
        for (int i = 3; i > 0; --i) { dA[f][i] = dA[f][i - 1]; aA[f][i] = aA[f][i - 1]; }
        const int64_t prevA = dA[f][1];
        dA[f][0] = lastA[f];
        aA[f][0] = sign_neg(dA[f][0]);
        dA[f][1] = dA[f][0] - prevA;
        aA[f][1] = sign_neg(dA[f][1]);
        int64_t pa = 0;
        SBA_UNROLL
        for (int i = 0; i < 4; ++i) pa += dA[f][i] * cA[f][i];
        SBA_UNROLL
        for (int i = 4; i > 0; --i) { dB[f][i] = dB[f][i - 1]; aB[f][i] = aB[f][i - 1]; }
        const int64_t prevB = dB[f][1];
        dB[f][0] = filterA[f ^ 1] - ((int64_t)((uint64_t)filterB[f] * 31u) >> 5);
        aB[f][0] = sign_neg(dB[f][0]);
        dB[f][1] = dB[f][0] - prevB;
        aB[f][1] = sign_neg(dB[f][1]);
        filterB[f] = filterA[f ^ 1];
        int64_t pb = 0;
        SBA_UNROLL
        for (int i = 0; i < 5; ++i) pb += dB[f][i] * cB[f][i];
        const int32_t p = (int32_t)((int64_t)(int32_t)pa + ((int64_t)(int32_t)pb >> 1));
        lastA[f] = (int32_t)((uint32_t)decoded + (uint32_t)(p >> 10));
        filterA[f] = lastA[f] + ((int64_t)((uint64_t)filterA[f] * 31u) >> 5);
        const int s = sign_neg(decoded);
        SBA_UNROLL
        for (int i = 0; i < 4; ++i) cA[f][i] += aA[f][i] * s;
        SBA_UNROLL
        for (int i = 0; i < 5; ++i) cB[f][i] += aB[f][i] * s;
        return (int32_t)filterA[f];
    }
    // FFmpeg's predictor_decode_mono_3950, one sample
    SBA_HD int32_t mono(int32_t decoded) {
        SBA_UNROLL
        for (int i = 3; i > 0; --i) { dA[0][i] = dA[0][i - 1]; aA[0][i] = aA[0][i - 1]; }
        const int64_t prevA = dA[0][1];
        dA[0][0] = lastA[0];
        dA[0][1] = dA[0][0] - prevA;
        int64_t pa = 0;
        SBA_UNROLL
        for (int i = 0; i < 4; ++i) pa += dA[0][i] * cA[0][i];
        lastA[0] = (int32_t)((uint32_t)decoded + (uint32_t)((int32_t)pa >> 10));
        aA[0][0] = sign_neg(dA[0][0]);
        aA[0][1] = sign_neg(dA[0][1]);
        const int s = sign_neg(decoded);
        SBA_UNROLL
        for (int i = 0; i < 4; ++i) cA[0][i] += aA[0][i] * s;
        filterA[0] = lastA[0] + ((int64_t)((uint64_t)filterA[0] * 31u) >> 5);
        return (int32_t)filterA[0];
    }
};

// the top 16 bits of FFmpeg's output sample: S16 as is, S32 (24-bit sample << 8) >> 16
SBA_HD int16_t store(int32_t v, int bits) {
    return bits == 16 ? (int16_t)(uint16_t)(uint32_t)v : (int16_t)(uint16_t)((uint32_t)v >> 8);
}

// The predictor and the decorrelation over the frame's filtered residuals (in the scratch), the output samples back
// into the scratch and their top 16 bits into pcm (interleaved, at the frame's sample position).
SBA_HD int predictor_frame(const Frame& f, const Config& c, int kind, int32_t* scratch, int16_t* pcm) {
    int32_t* d = scratch + f.sample * c.channels;
    int16_t* out = pcm + f.sample * c.channels;
    const int64_t n = (int64_t)f.blocks * c.channels;
    if (kind == kSilence) {
        for (int64_t i = 0; i < n; ++i) { d[i] = 0; out[i] = 0; }
        return kOk;
    }
    Predictor p;
    p.init();
    int status = kOk;
    for (int32_t i = 0; i < f.blocks; ++i) {
        int32_t* s = d + (int64_t)i * c.channels;
        if (kind == kMono) {
            s[0] = p.mono(s[0]);
            if (c.channels == 2) s[1] = s[0];
        } else {
            const int32_t y = p.stereo(0, s[0]);
            const int32_t x = p.stereo(1, s[1]);
            const int32_t left = (int32_t)((uint32_t)x - (uint32_t)(y / 2));
            const int32_t right = (int32_t)((uint32_t)left + (uint32_t)y);
            s[0] = left;
            s[1] = right;
            // FFmpeg's test, FFMIN(FFNABS(left), FFNABS(right)) < -(1 << 23): +-2^23 itself decodes
            if (c.bits == 24 && (left > (1 << 23) || left < -(1 << 23) || right > (1 << 23) || right < -(1 << 23)))
                status = kInterim;
        }
        for (int ch = 0; ch < c.channels; ++ch) out[(int64_t)i * c.channels + ch] = store(s[ch], c.bits);
    }
    return status;
}

// ---- CRC ----

// CRC-32 (IEEE, reflected, zlib's): table[b] for one byte
SBA_HD uint32_t crc_entry(uint32_t b) {
    uint32_t c = b;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
    return c;
}

// a * b modulo the CRC polynomial, in the reflected bit order (zlib's multmodp)
SBA_HD uint32_t gf_mul(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

// x^(8 n) modulo the polynomial (zlib's x2nmodp(n, 3))
SBA_HD uint32_t x_pow8(int64_t n) {
    uint32_t p = 1u << 31, sq = 1u << 30;             // 1 and x
    for (int k = 0; k < 3; ++k) sq = gf_mul(sq, sq);  // x^8
    while (n) {
        if (n & 1) p = gf_mul(sq, p);
        n >>= 1;
        sq = gf_mul(sq, sq);
    }
    return p;
}

// zlib's crc32_combine: the CRC of A then B from crc(A), crc(B) and |B|
SBA_HD uint32_t crc_combine(uint32_t a, uint32_t b, int64_t len_b) { return gf_mul(x_pow8(len_b), a) ^ b; }

// zlib's crc32 of the output bytes of samples [lo, hi) (interleaved, from the scratch): 2 or 3 little-endian bytes each
SBA_HD uint32_t crc_bytes(const int32_t* s, int64_t lo, int64_t hi, int bits, const uint32_t* table) {
    uint32_t c = 0xFFFFFFFFu;
    for (int64_t i = lo; i < hi; ++i) {
        const uint32_t v = (uint32_t)s[i];
        c = table[(c ^ v) & 255] ^ (c >> 8);
        c = table[(c ^ (v >> 8)) & 255] ^ (c >> 8);
        if (bits == 24) c = table[(c ^ (v >> 16)) & 255] ^ (c >> 8);
    }
    return c ^ 0xFFFFFFFFu;
}

// FFmpeg's test: the CRC of the output bytes shifted right by one is the header's
SBA_HD int check_crc(uint32_t crc, uint32_t stored) { return (crc >> 1) == stored ? kOk : kCrc; }

// ---- host side: what sb_ape_decode_frames does around the kernels; the CPU build of the tests runs the same ----

// config[0..6) (channels, bits, rate, compression level, blocks per frame, final frame blocks) into *c and *rate
inline bool parse_config(const int32_t* config, Config* c, int32_t* rate, char* msg, size_t msg_len) {
    c->channels = config[0];
    c->bits = config[1];
    *rate = config[2];
    const int32_t level = config[3];
    c->blocks = config[4];
    c->final_blocks = config[5];
    c->fset = level / 1000 - 1;
    if (c->channels < 1 || c->channels > 2)
        snprintf(msg, msg_len, "APE with %d channels is not supported (1 or 2)", c->channels);
    else if (c->bits != 16 && c->bits != 24)
        snprintf(msg, msg_len, "APE with %d bits per sample is not supported (16 or 24)", c->bits);
    else if (level % 1000 || level < 1000 || level > 5000)
        snprintf(msg, msg_len, "APE compression level %d is not supported", level);
    else if (*rate < 1 || c->blocks < 1 || c->final_blocks < 1 || c->final_blocks > c->blocks)
        snprintf(msg, msg_len, "sb_ape_decode_frames: bad stream parameters");
    else
        return true;
    return false;
}

// The kernels' frames.  offsets[f]: where frame f begins in the buffer (its seek-table position); the buffer holds the
// stream's bytes up to nbytes (the file less its WAV tail).  As FFmpeg's demuxer does, each frame's packet starts at
// the 32-bit word (counted from frame 0) that holds its first byte, ends at the next frame's start rounded up to a
// word, and the last ends at nbytes rounded down to a word, plus its skip, rounded up, and cut at nbytes.
inline bool frame_table(const int64_t* offsets, const int64_t* where, int64_t n, int64_t nbytes, const Config& c,
                        std::vector<Frame>& frames, int64_t* samples, char* msg, size_t msg_len) {
    frames.resize((size_t)n);
    for (int64_t f = 0; f < n; ++f) {
        Frame& d = frames[(size_t)f];
        if (offsets[f] < 0 || offsets[f] >= nbytes || (f && offsets[f] <= offsets[f - 1]))
            return sbframes::refuse(msg, msg_len, "APE frame", f, where[f], "frame starts outside the buffer");
        d.skip = (int32_t)((offsets[f] - offsets[0]) & 3);
        int64_t size = f + 1 < n ? offsets[f + 1] - offsets[f] : ((nbytes - offsets[f]) & ~(int64_t)3);
        if (size <= 0) return sbframes::refuse(msg, msg_len, "APE frame", f, where[f], "empty frame");
        size = (size + d.skip + 3) & ~(int64_t)3;
        d.start = offsets[f] - d.skip;
        if (d.start + size > nbytes) size = nbytes - d.start;
        d.size = size;
        d.whole = size & ~(int64_t)3;
        d.sample = f * (int64_t)c.blocks;
        d.blocks = f + 1 < n ? c.blocks : c.final_blocks;
    }
    *samples = (n - 1) * (int64_t)c.blocks + c.final_blocks;
    return true;
}

}  // namespace sbape
