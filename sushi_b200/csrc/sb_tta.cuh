// TTA (True Audio) frame decoding, written once for the GPU kernel of sb_tta.cu and for the CPU
// (tests/emu/emu_tta_driver.cpp compiles this header with g++).  Everything here is a __host__ __device__ function of
// plain integers and byte pointers: the bit reader (least significant bit first), the adaptive Rice code with its two
// parameters per channel, the 8-tap adaptive filter, the fixed first-order predictor, the inter-channel decorrelation,
// the frame's CRC-32 and the top-16-bit store.  The arithmetic is FFmpeg's `tta` decoder's, operation for operation,
// in 32-bit wrap-around.
//
// A frame is bytes [offset, offset + size) of the caller's buffer: its bitstream, then the CRC-32 of the bitstream
// (4 bytes, little-endian).  The reader loads no byte outside the frame: past its end it shifts in zeros, and every code
// is checked against the end of the bitstream after it is read.
//
// The per-channel state (filter taps, their steps and history, the filter's last residual, the predictor, the two Rice
// parameters and sums, and the channel's current sample) lives in a State slice: kStateWords int32 per channel, word w
// of channel c at p[(c * kStateWords + w) * stride].  The kernel gives each thread a column of shared memory (stride =
// the block's thread count), so the per-sample loop never touches local memory.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SBT_HD __host__ __device__ __forceinline__
#define SBT_UNROLL _Pragma("unroll")
#else
#define SBT_HD inline
#define SBT_UNROLL
#endif

namespace sbtta {

constexpr int kMaxChannels = 8;
constexpr int kMaxRice = 25;                         // FFmpeg refuses a Rice parameter above MIN_CACHE_BITS
constexpr int kCrcWords = 1024;                      // slice-by-4 CRC-32 table

// word offsets of one channel's state
enum { kQm = 0, kDx = 8, kDl = 16, kError = 24, kPredictor, kK0, kK1, kSum0, kSum1, kValue, kStateWords };

enum {
    kOk = 0,
    kShort,              // a frame shorter than its CRC
    kUnary,              // a unary run that reads past the bitstream
    kBitstream,          // a code that reads past the bitstream
    kRice,               // a Rice parameter above 25
    kEarly,              // a frame other than the last reaches the last frame's length with only its CRC left
    kNotOnCrc,           // bytes left between the last sample and the CRC
    kCrc,                // the frame CRC disagrees
};

SBT_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kShort: return "frame shorter than its CRC";
    case kUnary: return "unary code reads past the frame";
    case kBitstream: return "bitstream reads past the frame";
    case kRice: return "Rice parameter above 25";
    case kEarly: return "frame ends at the last frame's sample count before the last frame (FFmpeg cuts it short)";
    case kNotOnCrc: return "frame does not end on its CRC";
    case kCrc: return "CRC mismatch";
    default: return "unknown error";
    }
}

// the stream parameters every frame shares (sb_tta_decode_frames' config)
struct Config {
    int32_t channels;        // 1 to 8
    int32_t bits;            // 16 or 24
    int32_t frame_length;    // 256 * rate / 245
    int32_t last_length;     // samples of the last frame, 0 when it is a whole frame (FFmpeg's last_frame_length)
};

// what the host hands the kernel per frame
struct Frame {
    int64_t offset, size;    // the frame's bytes, CRC included
    int64_t sample;          // first sample of the frame in the track
    int32_t last;            // 1 for the stream's last frame
    int32_t pad;
};

// FFmpeg's ff_tta_shift_1: 1 << i, held at 1 << 31 past 31
SBT_HD uint32_t shift_1(int i) { return i < 31 ? 1u << i : 0x80000000u; }
SBT_HD uint32_t shift_16(int i) { return shift_1(i + 4); }

// CRC-32 (IEEE, reflected): table[b] for one byte, table[256 * j + b] the same byte j bytes further from the end
SBT_HD void crc_table_entry(uint32_t* table, int i) {
    const int b = i & 255, j = i >> 8;
    uint32_t c = (uint32_t)b;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
    for (int s = 0; s < j; ++s)
        for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
    table[i] = c;
}

SBT_HD uint32_t crc32(const uint8_t* p, int64_t n, const uint32_t* t) {
    uint32_t c = 0xFFFFFFFFu;
    int64_t i = 0;
    for (; i + 4 <= n; i += 4) {
        c ^= (uint32_t)p[i] | ((uint32_t)p[i + 1] << 8) | ((uint32_t)p[i + 2] << 16) | ((uint32_t)p[i + 3] << 24);
        c = t[768 + (c & 255)] ^ t[512 + ((c >> 8) & 255)] ^ t[256 + ((c >> 16) & 255)] ^ t[c >> 24];
    }
    for (; i < n; ++i) c = t[(c ^ p[i]) & 255] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

SBT_HD int trailing_zeros64(uint64_t v) {
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)v) - 1;
#else
    return __builtin_ctzll(v);
#endif
}

// least-significant-bit-first reader over bytes [0, end) of p; zeros past `end`
struct Reader {
    const uint8_t* p;
    int64_t at, end;         // next byte to load, end of the frame
    uint64_t cache;          // the next `n` bits, first in bit 0
    int n;
    int64_t pos, limit;      // bits consumed, bits of the bitstream

    SBT_HD void refill() {                 // to 56-63 bits, so that a shift by a whole run stays under 64
        while (n < 56) {
            const uint64_t b = at < end ? p[at] : 0;
            cache |= b << n;
            n += 8;
            ++at;
        }
    }
    SBT_HD uint32_t bits(int k) {            // k <= 25
        if (n < k) refill();
        const uint32_t v = (uint32_t)(cache & ((1ull << k) - 1));
        cache >>= k;
        n -= k;
        pos += k;
        return v;
    }
    // the count of 1 bits before the next 0 bit (consumed); false when the run or its 0 lies past the bitstream
    SBT_HD bool unary(uint32_t& u) {
        u = 0;
        for (;;) {
            refill();
            const int t = trailing_zeros64(~cache);          // bits past n are 0, so t <= n
            if (t < n) {
                cache >>= t + 1;
                n -= t + 1;
                pos += t + 1;
                u += (uint32_t)t;
                return pos <= limit;
            }
            u += (uint32_t)n;
            pos += n;
            cache = 0;
            n = 0;
            if (pos > limit) return false;
        }
    }
};

// Per-channel state view: word w of channel c at p[(c * kStateWords + w) * stride]
struct State {
    int32_t* p;
    int stride;
    SBT_HD int32_t& at(int c, int w) const { return p[(c * kStateWords + w) * stride]; }
};

// FFmpeg's tta_filter_process_c on channel c's taps: *in is the residual in, the filtered value out
SBT_HD int32_t filter(const State& s, int c, int32_t in, int shift) {
    int32_t* const q = &s.at(c, kQm);
    const int st = s.stride;
#define SBT_Q(i) q[(i) * st]
#define SBT_X(i) q[(kDx + (i)) * st]
#define SBT_L(i) q[(kDl + (i)) * st]
    const int32_t err = SBT_Q(kError);
    uint32_t qm[8], dl[8], dx[8];
    SBT_UNROLL
    for (int i = 0; i < 8; ++i) {
        qm[i] = (uint32_t)SBT_Q(i);
        dl[i] = (uint32_t)SBT_L(i);
        dx[i] = (uint32_t)SBT_X(i);
    }
    if (err < 0) {
        SBT_UNROLL
        for (int i = 0; i < 8; ++i) qm[i] -= dx[i];
    } else if (err > 0) {
        SBT_UNROLL
        for (int i = 0; i < 8; ++i) qm[i] += dx[i];
    }
    uint32_t sum = 1u << (shift - 1);
    SBT_UNROLL
    for (int i = 0; i < 8; ++i) sum += dl[i] * qm[i];
    const uint32_t x4 = (uint32_t)(((int32_t)dl[4] >> 30) | 1);
    const uint32_t x5 = (uint32_t)((((int32_t)dl[5] >> 30) | 2) & ~1);
    const uint32_t x6 = (uint32_t)((((int32_t)dl[6] >> 30) | 2) & ~1);
    const uint32_t x7 = (uint32_t)((((int32_t)dl[7] >> 30) | 4) & ~3);
    const uint32_t out = (uint32_t)in + (uint32_t)((int32_t)sum >> shift);
    const uint32_t d6 = out - dl[7];
    const uint32_t d5 = d6 - dl[6];
    const uint32_t d4 = d5 - dl[5];
    // dl[0..3] = dl[1..4], dx[0..3] = dx[1..4]
    SBT_L(0) = (int32_t)dl[1]; SBT_L(1) = (int32_t)dl[2]; SBT_L(2) = (int32_t)dl[3]; SBT_L(3) = (int32_t)dl[4];
    SBT_L(4) = (int32_t)d4; SBT_L(5) = (int32_t)d5; SBT_L(6) = (int32_t)d6; SBT_L(7) = (int32_t)out;
    SBT_X(0) = (int32_t)dx[1]; SBT_X(1) = (int32_t)dx[2]; SBT_X(2) = (int32_t)dx[3]; SBT_X(3) = (int32_t)dx[4];
    SBT_X(4) = (int32_t)x4; SBT_X(5) = (int32_t)x5; SBT_X(6) = (int32_t)x6; SBT_X(7) = (int32_t)x7;
    SBT_UNROLL
    for (int i = 0; i < 8; ++i) SBT_Q(i) = (int32_t)qm[i];
    SBT_Q(kError) = in;
#undef SBT_Q
#undef SBT_X
#undef SBT_L
    return (int32_t)out;
}

// the top 16 bits of FFmpeg's output sample: S16 as is, S32 (24-bit sample << 8) >> 16
SBT_HD int16_t store(int32_t v, int bits) {
    return bits == 16 ? (int16_t)(uint16_t)(uint32_t)v : (int16_t)(uint16_t)((uint32_t)v >> 8);
}

// Decode frame `f` into pcm + f.sample * channels (interleaved int16).  crc_table: kCrcWords entries.
SBT_HD int decode_frame(const uint8_t* buf, const Frame& f, const Config& c, const State& s, const uint32_t* crc_table,
                        int16_t* pcm) {
    if (f.size < 4) return kShort;
    const int channels = c.channels;
    const int shift = c.bits == 16 ? 9 : 10;         // ff_tta_filter_configs[bytes - 1]
    for (int ch = 0; ch < channels; ++ch) {
        for (int w = 0; w < kStateWords; ++w) s.at(ch, w) = 0;
        s.at(ch, kK0) = 10;
        s.at(ch, kK1) = 10;
        s.at(ch, kSum0) = (int32_t)shift_16(10);
        s.at(ch, kSum1) = (int32_t)shift_16(10);
    }
    Reader r;
    r.p = buf + f.offset;
    r.at = 0;
    r.end = f.size;
    r.cache = 0;
    r.n = 0;
    r.pos = 0;
    r.limit = (f.size - 4) * 8;
    const int64_t total_bits = f.size * 8;           // FFmpeg's get_bits_left counts the CRC too
    const int32_t want = f.last && c.last_length ? c.last_length : c.frame_length;
    int16_t* out = pcm + f.sample * channels;
    for (int32_t i = 0; i < want;) {
        for (int ch = 0; ch < channels; ++ch) {
            uint32_t u;
            if (!r.unary(u)) return kUnary;
            uint32_t k0 = (uint32_t)s.at(ch, kK0);
            uint32_t k;
            int depth;
            if (u == 0) {
                depth = 0;
                k = k0;
            } else {
                depth = 1;
                k = (uint32_t)s.at(ch, kK1);
                --u;
            }
            if (k > (uint32_t)kMaxRice) return kRice;
            uint32_t value = k ? (u << k) + r.bits((int)k) : u;
            if (r.pos > r.limit) return kBitstream;
            if (depth) {
                uint32_t sum1 = (uint32_t)s.at(ch, kSum1), k1 = k;
                sum1 += value - (sum1 >> 4);
                if (k1 > 0 && sum1 < shift_16((int)k1)) --k1;
                else if (sum1 > shift_16((int)k1 + 1)) ++k1;
                s.at(ch, kSum1) = (int32_t)sum1;
                s.at(ch, kK1) = (int32_t)k1;
                value += shift_1((int)k0);
            }
            uint32_t sum0 = (uint32_t)s.at(ch, kSum0);
            sum0 += value - (sum0 >> 4);
            if (k0 > 0 && sum0 < shift_16((int)k0)) --k0;
            else if (sum0 > shift_16((int)k0 + 1)) ++k0;
            s.at(ch, kSum0) = (int32_t)sum0;
            s.at(ch, kK0) = (int32_t)k0;
            const int32_t v = (int32_t)value;
            const int32_t res = (int32_t)(1u + (uint32_t)((v >> 1) ^ ((v & 1) - 1)));
            int32_t x = filter(s, ch, res, shift);
            const int32_t pred = s.at(ch, kPredictor);
            x = (int32_t)((uint32_t)x + (uint32_t)(int32_t)(((int64_t)pred * 31) >> 5));
            s.at(ch, kPredictor) = x;
            s.at(ch, kValue) = x;
        }
        if (channels > 1) {
            // FFmpeg: the last channel gains half the one before it, then each channel is the next minus itself
            int32_t next = (int32_t)((uint32_t)s.at(channels - 1, kValue) + (uint32_t)(s.at(channels - 2, kValue) / 2));
            out[(int64_t)i * channels + channels - 1] = store(next, c.bits);
            for (int ch = channels - 2; ch >= 0; --ch) {
                next = (int32_t)((uint32_t)next - (uint32_t)s.at(ch, kValue));
                out[(int64_t)i * channels + ch] = store(next, c.bits);
            }
        } else {
            out[i] = store(s.at(0, kValue), c.bits);
        }
        ++i;
        // FFmpeg's test for the short last frame, made in every frame: the last frame's count, and only the CRC left
        if (i == c.last_length && i < want && (total_bits - r.pos) / 8 == 4) return kEarly;
    }
    if ((r.pos + 7) / 8 != f.size - 4) return kNotOnCrc;
    const uint8_t* q = buf + f.offset + f.size - 4;
    const uint32_t stored = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
    if (crc32(buf + f.offset, f.size - 4, crc_table) != stored) return kCrc;
    return kOk;
}

}  // namespace sbtta
