// ALAC (Apple Lossless) frame decoding, written once for the GPU kernels of sb_alac.cu and for the CPU
// (tests/emu/emu_alac_driver.cpp compiles this header with g++).  Everything here is a __host__ __device__ function of
// plain integers and byte pointers: the bit reader, the first element header (k_alac_frames), and the whole frame
// (k_alac_decode): SCE / CPE / LFE elements up to END, escape (uncompressed) elements, the adaptive Golomb code with
// its escape and zero runs, adaptive LPC of orders 0-31 (31: first differences), prediction type 15, stereo unmixing
// and the shifted low bytes.  The arithmetic is FFmpeg's `alac` decoder's, operation for operation: unsigned
// wrap-around where it wraps, sign extension to the element's width after each prediction.
//
// A frame's bytes are [offset, limit) of the caller's buffer, which must hold at least 8 readable bytes past the last
// limit.  Reads stay inside that: every fixed-size field (element header, sample count, unmix parameters, each
// channel's predictor header and coefficients, escape samples, shifted low bits) is checked against the frame's end
// before it is read, and a variable-length Golomb code is read only from a position inside the frame and checked
// after; the reader fetches 5 bytes at a time, so no read reaches more than 6 bytes past the limit.  Bit positions
// are 64-bit.
#pragma once
#include <stdint.h>
#include <vector>

#include "sb_frames.h"

#if defined(__CUDACC__)
#define SBA_HD __host__ __device__ __forceinline__
#else
#define SBA_HD inline
#endif

namespace sbalac {

constexpr int kMaxFrameLength = 65536;     // longer frames are refused (a limit of this decoder, not of the format)

enum {
    kOk = 0,
    kNoElement,          // the first element is END: no samples
    kBadTag,             // an element other than SCE, CPE, LFE or END
    kTooManyChannels,    // more channels than the config declares
    kFewChannels,        // END before every channel of the config
    kBadCount,           // sample count 0 or above frameLength
    kCountMismatch,      // an element whose sample count differs from the first one's
    kBadPrediction,      // prediction type other than 0 and 15
    kBadElement,         // element width above 32 bits, LPC order / quantisation, unmix shift, rice limit 0
    kOverrun,            // the frame reads past its sample's bytes
    kNoEnd,              // no END element
};

SBA_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kNoElement: return "frame holds no element (sample count 0)";
    case kBadTag: return "element tag other than SCE, CPE, LFE or END";
    case kTooManyChannels: return "more channels than the config declares";
    case kFewChannels: return "fewer channels than the config declares";
    case kBadCount: return "sample count 0 or above frameLength";
    case kCountMismatch: return "element sample count differs from the frame's";
    case kBadPrediction: return "prediction type other than 0 or 15";
    case kBadElement: return "invalid element header";
    case kOverrun: return "frame reads past its sample's bytes";
    case kNoEnd: return "frame without END element";
    default: return "unknown error";
    }
}

// ALACSpecificConfig, as sb_alac_index_frames receives it
struct Config {
    int frame_length, bit_depth, pb, mb, kb, channels, rate;
};

// what k_alac_frames finds at a frame's start
struct Listed {
    int32_t samples;
    int32_t code;
};

// what the host hands k_alac_decode per frame
struct FrameDesc {
    int64_t offset, limit;     // bytes [offset, limit) of the buffer
    int64_t sample;            // first sample of the frame in the track
};

// FFmpeg's ff_alac_channel_layout_offsets: output channel of the element at coded channel position `ch`, for
// 1-8 channels; four bits per entry
SBA_HD int layout_offset(int channels, int ch) {
    uint32_t row = 0;
    switch (channels) {
    case 2: row = 0x10u; break;
    case 3: row = 0x102u; break;
    case 4: row = 0x3102u; break;
    case 5: row = 0x43102u; break;
    case 6: row = 0x354102u; break;
    case 7: row = 0x3654102u; break;
    case 8: row = 0x35410762u; break;
    default: row = 0; break;
    }
    return (int)((row >> (4 * ch)) & 15u);
}

SBA_HD int clz32(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __clz((int)v);
#else
    return v ? __builtin_clz(v) : 32;
#endif
}

SBA_HD int log2_floor(uint32_t v) { return v ? 31 - clz32(v) : 0; }     // av_log2 (0 for 0)

// MSB-first bit reader over [pos, end) bits
struct Bits {
    const uint8_t* p;
    int64_t pos, end;
    // the 32 bits from pos
    SBA_HD uint32_t peek32() const {
        const uint8_t* q = p + (pos >> 3);
        const uint64_t v = ((uint64_t)q[0] << 32) | ((uint64_t)q[1] << 24) | ((uint64_t)q[2] << 16) |
                           ((uint64_t)q[3] << 8) | (uint64_t)q[4];
        return (uint32_t)(v >> (8 - (pos & 7)));
    }
    SBA_HD uint32_t read(int n) {              // 0 <= n <= 32
        if (n == 0) return 0;
        const uint32_t v = peek32() >> (32 - n);
        pos += n;
        return v;
    }
    SBA_HD int32_t read_signed(int n) {        // 1 <= n <= 32
        const uint32_t v = read(n);
        return n == 32 ? (int32_t)v : (int32_t)(v << (32 - n)) >> (32 - n);
    }
    SBA_HD bool over() const { return pos > end; }
    SBA_HD int64_t left() const { return end - pos; }
};

SBA_HD int32_t sign_extend(uint32_t v, int bits) {
    const int shift = 32 - bits;
    return (int32_t)(v << shift) >> shift;
}

SBA_HD int sign_only(int32_t v) { return v > 0 ? 1 : (v < 0 ? -1 : 0); }

// FFmpeg's decode_scalar: unary prefix of at most 9 ones; 9 ones escape to `bps` raw bits
SBA_HD uint32_t decode_scalar(Bits& b, int k, int bps) {
    const int ones = clz32(~b.peek32());
    uint32_t x = (uint32_t)(ones < 9 ? ones : 9);
    b.pos += x < 9 ? x + 1 : 9;
    if (x > 8) return b.read(bps);
    if (k != 1) {
        const uint32_t extra = k ? b.peek32() >> (32 - k) : 0;
        x = (x << k) - x;
        if (extra > 1) { x += extra - 1; b.pos += k; }
        else b.pos += k - 1;
    }
    return x;
}

// FFmpeg's rice_decompress into out[0..n): the adaptive Golomb code, its history and its zero runs
SBA_HD int rice_decompress(Bits& b, int32_t* out, int n, int bps, int history_mult, const Config& c) {
    uint32_t history = (uint32_t)c.mb;
    int sign_modifier = 0;
    for (int i = 0; i < n; ++i) {
        if (b.left() <= 0) return kOverrun;
        int k = log2_floor((history >> 9) + 3);
        if (k > c.kb) k = c.kb;
        uint32_t x = decode_scalar(b, k, bps);
        if (b.over()) return kOverrun;
        x += (uint32_t)sign_modifier;
        sign_modifier = 0;
        out[i] = (int32_t)((x >> 1) ^ (0u - (x & 1u)));
        if (x > 0xffffu) history = 0xffff;
        else history += x * (uint32_t)history_mult - ((history * (uint32_t)history_mult) >> 9);
        if (history < 128 && i + 1 < n) {
            k = 7 - log2_floor(history) + (int)((history + 16) >> 6);
            if (k > c.kb) k = c.kb;
            int run = (int)decode_scalar(b, k, 16);
            if (b.over()) return kOverrun;
            if (run > 0) {
                if (run >= n - i) return kBadElement;      // FFmpeg clamps this and goes on; a damaged frame here
                for (int j = 1; j <= run; ++j) out[i + j] = 0;
                i += run;
            }
            if (run <= 0xffff) sign_modifier = 1;
            history = 0;
        }
    }
    return kOk;
}

// FFmpeg's lpc_prediction, in place: buf holds the residuals and receives the samples.  coefs (order entries, the one
// for the nearest sample last) adapt as it runs.  order 31: first differences, coefs unused.
SBA_HD void lpc_prediction(int32_t* buf, int n, int bps, int16_t* coefs, int order, int quant) {
    if (n <= 1) return;
    if (order == 0) return;
    if (order == 31) {
        for (int i = 1; i < n; ++i) buf[i] = sign_extend((uint32_t)buf[i - 1] + (uint32_t)buf[i], bps);
        return;
    }
    int i = 1;
    for (; i <= order && i < n; ++i) buf[i] = sign_extend((uint32_t)buf[i - 1] + (uint32_t)buf[i], bps);
    for (; i < n; ++i) {
        const uint32_t* pred = reinterpret_cast<const uint32_t*>(buf + i - order);
        const int32_t d = buf[i - order - 1];
        uint32_t acc = 0;
        for (int j = 0; j < order; ++j) acc += (pred[j] - (uint32_t)d) * (uint32_t)(int32_t)coefs[j];
        int32_t val = (int32_t)(((int64_t)(int32_t)acc + ((int64_t)1 << (quant - 1))) >> quant);
        uint32_t error_val = (uint32_t)buf[i];
        buf[i] = sign_extend((uint32_t)val + (uint32_t)d + error_val, bps);
        const int error_sign = sign_only((int32_t)error_val);
        if (error_sign) {
            for (int j = 0; j < order && (int32_t)(error_val * (uint32_t)error_sign) > 0; ++j) {
                int32_t v = (int32_t)((uint32_t)d - pred[j]);
                const int sign = sign_only(v) * error_sign;
                coefs[j] = (int16_t)(coefs[j] - sign);
                v = (int32_t)((uint32_t)v * (uint32_t)sign);
                error_val -= (uint32_t)(v >> quant) * (uint32_t)(j + 1);
            }
        }
    }
}

// The first element's header at the frame's start: its sample count (k_alac_frames)
SBA_HD Listed first_element(const uint8_t* buf, int64_t offset, int64_t limit, const Config& c) {
    Listed r; r.samples = 0; r.code = kOk;
    Bits b; b.p = buf; b.pos = offset * 8; b.end = limit * 8;
    if (b.left() < 3) { r.code = kNoEnd; return r; }
    const int tag = (int)b.read(3);
    if (tag == 7) { r.code = kNoElement; return r; }
    if (tag != 0 && tag != 1 && tag != 3) { r.code = kBadTag; return r; }
    if (b.left() < 20) { r.code = kOverrun; return r; }
    b.pos += 16;
    const int has_size = (int)b.read(1);
    b.pos += 3;
    if (has_size && b.left() < 32) { r.code = kOverrun; return r; }
    const uint32_t n = has_size ? b.read(32) : (uint32_t)c.frame_length;
    if (n == 0 || n > (uint32_t)c.frame_length) { r.code = kBadCount; return r; }
    r.samples = (int32_t)n;
    return r;
}

SBA_HD int16_t top16(int32_t v, int depth) {
    return depth == 16 ? (int16_t)v : (int16_t)(((uint32_t)v << (32 - depth)) >> 16);
}

// One element of `nch` channels whose first output channel is `ch_out`.  scratch holds 2 * frame_length int32; out
// is the frame's first interleaved int16 sample.  *nb is the frame's sample count (0 before the first element).
SBA_HD int decode_element(Bits& b, const Config& c, int nch, int ch_out, int* nb, int32_t* scratch, int16_t* out) {
    if (b.left() < 20) return kOverrun;
    b.pos += 16;                                           // element instance tag, unused header bits
    const int has_size = (int)b.read(1);
    int extra = (int)b.read(2) << 3;
    const int bps = c.bit_depth - extra + nch - 1;
    if (bps > 32 || bps < 1) return kBadElement;
    const int compressed = !b.read(1);
    if (has_size && b.left() < 32) return kOverrun;
    const uint32_t n = has_size ? b.read(32) : (uint32_t)c.frame_length;
    if (n == 0 || n > (uint32_t)c.frame_length) return kBadCount;
    if (*nb == 0) *nb = (int)n;
    else if ((int)n != *nb) return kCountMismatch;
    const int ns = (int)n;
    int shift = 0, weight = 0;
    int64_t extra_pos = 0;
    if (compressed) {
        int16_t coefs[2][32];
        int ptype[2], quant[2], rhm[2], order[2];
        if (c.kb == 0) return kBadElement;
        if (b.left() < 16) return kOverrun;
        shift = (int)b.read(8);
        weight = (int)b.read(8);
        if (nch == 2 && weight && shift > 31) return kBadElement;
        for (int ch = 0; ch < nch; ++ch) {
            if (b.left() < 16) return kOverrun;
            ptype[ch] = (int)b.read(4);
            quant[ch] = (int)b.read(4);
            rhm[ch] = (int)b.read(3);
            order[ch] = (int)b.read(5);
            if (order[ch] >= c.frame_length || !quant[ch]) return kBadElement;
            if (ptype[ch] != 0 && ptype[ch] != 15) return kBadPrediction;
            if (b.left() < 16 * order[ch]) return kOverrun;
            for (int i = order[ch] - 1; i >= 0; --i) coefs[ch][i] = (int16_t)b.read_signed(16);
        }
        if (extra) {
            if (b.left() < (int64_t)ns * nch * extra) return kOverrun;
            extra_pos = b.pos;                             // read again after the unmixing
            b.pos += (int64_t)ns * nch * extra;
        }
        for (int ch = 0; ch < nch; ++ch) {
            int32_t* s = scratch + (int64_t)ch * c.frame_length;
            const int rc = rice_decompress(b, s, ns, bps, rhm[ch] * c.pb / 4, c);
            if (rc != kOk) return rc;
            if (ptype[ch] == 15) lpc_prediction(s, ns, bps, nullptr, 31, 0);
            lpc_prediction(s, ns, bps, coefs[ch], order[ch], quant[ch]);
        }
    } else {
        if (b.left() < (int64_t)ns * nch * c.bit_depth) return kOverrun;
        for (int i = 0; i < ns; ++i)
            for (int ch = 0; ch < nch; ++ch) scratch[(int64_t)ch * c.frame_length + i] = b.read_signed(c.bit_depth);
        extra = 0;
    }
    int32_t* s0 = scratch;
    int32_t* s1 = scratch + c.frame_length;
    if (nch == 2 && weight) {
        for (int i = 0; i < ns; ++i) {
            uint32_t a = (uint32_t)s0[i], bb = (uint32_t)s1[i];
            a -= (uint32_t)((int32_t)(bb * (uint32_t)weight) >> shift);
            bb += a;
            s0[i] = (int32_t)bb;
            s1[i] = (int32_t)a;
        }
    }
    Bits e; e.p = b.p; e.pos = extra_pos; e.end = b.end;
    for (int i = 0; i < ns; ++i)
        for (int ch = 0; ch < nch; ++ch) {
            int32_t v = scratch[(int64_t)ch * c.frame_length + i];
            if (extra) v = (int32_t)(((uint32_t)v << extra) | e.read(extra));
            out[(int64_t)i * c.channels + ch_out + ch] = top16(v, c.bit_depth);
        }
    return kOk;
}

// A whole frame: its elements in bitstream order up to END.  `samples` is what k_alac_frames read from the first
// element; every element must agree with it.
SBA_HD int decode_frame(const uint8_t* buf, int64_t offset, int64_t limit, const Config& c, int samples,
                        int32_t* scratch, int16_t* out) {
    Bits b; b.p = buf; b.pos = offset * 8; b.end = limit * 8;
    int ch = 0, nb = 0;
    bool got_end = false;
    while (b.left() >= 3) {
        const int tag = (int)b.read(3);
        if (tag == 7) { got_end = true; break; }
        if (tag != 0 && tag != 1 && tag != 3) return kBadTag;
        const int nch = tag == 1 ? 2 : 1;
        if (ch + nch > c.channels || layout_offset(c.channels, ch) + nch > c.channels) return kTooManyChannels;
        const int rc = decode_element(b, c, nch, layout_offset(c.channels, ch), &nb, scratch, out);
        if (rc != kOk) return rc;
        if (nb != samples) return kCountMismatch;
        ch += nch;
    }
    if (!got_end) return kNoEnd;
    if (ch == 0) return kNoElement;
    if (ch != c.channels) return kFewChannels;
    return kOk;
}

// ---- host side: what sb_alac_decode_frames does around the kernels; the CPU build of the tests runs the same ----

// config[0..7) (frameLength, bitDepth, pb, mb, kb, channels, rate) into *c.  Returns false with a message.
inline bool parse_config(const int32_t* config, Config* c, char* msg, size_t msg_len) {
    c->frame_length = config[0]; c->bit_depth = config[1]; c->pb = config[2]; c->mb = config[3];
    c->kb = config[4]; c->channels = config[5]; c->rate = config[6];
    if (c->bit_depth != 16 && c->bit_depth != 20 && c->bit_depth != 24 && c->bit_depth != 32)
        snprintf(msg, msg_len, "ALAC with %d bits per sample is not supported (16, 20, 24 or 32)", c->bit_depth);
    else if (c->frame_length < 1 || c->frame_length > kMaxFrameLength)
        snprintf(msg, msg_len, "ALAC frameLength %d is not supported (1 to %d)", c->frame_length, kMaxFrameLength);
    else if (c->channels < 1 || c->channels > 8)
        snprintf(msg, msg_len, "ALAC with %d channels is not supported (1 to 8)", c->channels);
    else if (c->rate < 1 || c->pb < 0 || c->pb > 255 || c->mb < 0 || c->mb > 255 || c->kb < 0 || c->kb > 255)
        snprintf(msg, msg_len, "sb_alac_decode_frames: bad stream parameters");
    else
        return true;
    return false;
}

// Frame f holds bytes [offsets[f], offsets[f + 1]) of the buffer, the last up to nbytes: every frame must start
// inside the buffer and hold a byte.  `where` names each frame's file offset.  Returns false with a message.
inline bool check_offsets(const int64_t* offsets, const int64_t* where, int64_t n, int64_t nbytes, char* msg,
                          size_t msg_len) {
    for (int64_t f = 0; f < n; ++f) {
        const int64_t end = f + 1 < n ? offsets[f + 1] : nbytes;
        if (offsets[f] < 0 || offsets[f] >= nbytes)
            return sbframes::refuse(msg, msg_len, "ALAC frame", f, where[f], "frame starts outside the buffer");
        if (end <= offsets[f]) return sbframes::refuse(msg, msg_len, "ALAC frame", f, where[f], "empty frame");
    }
    return true;
}

// The frame table from what k_alac_frames read: sample positions are the prefix sum of the frames' sample counts.
// Returns false with the message of the first frame whose first element was refused.
inline bool frame_table(const Listed* listed, const int64_t* offsets, const int64_t* where, int64_t n, int64_t nbytes,
                        std::vector<FrameDesc>& frames, int64_t* samples, char* msg, size_t msg_len) {
    frames.resize((size_t)n);
    int64_t sample = 0;
    for (int64_t f = 0; f < n; ++f) {
        if (listed[f].code != kOk) return sbframes::refuse(msg, msg_len, "ALAC frame", f, where[f], error_text(listed[f].code));
        frames[(size_t)f] = FrameDesc{offsets[f], f + 1 < n ? offsets[f + 1] : nbytes, sample};
        sample += listed[f].samples;
    }
    *samples = sample;
    return true;
}

}  // namespace sbalac
