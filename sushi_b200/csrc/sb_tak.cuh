// TAK (Tom's lossless Audio Kompressor) frame decoding, written once for the kernels of sb_tak.cu and for the CPU
// (tests/emu/emu_tak_driver.cpp compiles this header with g++).  Everything here is a __host__ __device__ function of
// plain integers and byte pointers; the arithmetic is FFmpeg's `tak` decoder's, operation for operation:
//   the frame header (sync 0xA0FF, flags, frame number, optional last-frame length and stream info) and its CRC-24,
//     FFmpeg's tak parser's test for a frame start;
//   per channel: the sample shift, the raw first sample, the channel lpc mode and the subframe layout; per subframe the
//     residual codes (one mode, or a mode per window of `uval` samples), the warm-up samples with their own lpc mode,
//     and the prediction filter: predictors turned into int16 taps by FFmpeg's recurrence, the dot product over an
//     int16 history in 32-bit wrap-around, the clip to 14 bits and the shift;
//   the inter-channel decorrelation (stereo dmodes 1 to 7, multichannel pairs in list order), the channel lpc mode as
//     one to three nested prefix sums, the sample shift, and the int16 store (24-bit: the top 16 bits of FFmpeg's S32).
//
// A frame decodes in four stages (sb_tak.cu runs one kernel per stage, the emulation one loop):
//   entropy    entropy_frame: every residual into the int32 scratch, planar per frame (channel ch of frame f at
//              scratch[f.sample * channels + ch * f.nb]); per filtered subframe a Sub (where its parameters start in
//              the bitstream, its history and its length); per decorrelated pair a Pair; the data's end;
//   filter     per (frame, channel), each filtered subframe in turn: filter_taps (the recurrence, one pair step at a
//              time), then each sample's dot product as 32 lanes' lane_part summed, and finish_sample;
//   finish     decorrelate_sample per pair in list order, the lpc scans, the shift and the store;
//   CRC        crc_bytes over slices of the frame's data, joined by crc_combine, checked against the stored CRC.
// Each stage leaves a status per frame; a later stage skips a frame whose status is not kOk.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "sb_frames.h"

#if defined(__CUDACC__)
#define SBT_HD __host__ __device__ __forceinline__
#else
#define SBT_HD inline
#endif

namespace sbtak {

constexpr int kMaxChannels = 6;         // FFmpeg's decoder refuses more
constexpr int kMaxSubframes = 8;
constexpr int kMaxOrder = 256;
constexpr int kMaxFrame = 16384;          // FFmpeg's largest frame, in samples per channel
constexpr int kRing = 512;                // filter history ring (a power of two above the longest filter)
constexpr int kCodecMonoStereo = 2, kCodecMulti = 4;

enum {
    kOk = 0,
    kOverread,          // a read past the end of the frame
    kShift,             // a sample shift at or above the bit depth
    kSubframes,         // a subframe layout FFmpeg rejects
    kOrder,             // a filter order, warm-up lpc mode or filter quantisation FFmpeg rejects
    kCoding,            // a residual coding FFmpeg rejects (window count, coding mode, escape width)
    kShortDecor,        // filtered decorrelation on fewer than 256 samples
    kMcd,               // multichannel decorrelation parameters FFmpeg rejects, or that leave a channel undecoded
    kTrailing,          // bytes between the data CRC and the next frame
    kCrc,               // the data CRC disagrees
};

SBT_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kOverread: return "data runs past the frame";
    case kShift: return "sample shift at or above the bit depth";
    case kSubframes: return "invalid subframe layout";
    case kOrder: return "invalid filter order, warm-up lpc mode or filter quantisation";
    case kCoding: return "invalid residual coding";
    case kShortDecor: return "filtered decorrelation on fewer than 256 samples";
    case kMcd: return "invalid multichannel decorrelation parameters";
    case kTrailing: return "bytes left after the data CRC";
    case kCrc: return "data CRC mismatch";
    default: return "unknown error";
    }
}

// FFmpeg's predictor_sizes, xcodes (init, escape, scale, aescape, bias), mc_dmodes and frame_duration_type_quants
SBT_HD int predictor_size(int i) {
    const int16_t t[16] = {4, 8, 12, 16, 24, 32, 48, 64, 80, 96, 128, 160, 192, 224, 256, 0};
    return t[i & 15];
}
struct Code { uint32_t init, escape, scale, aescape, bias; };
SBT_HD Code xcode(int mode) {                 // mode 1..50; the table's rows 2k and 2k + 1 follow a rule from k = 2 on
    const int m = mode - 1, k = m >> 1;
    Code c;
    if (m == 0) { c.init = 1; c.escape = 1; c.scale = 1; c.aescape = 3; c.bias = 8; return c; }
    if (m == 1) { c.init = 2; c.escape = 3; c.scale = 1; c.aescape = 7; c.bias = 6; return c; }
    if (m == 2) { c.init = 3; c.escape = 5; c.scale = 2; c.aescape = 0xE; c.bias = 0xD; return c; }
    if (m & 1) {
        c.init = (uint32_t)k + 2; c.escape = 3u << (k - 1); c.scale = 3u << (k - 1);
        c.aescape = 0xDu << (k - 1); c.bias = 0x18u << (k - 1);
    } else {
        c.init = (uint32_t)k + 2; c.escape = 0xBu << (k - 2); c.scale = 1u << k;
        c.aescape = 0x1Cu << (k - 2); c.bias = 0x19u << (k - 2);
    }
    return c;
}
SBT_HD int mc_dmode(int index) { return index == 0 ? 1 : index == 1 ? 3 : index == 2 ? 4 : 6; }

// FFmpeg's tak_get_nb_samples: samples per frame of a frame size type at a rate, or 0 when FFmpeg refuses it
SBT_HD int frame_samples(int rate, int type) {
    const int q[10] = {3, 4, 6, 8, 4096, 8192, 16384, 512, 1024, 2048};
    int n, max_n;
    if (type < 0 || type > 9) return 0;
    if (type <= 3) { n = (int)((int64_t)rate * q[type] >> 5); max_n = 16384; }
    else { n = q[type]; max_n = (int)((int64_t)rate * 8 >> 5); }
    return n <= 0 || n > max_n ? 0 : n;
}

// FFmpeg's set_sample_rate_params: the residual window (uval) and the subframe length unit (subframe_scale)
SBT_HD int rate_units(int rate) { return (int)(((((int64_t)rate + 511) >> 9) + 3) & ~(int64_t)3); }
SBT_HD int uval_of(int rate) {
    const int shift = rate < 11025 ? 3 : rate < 22050 ? 2 : rate < 44100 ? 1 : 0;
    return rate_units(rate) << shift;
}
SBT_HD int subframe_scale_of(int rate) { return rate_units(rate) << 1; }

// ---- CRC-24 (poly 0x864CFB, unreflected), FFmpeg's av_crc with AV_CRC_24_IEEE from 0xCE04B7 ----
// The register R is kept as a plain 24-bit value; FFmpeg's byte-swapped 0xCE04B7 is R = 0xB704CE, and its comparison
// of the swapped register with the stored bytes read big-endian means the stored CRC is R in little-endian byte order.
constexpr uint32_t kCrcPoly = 0x864CFB, kCrcInit = 0xB704CE;
SBT_HD uint32_t crc_entry(uint32_t i) {
    uint32_t r = i << 16;
    for (int k = 0; k < 8; ++k) r = ((r << 1) ^ ((r & 0x800000u) ? kCrcPoly : 0u)) & 0xFFFFFFu;
    return r;
}
SBT_HD uint32_t crc_byte(uint32_t r, uint32_t b) {            // one byte, without a table
    r ^= b << 16;
    for (int k = 0; k < 8; ++k) r = ((r << 1) ^ ((r & 0x800000u) ? kCrcPoly : 0u)) & 0xFFFFFFu;
    return r;
}
SBT_HD uint32_t crc_mulmod(uint32_t a, uint32_t b) {          // a * b mod (x^24 + poly), GF(2)
    uint32_t r = 0;
    for (int k = 23; k >= 0; --k) {
        r = ((r << 1) ^ ((r & 0x800000u) ? kCrcPoly : 0u)) & 0xFFFFFFu;
        if ((b >> k) & 1u) r ^= a;
    }
    return r;
}
// the CRC of A followed by B, from crc(A) (any start) and crc(B) started from 0, B being len bytes
SBT_HD uint32_t crc_combine(uint32_t crc_a, uint32_t crc_b0, int64_t len) {
    uint32_t p = 1, sq = 0x100;                                  // x^(8 len) by squaring x^8
    for (int64_t n = len; n; n >>= 1) {
        if (n & 1) p = crc_mulmod(p, sq);
        sq = crc_mulmod(sq, sq);
    }
    return crc_mulmod(crc_a, p) ^ crc_b0;
}
SBT_HD uint32_t stored_crc(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16; }

// ---- the bit reader: FFmpeg's little-endian GetBitContext over bytes [0, nbytes) of the buffer ----
struct Bits {
    const uint8_t* buf;
    int64_t nbytes;          // readable bytes (zeros are read past them)
    int64_t pos;             // bit position from buf
    int64_t end;             // bit position of the frame's end: a read past it sets `over`
    bool over;

    SBT_HD uint32_t word(int64_t w) const {
        const int64_t b = 4 * w;
        if (b + 4 <= nbytes) {
#if defined(__CUDA_ARCH__)
            return __ldg(reinterpret_cast<const uint32_t*>(buf) + w);
#else
            uint32_t v;
            memcpy(&v, buf + b, 4);
            return v;
#endif
        }
        uint32_t v = 0;
        for (int k = 0; k < 4; ++k)
            if (b + k < nbytes) v |= (uint32_t)buf[b + k] << (8 * k);
        return v;
    }
    // the next n bits (n <= 32), first bit lowest, without moving
    SBT_HD uint32_t peek(int n) const {
        if (pos >= end) return 0;
        const int64_t w = pos >> 5;
        const uint64_t v = ((uint64_t)word(w + 1) << 32 | word(w)) >> (pos & 31);
        return n >= 32 ? (uint32_t)v : (uint32_t)v & ((1u << n) - 1u);
    }
    SBT_HD void skip(int n) { pos += n; if (pos > end) over = true; }
    SBT_HD uint32_t get(int n) { const uint32_t v = n ? peek(n) : 0u; skip(n); return v; }
    SBT_HD int32_t sget(int n) { const uint32_t v = get(n); return n ? (int32_t)(v << (32 - n)) >> (32 - n) : 0; }
    SBT_HD int bit() { return (int)get(1); }
    SBT_HD int esc4() { return bit() ? (int)get(4) + 1 : 0; }
    // FFmpeg's get_unary(gb, 1, len): the number of 0 bits before a 1, at most len (the 1 is not read then)
    SBT_HD int unary(int len) {
        const uint32_t v = peek(len + 1) | (1u << len);
        int z = 0;
        while (!((v >> z) & 1u)) ++z;
        skip(z < len ? z + 1 : len);
        return z;
    }
    SBT_HD void align() { pos = (pos + 7) & ~(int64_t)7; if (pos > end) over = true; }
};

// ---- the stream parameters and the frame header ----

struct Info {                 // FFmpeg's TAKStreamInfo fields a frame's decode depends on
    int32_t codec, data_type, rate, bits, channels, frame_type;
    uint32_t mask;            // the channel layout's mask, 0 when the stream gives none
    int64_t samples;
};

// FFmpeg's ff_tak_parse_streaminfo; mask_ok is false when a layout entry is outside FFmpeg's table
SBT_HD uint32_t layout_bit(int value) {
    const uint32_t t[19] = {0, 0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40, 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000,
                            0x2000, 0x4000, 0x8000, 0x10000, 0x20000};
    return value > 0 && value < 19 ? t[value] : 0u;
}
SBT_HD void parse_info(Bits& b, Info* s) {
    s->codec = (int32_t)b.get(6);
    b.skip(4);
    s->frame_type = (int32_t)b.get(4);
    const uint32_t lo = b.get(32);
    s->samples = (int64_t)lo | (int64_t)b.get(3) << 32;
    s->data_type = (int32_t)b.get(3);
    s->rate = (int32_t)b.get(18) + 6000;
    s->bits = (int32_t)b.get(5) + 8;
    s->channels = (int32_t)b.get(4) + 1;
    s->mask = 0;
    if (b.bit()) {
        b.skip(5);
        if (b.bit())
            for (int i = 0; i < s->channels; ++i) s->mask |= layout_bit((int)b.get(6));
    }
}

struct Config {
    int32_t channels, bits, rate, codec, frame_type, nb;   // nb: samples per frame but the last
    uint32_t mask;
    int64_t samples;
    int32_t uval, subframe_scale;
};

SBT_HD bool info_matches(const Info& s, const Config& c) {
    return s.codec == c.codec && s.data_type == 0 && s.rate == c.rate && s.bits == c.bits && s.channels == c.channels &&
           s.frame_type == c.frame_type && s.mask == c.mask;
}

enum { kFlagLast = 1, kFlagInfo = 2, kFlagMetadata = 4 };

// a position where FFmpeg's tak parser starts a frame: the sync word, a header that parses, and its CRC-24
struct Candidate {
    int64_t offset;
    int32_t number, flags, last, hsize;
    int32_t info_ok;          // 1: no stream info, or one that matches the stream's
    int32_t pad;
};

// the header at byte i of buf (nbytes readable), as FFmpeg's ff_tak_decode_frame_header and ff_tak_check_crc test it;
// a header with the metadata flag is returned too (flagged), so that its refusal can name it
SBT_HD bool parse_header(const uint8_t* buf, int64_t nbytes, int64_t i, const Config& c, Candidate* out) {
    if (i + 8 > nbytes || buf[i] != 0xFF || buf[i + 1] != 0xA0) return false;
    Bits b{buf, nbytes, 8 * i, 8 * nbytes, false};
    b.skip(16);
    Candidate h;
    h.offset = i;
    h.flags = (int32_t)b.get(3);
    h.number = (int32_t)b.get(21);
    h.last = 0;
    h.info_ok = 1;
    h.pad = 0;
    if (h.flags & kFlagLast) {
        h.last = (int32_t)b.get(14) + 1;
        b.skip(2);
    }
    if (h.flags & kFlagInfo) {
        Info s;
        parse_info(b, &s);
        if (b.get(6)) b.skip(25);
        b.align();
        h.info_ok = info_matches(s, c) ? 1 : 0;
    }
    b.skip(24);
    if (b.over) return false;
    h.hsize = (int32_t)(b.pos / 8 - i);
    uint32_t r = kCrcInit;
    for (int64_t k = i; k < i + h.hsize - 3; ++k) r = crc_byte(r, buf[k]);
    if (r != stored_crc(buf + i + h.hsize - 3)) return false;
    *out = h;
    return true;
}

// one frame of the table: header at `start`, data from start + hsize, the frame ending at `end` (the next frame)
struct Frame {
    int64_t start, end;
    int64_t sample;          // first sample of the frame in the stream
    int32_t nb, hsize;
};

// a filtered subframe, for the filter stage: its parameters start at bit `bits`; its history is the `order` samples
// from `hist` (in the channel), and `count` samples follow it
struct Sub {
    int64_t bits;
    int32_t hist, count, order, pad;
};

// a decorrelated channel pair, in FFmpeg's decorrelate(c1, c2) naming; its parameters start at bit `bits`
struct Pair {
    int64_t bits;
    int32_t dmode, c1, c2, pad;
};

// what the entropy stage leaves for the others
struct State {
    int64_t data_end;        // byte just past the data CRC
    int32_t npairs, raw;     // raw: a frame of fewer than 16 samples (stored as read)
    int8_t shift[kMaxChannels], lpc[kMaxChannels], nsub[kMaxChannels];
    Pair pair[kMaxChannels];
};

// config: channels, bits, rate, codec, frame size type, samples (low, high 32 bits), channel mask
inline bool parse_config(const int32_t* config, Config* c, char* msg, size_t msg_len) {
    c->channels = config[0]; c->bits = config[1]; c->rate = config[2]; c->codec = config[3];
    c->frame_type = config[4];
    c->samples = (int64_t)(uint32_t)config[5] | (int64_t)config[6] << 32;
    c->mask = (uint32_t)config[7];
    if (c->bits != 16 && c->bits != 24) {
        snprintf(msg, msg_len, "TAK with %d bits per sample is not supported (16 or 24)", c->bits);
        return false;
    }
    if (c->channels < 1 || c->channels > kMaxChannels) {
        snprintf(msg, msg_len, "TAK with %d channels is not supported (1 to %d)", c->channels, kMaxChannels);
        return false;
    }
    if ((c->codec != kCodecMonoStereo && c->codec != kCodecMulti) || (c->codec == kCodecMonoStereo && c->channels > 2)) {
        snprintf(msg, msg_len, "TAK codec type %d with %d channels is not supported", c->codec, c->channels);
        return false;
    }
    c->nb = frame_samples(c->rate, c->frame_type);
    if (c->rate < 6000 || c->rate >= 6000 + (1 << 18) || c->nb == 0 || c->samples < 1) {
        snprintf(msg, msg_len, "sb_tak_decode_file: bad stream parameters");
        return false;
    }
    c->uval = uval_of(c->rate);
    c->subframe_scale = subframe_scale_of(c->rate);
    return true;
}

// The frames, from every candidate in [audio_start, audio_end) in file order (FFmpeg's parser cuts a packet at each):
// numbered from 0, the first at audio_start carrying stream info, every stream info the stream's, none with the
// metadata flag, the last (and only the last) flagged as the last frame, and the lengths adding up to the stream's.
inline bool frame_table(const Candidate* cand, int64_t n, int64_t audio_start, int64_t audio_end, const Config& c,
                        std::vector<Frame>& frames, int64_t* samples, char* msg, size_t msg_len) {
    frames.clear();
    int64_t total = 0;
    for (int64_t k = 0; k < n; ++k) {
        const Candidate& h = cand[k];
        const int64_t f = (int64_t)frames.size();
        const char* bad = nullptr;
        if (k == 0 && h.offset != audio_start) {
            snprintf(msg, msg_len, "TAK frame 0 at byte offset %lld: no frame header where the audio starts (the first "
                     "is at byte offset %lld)", (long long)audio_start, (long long)h.offset);
            return false;
        }
        if (h.flags & kFlagMetadata) bad = "frame metadata is not supported (FFmpeg does not decode it)";
        else if (h.number != (f & ((1 << 21) - 1))) bad = "frame number out of sequence";
        else if (!h.info_ok) bad = "frame header contradicts the stream info";
        else if (f == 0 && !(h.flags & kFlagInfo)) bad = "the first frame carries no stream info";
        else if ((h.flags & kFlagLast) && k + 1 < n) bad = "a frame before the last is flagged as the last";
        else if (!(h.flags & kFlagLast) && k + 1 == n) bad = "the last frame is not flagged as the last";
        if (bad) return sbframes::refuse(msg, msg_len, "TAK frame", f, h.offset, bad);
        Frame fr;
        fr.start = h.offset;
        fr.end = k + 1 < n ? cand[k + 1].offset : audio_end;
        fr.sample = total;
        fr.nb = (h.flags & kFlagLast) ? h.last : c.nb;
        fr.hsize = h.hsize;
        total += fr.nb;
        frames.push_back(fr);
    }
    if (frames.empty()) {
        snprintf(msg, msg_len, "TAK: no frame between byte offsets %lld and %lld", (long long)audio_start,
                 (long long)audio_end);
        return false;
    }
    if (total != c.samples) {
        snprintf(msg, msg_len, "TAK: the frames hold %lld samples per channel, the stream info %lld", (long long)total,
                 (long long)c.samples);
        return false;
    }
    *samples = total;
    return true;
}

// ---- entropy ----

SBT_HD int32_t zigzag(uint32_t x) { return (int32_t)((x >> 1) ^ (0u - (x & 1u))); }

// FFmpeg's decode_segment: len residuals of coding mode `mode`
SBT_HD int segment(Bits& b, int mode, int32_t* d, int len) {
    if (mode == 0) {
        for (int i = 0; i < len; ++i) d[i] = 0;
        return kOk;
    }
    if (mode < 0 || mode > 50) return kCoding;
    const Code c = xcode(mode);
    for (int i = 0; i < len; ++i) {
        uint32_t x = b.get((int)c.init);
        if (x >= c.escape && b.bit()) {
            x |= 1u << c.init;
            if (x >= c.aescape) {
                uint32_t scale = (uint32_t)b.unary(9);
                if (scale == 9) {
                    int scale_bits = (int)b.get(3);
                    if (scale_bits > 0) {
                        if (scale_bits == 7) {
                            scale_bits += (int)b.get(5);
                            if (scale_bits > 29) return kCoding;
                        }
                        scale = b.get(scale_bits) + 1u;
                        x += c.scale * scale;
                    }
                    x += c.bias;
                } else {
                    x += c.scale * scale - c.escape;
                }
            } else {
                x -= c.escape;
            }
        }
        d[i] = zigzag(x);
        if (b.over) return kOverread;
    }
    return kOk;
}

// FFmpeg's decode_residues: length residuals, one coding mode, or one per window of uval samples
SBT_HD int residues(Bits& b, const Config& c, int nb, int32_t* d, int length) {
    if (length > nb) return kCoding;
    if (b.bit()) {
        int wlength = length / c.uval;
        int rval = length - wlength * c.uval;
        if (rval < c.uval / 2) rval += c.uval;
        else ++wlength;
        if (wlength <= 1 || wlength > 128) return kCoding;
        int8_t modes[128];
        int mode = (int)b.get(6);
        modes[0] = (int8_t)mode;
        for (int i = 1; i < wlength; ++i) {
            const int u = b.unary(6);
            if (u == 6) mode = (int)b.get(6);
            else if (u >= 3) { const int sign = b.bit(); mode += sign ? 1 - u : u - 1; }
            else if (u == 2) ++mode;
            else if (u == 1) --mode;
            modes[i] = (int8_t)mode;
        }
        if (b.over) return kOverread;
        int i = 0;
        while (i < wlength) {
            int len = 0;
            const int m = modes[i];
            do {
                len += i >= wlength - 1 ? rval : c.uval;
                ++i;
            } while (i < wlength && modes[i] == m);
            const int st = segment(b, m, d, len);
            if (st) return st;
            d += len;
        }
        return kOk;
    }
    const int st = segment(b, (int)b.get(6), d, length);
    return st ? st : b.over ? kOverread : kOk;
}

// FFmpeg's decode_lpc: `mode` (1 to 3) nested inclusive prefix sums in 32-bit wrap-around, level l from element
// mode - l, over d[0, n)
SBT_HD void lpc_serial(int32_t* d, int mode, int n) {
    for (int l = 1; l <= mode; ++l) {
        uint32_t acc = 0;
        for (int i = mode - l; i < n; ++i) {
            acc += (uint32_t)d[i];
            d[i] = (int32_t)acc;
        }
    }
}

// the filtered subframe's parameters after its layout bits: skipped here, read again by the filter stage
struct FilterParams { int dshift, quant; };
template <class Pred>
SBT_HD int filter_params(Bits& b, int order, FilterParams* p, Pred pred) {
    p->dshift = b.esc4();
    const int size = b.bit() + 6;
    p->quant = 10;
    if (b.bit()) {
        p->quant -= (int)b.get(3) + 1;
        if (p->quant < 3) return kOrder;
    }
    pred(0, (int16_t)b.sget(10));
    pred(1, (int16_t)b.sget(10));
    pred(2, (int16_t)(b.sget(size) * (1 << (10 - size))));
    pred(3, (int16_t)(b.sget(size) * (1 << (10 - size))));
    if (order > 4) {
        const int tmp = size - b.bit();
        int x = 0;
        for (int i = 4; i < order; ++i) {
            if (!(i & 3)) x = tmp - (int)b.get(2);
            pred(i, (int16_t)(b.sget(x) * (1 << (10 - size))));
        }
    }
    return b.over ? kOverread : kOk;
}
struct NoPred { SBT_HD void operator()(int, int16_t) const {} };

// FFmpeg's decode_channel up to the filters: every residual and warm-up sample of channel ch into d (nb samples), a
// Sub per filtered subframe into subs
SBT_HD int channel(Bits& b, const Config& c, int nb, int ch, int32_t* d, Sub* subs, State* s) {
    const int shift = b.esc4();
    if (shift >= c.bits) return kShift;
    s->shift[ch] = (int8_t)shift;
    d[0] = b.sget(c.bits - shift);
    s->lpc[ch] = (int8_t)b.get(2);
    const int nsub = (int)b.get(3) + 1;
    int len[kMaxSubframes];
    int left = nb - 1, prev = 0, i = 0;
    if (nsub > 1) {
        for (; i < nsub - 1; ++i) {
            const int v = (int)b.get(6);
            len[i] = (int16_t)((v - prev) * c.subframe_scale);
            if (len[i] <= 0) return b.over ? kOverread : kSubframes;
            left -= len[i];
            prev = v;
        }
        if (left <= 0) return b.over ? kOverread : kSubframes;
    }
    len[i] = left;
    int at = 1, prev_len = 0, nf = 0;
    for (i = 0; i < nsub; ++i) {
        const int sz = len[i];
        if (!b.bit()) {
            const int st = residues(b, c, nb, d + at, sz);
            if (st) return st;
        } else {
            const int order = predictor_size((int)b.get(4));
            Sub u;
            u.pad = 0;
            u.order = order;
            if (prev_len > 0 && b.bit()) {
                if (order > prev_len) return kOrder;
                u.hist = at - order;
                u.count = sz;
            } else {
                if (order > sz) return kOrder;
                const int lpc = (int)b.get(2);
                if (lpc > 2) return kOrder;
                const int st = residues(b, c, nb, d + at, order);
                if (st) return st;
                if (lpc) lpc_serial(d + at, lpc, order);
                u.hist = at;
                u.count = sz - order;
            }
            u.bits = b.pos;
            FilterParams p;
            int st = filter_params(b, order, &p, NoPred());
            if (st) return st;
            st = residues(b, c, nb, d + u.hist + order, u.count);
            if (st) return st;
            subs[nf++] = u;
        }
        at += sz;
        prev_len = sz;
    }
    s->nsub[ch] = (int8_t)nf;
    return b.over ? kOverread : kOk;
}

// the decorrelation parameters after a pair's dmode (FFmpeg's decorrelate reads them there): skipped
SBT_HD int skip_decor(Bits& b, int dmode, int nb) {
    if (dmode == 4 || dmode == 5) {
        b.esc4();
        b.skip(10);
    } else if (dmode >= 6) {
        if (nb - 1 < 256) return kShortDecor;
        b.esc4();
        const int order = 8 << b.bit();
        b.skip(2);
        int size = 0;
        for (int i = 0; i < order; ++i) {
            if (!(i & 3)) size = 14 - (int)b.get(3);
            b.skip(size);
        }
    }
    return b.over ? kOverread : kOk;
}

// Stage 1 of a frame: its residuals into the frame's scratch, its Subs (kMaxSubframes per channel) and its State
SBT_HD int entropy_frame(const uint8_t* buf, int64_t nbytes, const Frame& f, const Config& c, int32_t* scratch,
                         Sub* subs, State* s) {
    Bits b{buf, nbytes, 8 * (f.start + f.hsize), 8 * f.end, false};
    int32_t* base = scratch + f.sample * c.channels;
    const int nb = f.nb;
    s->npairs = 0;
    s->raw = nb < 16;
    for (int ch = 0; ch < c.channels; ++ch) { s->shift[ch] = 0; s->lpc[ch] = 0; s->nsub[ch] = 0; }
    if (nb < 16) {
        for (int ch = 0; ch < c.channels; ++ch)
            for (int i = 0; i < nb; ++i) base[ch * nb + i] = b.sget(c.bits);
    } else if (c.codec == kCodecMonoStereo) {
        for (int ch = 0; ch < c.channels; ++ch) {
            const int st = channel(b, c, nb, ch, base + ch * nb, subs + ch * kMaxSubframes, s);
            if (st) return st;
        }
        if (c.channels == 2) {
            if (b.bit()) b.skip(6);
            Pair& p = s->pair[0];
            p.dmode = (int32_t)b.get(3);
            p.c1 = 0; p.c2 = 1; p.pad = 0;
            p.bits = b.pos;
            const int st = skip_decor(b, p.dmode, nb);
            if (st) return st;
            s->npairs = p.dmode ? 1 : 0;
        }
    } else {
        int n = c.channels;
        int8_t c1[16], c2[16], present[16], index[16];
        if (b.bit()) {
            n = (int)b.get(4) + 1;
            if (n > c.channels) return b.over ? kOverread : kMcd;
            int mask = 0;
            for (int i = 0; i < n; ++i) {
                const int nbit = (int)b.get(4);
                if (nbit >= c.channels || (mask & (1 << nbit))) return b.over ? kOverread : kMcd;
                present[i] = (int8_t)b.bit();
                if (present[i]) {
                    index[i] = (int8_t)b.get(2);
                    c2[i] = (int8_t)b.get(4);
                    if (c2[i] >= c.channels) return b.over ? kOverread : kMcd;
                    if (index[i] == 1) {
                        if (nbit == c2[i] || (mask & (1 << c2[i]))) return b.over ? kOverread : kMcd;
                        mask |= 1 << c2[i];
                    } else if (!(mask & (1 << c2[i]))) {
                        return b.over ? kOverread : kMcd;
                    }
                }
                c1[i] = (int8_t)nbit;
                mask |= 1 << nbit;
            }
            // FFmpeg leaves a channel the list does not reach as it finds its buffer; refused here
            if (mask != (1 << c.channels) - 1) return b.over ? kOverread : kMcd;
        } else {
            for (int i = 0; i < n; ++i) { present[i] = 0; c1[i] = (int8_t)i; }
        }
        if (b.over) return kOverread;
        for (int i = 0; i < n; ++i) {
            if (present[i] && index[i] == 1) {
                const int st = channel(b, c, nb, c2[i], base + c2[i] * nb, subs + c2[i] * kMaxSubframes, s);
                if (st) return st;
            }
            int st = channel(b, c, nb, c1[i], base + c1[i] * nb, subs + c1[i] * kMaxSubframes, s);
            if (st) return st;
            if (present[i]) {
                Pair& p = s->pair[s->npairs++];
                p.dmode = mc_dmode(index[i]);
                p.c1 = c2[i]; p.c2 = c1[i]; p.pad = 0;
                p.bits = b.pos;
                st = skip_decor(b, p.dmode, nb);
                if (st) return st;
            }
        }
    }
    b.align();
    b.skip(24);
    if (b.over) return kOverread;
    s->data_end = b.pos / 8;
    if (s->data_end != f.end) return kTrailing;
    return kOk;
}

// ---- filter ----

// A filtered subframe's parameters at Sub.bits: dshift, quantisation and the predictors (pred[0, order))
SBT_HD int read_filter(const uint8_t* buf, int64_t nbytes, int64_t bits, int order, int16_t* pred, FilterParams* p) {
    Bits b{buf, nbytes, bits, bits + 64 + 16 * order, false};
    return filter_params(b, order, p, [pred](int i, int16_t v) { pred[i] = v; });
}

// FFmpeg's predictor-to-filter recurrence, step i (1 <= i < order), pair j (j < (i + 1) / 2): the pairs of one step
// are independent, so they may run in any order or at once
SBT_HD void taps_pair(int32_t* t, int i, int j, int16_t p) {
    const uint32_t a = (uint32_t)t[j], z = (uint32_t)t[i - 1 - j];
    const int32_t x = (int32_t)(a + (uint32_t)((int32_t)((uint32_t)(int32_t)p * z + 256u) >> 9));
    t[i - 1 - j] = (int32_t)(z + (uint32_t)((int32_t)((uint32_t)(int32_t)p * a + 256u) >> 9));
    t[j] = x;
}
// tap k of the filter from the recurrence's result t
SBT_HD int16_t tap(const int32_t* t, int order, int quant, int k) {
    const int sh = 15 - quant;
    const uint32_t x = 1u << (32 - sh);
    const int32_t y = 1 << (sh - 1);
    return (int16_t)(x - (uint32_t)((int32_t)((uint32_t)t[order - 1 - k] + (uint32_t)y) >> sh));
}
SBT_HD void filter_taps_serial(const int16_t* pred, int order, int quant, int32_t* t, int16_t* filter) {
    if (order > 0) t[0] = pred[0] * 64;
    for (int i = 1; i < order; ++i) {
        for (int j = 0; j < (i + 1) / 2; ++j) taps_pair(t, i, j, pred[i]);
        t[i] = pred[i] * 64;
    }
    for (int k = 0; k < order; ++k) filter[k] = tap(t, order, quant, k);
}

// lane `lane`'s share of the dot product for output t of a subframe: taps lane, lane + 32, ... over the history ring
// (ring[(t + k) % kRing] is history value t + k)
SBT_HD uint32_t lane_part(const int16_t* ring, const int16_t* filter, int order, int64_t t, int lane) {
    uint32_t v = 0;
    for (int k = lane; k < order; k += 32) v += (uint32_t)((int32_t)ring[(t + k) & (kRing - 1)] * filter[k]);
    return v;
}
// the output sample from the dot product and its residual
SBT_HD int32_t finish_sample(uint32_t dot, int quant, int dshift, int32_t resid) {
    int32_t v = (int32_t)(dot + (1u << (quant - 1))) >> quant;
    v = v < -8192 ? -8192 : v > 8191 ? 8191 : v;
    return (int32_t)((uint32_t)v * (1u << dshift) - (uint32_t)resid);
}

// FFmpeg's filter loop as it writes it, one sample at a time over a plain history: the reference the warp-split
// filter is held to (host code)
inline void filter_serial(int32_t* d, int order, int count, int quant, int dshift, const int16_t* filter) {
    std::vector<int16_t> res((size_t)(order + count));
    for (int i = 0; i < order; ++i) res[i] = (int16_t)(d[i] >> dshift);
    for (int i = 0; i < count; ++i) {
        uint32_t v = 1u << (quant - 1);
        for (int j = 0; j < order; ++j) v += (uint32_t)((int32_t)res[i + j] * filter[j]);
        int32_t w = (int32_t)v >> quant;
        w = w < -8192 ? -8192 : w > 8191 ? 8191 : w;
        const int32_t out = (int32_t)((uint32_t)w * (1u << dshift) - (uint32_t)d[order + i]);
        d[order + i] = out;
        res[order + i] = (int16_t)(out >> dshift);
    }
}

// ---- finish ----

// the decorrelation parameters of a pair, read at Pair.bits
struct Decor {
    int dmode, dshift, dfactor, order, dval1, dval2;
    int16_t filter[16];
};
SBT_HD void read_decor(const uint8_t* buf, int64_t nbytes, const Pair& p, Decor* d) {
    Bits b{buf, nbytes, p.bits, p.bits + 512, false};
    d->dmode = p.dmode;
    d->dshift = d->dfactor = d->order = d->dval1 = d->dval2 = 0;
    if (p.dmode == 4 || p.dmode == 5) {
        d->dshift = b.esc4();
        d->dfactor = b.sget(10);
    } else if (p.dmode >= 6) {
        d->dshift = b.esc4();
        d->order = 8 << b.bit();
        d->dval1 = b.bit();
        d->dval2 = b.bit();
        int size = 0;
        for (int i = 0; i < d->order; ++i) {
            if (!(i & 3)) size = 14 - (int)b.get(3);
            d->filter[i] = (int16_t)b.sget(size);
        }
    }
}

// Sample i of one pair's decorrelation (FFmpeg's decorrelate and its takdsp functions), writing only sample i of the
// channel(s) it changes and reading only sample i, or (filtered modes) the unchanged channel: so every i may run at
// once.  a = channel c1, b = channel c2, nb samples each.  Sample 0 is never changed.
SBT_HD void decorrelate_sample(const Decor& d, int32_t* a, int32_t* b, int nb, int i) {
    if (i == 0) return;
    switch (d.dmode) {
    case 1: b[i] = (int32_t)((uint32_t)a[i] + (uint32_t)b[i]); break;
    case 2: a[i] = (int32_t)((uint32_t)b[i] - (uint32_t)a[i]); break;
    case 3: {
        const uint32_t x = (uint32_t)a[i] - (uint32_t)(b[i] >> 1);
        const uint32_t y = x + (uint32_t)b[i];
        a[i] = (int32_t)x;
        b[i] = (int32_t)y;
        break;
    }
    case 4: case 5: {
        int32_t* p1 = d.dmode == 4 ? b : a;
        const int32_t* p2 = d.dmode == 4 ? a : b;
        const int32_t v = (int32_t)(d.dfactor * (uint32_t)(p2[i] >> d.dshift) + 128u) >> 8;
        p1[i] = (int32_t)(((uint32_t)v << d.dshift) - (uint32_t)p1[i]);
        break;
    }
    case 6: case 7: {
        int32_t* p1 = (d.dmode == 6 ? b : a) + 1;          // FFmpeg's pointers for these modes start at sample 1
        const int32_t* p2 = (d.dmode == 6 ? a : b) + 1;
        const int m = i - 1, length = nb - 1, half = d.order / 2, length2 = length - (d.order - 1);
        if (m < half) {
            if (d.dval1) p1[m] = (int32_t)((uint32_t)p1[m] + (uint32_t)p2[m]);
        } else if (m >= length2 + half) {
            if (d.dval2) p1[m] = (int32_t)((uint32_t)p1[m] + (uint32_t)p2[m]);
        } else {
            const int s = m - half;
            uint32_t v = 1u << 9;
            for (int k = 0; k < d.order; ++k) v += (uint32_t)((int32_t)(int16_t)(p2[s + k] >> d.dshift) * d.filter[k]);
            int32_t w = (int32_t)v >> 10;
            w = w < -8192 ? -8192 : w > 8191 ? 8191 : w;
            p1[m] = (int32_t)((uint32_t)w * (1u << d.dshift) - (uint32_t)p1[m]);
        }
        break;
    }
    default: break;
    }
}

// the stored sample: 16-bit as is (FFmpeg's S16P), 24-bit as the top 16 bits of FFmpeg's S32P (the sample times 256)
SBT_HD int16_t store(int32_t v, int shift, int bits) {
    const uint32_t x = (uint32_t)v << shift;
    return bits == 16 ? (int16_t)(uint16_t)x : (int16_t)(uint16_t)(x >> 8);
}

// ---- CRC ----

// the CRC-24 register over bytes [lo, hi) of buf from register r, with a table of crc_entry
SBT_HD uint32_t crc_bytes(const uint8_t* buf, int64_t lo, int64_t hi, uint32_t r, const uint32_t* table) {
    for (int64_t k = lo; k < hi; ++k) r = ((r << 8) & 0xFFFFFFu) ^ table[((r >> 16) ^ buf[k]) & 0xFF];
    return r;
}

}  // namespace sbtak
