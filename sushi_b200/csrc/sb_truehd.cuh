// Dolby TrueHD decoding, written once for the GPU kernels of sb_truehd.cu and for the CPU (tests/emu/emu_truehd_driver.cpp
// compiles this header with g++).  Everything here is a __host__ __device__ function of plain integers and byte
// pointers: the bit reader, the access-unit (AU) header and its check nibble, the major sync and its CRC, the substream
// directory, the restart header and its checksum, the decoding parameters (block size, matrices, output shifts, quant
// steps, FIR / IIR filters with IIR state, Huffman offset and codebook), the block data (three Huffman codebooks and raw
// LSBs), FIR / IIR prediction, rematrixing with LSB bypass and the noise of noise type 0, the end-of-stream marker, the
// substream parity / CRC and the lossless check.
//
// The decoded presentation is the one FFmpeg's decoder gives without a downmix: substream min(n - 1, 2), in the channel
// layout of the major sync's 13-bit (8-channel presentation) field; lower substreams are decoded too (their channels
// feed the same sample buffer), higher ones (the object substream of a 4-substream stream) are skipped by their end
// pointers.  Samples are 24-bit; the loader keeps their top 16 bits.
//
// A restart segment is a major-sync AU whose decoded substreams all open with a restart header, and the AUs up to the
// next one.  One thread decodes one segment from a fresh decoder's state: a restart resets every parameter but not the
// FIR / IIR history, so the decoder refuses a segment (other than the stream's first) whose prediction reaches back past
// its restart; the lossless check in the next restart header catches any other disagreement.
//
// Widths: byte and bit positions are 64-bit; accumulators are 64-bit as in FFmpeg.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>

#if defined(__CUDACC__)
#define SBT_HD __host__ __device__ __forceinline__
#else
#define SBT_HD inline
#endif

namespace sbthd {

constexpr int kMaxAu = 160;          // samples per AU at 192 kHz
constexpr int kMaxCh = 8;            // matrix channels plus the two noise channels of noise type 0
constexpr int kMaxSub = 3;           // decoded substreams
constexpr uint32_t kNoCheck = 0xFFFFFFFFu;

enum {
    kOk = 0,
    kTruncated, kBadLength, kBadNibble, kBadSyncCrc, kFormatChange, kMlp, kBadDirectory, kNoRestart,
    kBadRestart, kBadRestartCrc, kBadParams, kBadHuffman, kOverrun, kBadEnd, kBadParity, kBadCrc, kLossless,
    kShortAu, kHistory, kAfterEnd, kBadChain,
};

SBT_HD const char* error_text(int code) {
    switch (code) {
    case kOk: return "ok";
    case kTruncated: return "truncated access unit";
    case kBadLength: return "access unit length runs past its block or the file";
    case kBadNibble: return "access unit check nibble mismatch";
    case kBadSyncCrc: return "major sync CRC mismatch";
    case kFormatChange: return "major sync changes the stream format";
    case kMlp: return "MLP (DVD-Audio) major sync, not TrueHD";
    case kBadDirectory: return "invalid substream directory";
    case kNoRestart: return "restart segment starts without a restart header";
    case kBadRestart: return "invalid restart header";
    case kBadRestartCrc: return "restart header checksum mismatch";
    case kBadParams: return "invalid decoding parameters";
    case kBadHuffman: return "invalid Huffman code";
    case kOverrun: return "block data runs past its substream";
    case kBadEnd: return "substream does not end where its end pointer says";
    case kBadParity: return "substream parity mismatch";
    case kBadCrc: return "substream CRC mismatch";
    case kLossless: return "lossless check mismatch";
    case kShortAu: return "short access unit before the end of the stream";
    case kHistory: return "prediction reaches back past a restart";
    case kAfterEnd: return "data after the end-of-stream marker";
    case kBadChain: return "access units do not land on the next restart segment";
    default: return "unknown error";
    }
}

// ---- checks --------------------------------------------------------------------------------------------------------
SBT_HD uint32_t crc8_step(uint32_t poly, uint32_t c) {
    for (int b = 0; b < 8; ++b) c = (c & 0x80) ? ((c << 1) ^ poly) & 0xFF : (c << 1) & 0xFF;
    return c;
}
SBT_HD uint8_t xor_bytes(const uint8_t* p, int64_t n) {
    uint8_t x = 0;
    for (int64_t i = 0; i < n; ++i) x ^= p[i];
    return x;
}
// major sync CRC-16 (polynomial 0x2D) of bytes [0, n - 2), XORed with the big-endian word at n - 2
SBT_HD uint32_t checksum16(const uint8_t* p, int n) {
    uint32_t c = 0;
    for (int i = 0; i < n - 2; ++i) {
        c ^= (uint32_t)p[i] << 8;
        for (int b = 0; b < 8; ++b) c = (c & 0x8000) ? ((c << 1) ^ 0x2D) & 0xFFFF : (c << 1) & 0xFFFF;
    }
    return c ^ ((uint32_t)p[n - 2] << 8 | p[n - 1]);
}
// substream check byte: CRC-8 (0x63) from 0x3C over bytes [0, n - 1), XORed with the last
SBT_HD uint32_t checksum8(const uint8_t* p, int64_t n) {
    uint32_t c = 0x3C;
    for (int64_t i = 0; i + 1 < n; ++i) c = crc8_step(0x63, c ^ p[i]);
    return c ^ p[n - 1];
}
// restart header check byte over bit_size bits after the substream's first two bits
SBT_HD uint32_t restart_checksum(const uint8_t* buf, int64_t bit_size) {
    const int64_t nb = (bit_size + 2) / 8;
    uint32_t crc = crc8_step(0x1D, buf[0] & 0x3F);
    for (int64_t i = 1; i < nb - 1; ++i) crc = crc8_step(0x1D, crc ^ buf[i]);
    crc ^= buf[nb - 1];
    for (int i = 0; i < (int)((bit_size + 2) & 7); ++i) {
        crc <<= 1;
        if (crc & 0x100) crc ^= 0x11D;
        crc ^= (buf[nb] >> (7 - i)) & 1;
    }
    return crc & 0xFF;
}
SBT_HD uint32_t xor8(uint32_t v) { v ^= v >> 16; v ^= v >> 8; return v & 0xFF; }

// ---- bit reader ----------------------------------------------------------------------------------------------------
// MSB-first over p[start, start + nbytes); reads past the end give zeros and set `over`
struct Bits {
    const uint8_t* p;
    int64_t nbits, pos;
    SBT_HD void init(const uint8_t* base, int64_t nbytes) { p = base; nbits = nbytes * 8; pos = 0; }
    SBT_HD uint32_t get(int n) {                 // 0 <= n <= 32: the 5 bytes holding the bits, zeros past the end
        if (n == 0) return 0;
        const int64_t byte = pos >> 3, nbytes = nbits >> 3;
        uint64_t w = 0;
        if (byte + 5 <= nbytes) {
            w = (uint64_t)p[byte] << 32 | (uint64_t)p[byte + 1] << 24 | (uint64_t)p[byte + 2] << 16 |
                (uint64_t)p[byte + 3] << 8 | p[byte + 4];
        } else {
            for (int i = 0; i < 5; ++i) w = (w << 8) | (byte + i < nbytes ? p[byte + i] : 0);
        }
        const uint32_t v = (uint32_t)((w >> (40 - (int)(pos & 7) - n)) & ((1ull << n) - 1));
        pos += n;
        return v;
    }
    SBT_HD int32_t sget(int n) {
        if (n == 0) return 0;
        const uint32_t v = get(n);
        return n == 32 ? (int32_t)v : (int32_t)(v << (32 - n)) >> (32 - n);
    }
    SBT_HD uint32_t peek(int n) { const int64_t s = pos; const uint32_t v = get(n); pos = s; return v; }
    SBT_HD bool over() const { return pos > nbits; }
};

// ---- stream format -------------------------------------------------------------------------------------------------
SBT_HD uint32_t rb32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
SBT_HD int sync_size(const uint8_t* s) { return (s[25] & 1) ? 28 + 2 + (s[26] >> 4) * 2 : 28; }
SBT_HD int rate_of(int code) { return code == 0xF ? 0 : ((code & 8) ? 44100 : 48000) << (code & 7); }

// What the first major sync fixes for the whole stream (the host fills it; a later major sync must agree)
struct Format {
    uint8_t fmt[4];                  // bytes 4..7 of the major sync: rate and the channel arrangements
    int32_t rate, spa, n_sub, out_sub, channels;
    int8_t code_to_out[kMaxSub][kMaxCh];  // restart-header channel code -> channel of the substream's layout (-1: none)
};

// ---- decoder state -------------------------------------------------------------------------------------------------
struct Chan {
    int32_t fir_coeff[8], iir_coeff[4], fir_hist[8], iir_hist[4];
    int32_t huff_offset, sho;
    int8_t fir_order, iir_order, fir_shift, iir_shift, codebook, huff_lsbs;
    int8_t known, known_iir;         // samples of FIR / IIR history decoded in this segment (or given by IIR state)
};
struct Sub {
    Chan ch[kMaxCh];
    int32_t coeff[8][kMaxCh + 2];
    uint32_t seed, check;
    int8_t min_ch, max_ch, max_mat, noise_type, noise_shift, presence, n_mat, data_check;
    int8_t mat_out[8], bypass[8], mat_noise[8], out_shift[kMaxCh], quant[kMaxCh], assign[kMaxCh];
    int16_t blocksize, blockpos;
    int8_t restart_seen, eos, restarted, pad;
    uint32_t stored_check;           // the lossless check byte of the last restart header (first one of the segment)
};
struct State {
    Sub sub[kMaxSub];
    int32_t buf[kMaxAu][kMaxCh];     // shared sample buffer of all decoded substreams
    uint8_t byp[kMaxAu][8];
};

SBT_HD void sign_huff(Chan& c, int q) {
    const int lsb = c.huff_lsbs - q;
    const int sh = lsb + (c.codebook ? 2 - c.codebook : -1);
    int32_t v = c.huff_offset;
    if (c.codebook) v -= 7 << lsb;
    if (sh >= 0) v -= 1 << sh;
    c.sho = v;
}

// Huffman codebooks 1..3 -> symbol 0..17: symbols 0..6 are 0..01 (9 down to 3 bits), then a middle group (1xx, 1x or
// 1), then the tail 011, 0101, 01001, ... 010000001
SBT_HD int huff_decode(Bits& br, int cb) {
    const uint32_t v = br.peek(9);
    if (v < 0x80) {
        if (v == 0) return -1;
        int z = 0;
        while (!((v << z) & 0x100)) ++z;
        br.pos += z + 1;
        return 8 - z;
    }
    if (v & 0x100) {
        if (cb == 1) { br.pos += 3; return 7 + (int)((v >> 6) & 3); }
        if (cb == 2) { br.pos += 2; return 7 + (int)((v >> 7) & 1); }
        br.pos += 1;
        return 7;
    }
    int z = 0;                                    // after 01: zeros before the closing 1
    while (z < 7 && !((v >> (6 - z)) & 1)) ++z;
    if (z == 7) return -1;
    br.pos += 3 + z;
    return 7 + (cb == 1 ? 4 : cb == 2 ? 2 : 1) + z;
}

// restart header; `sbuf` is the substream data (the checksum runs from its start)
SBT_HD int restart_header(Bits& br, const uint8_t* sbuf, const Format& f, int substr, Sub& s) {
    const int64_t start = br.pos;
    if (br.get(13) != (0x31EA >> 1)) return kBadRestart;
    s.noise_type = (int8_t)br.get(1);
    br.get(16);
    const int minc = (int)br.get(4), maxc = (int)br.get(4), maxm = (int)br.get(4);
    if (maxm > 7 || maxc != maxm || (maxm > 5 && !s.noise_type) || minc > maxc) return kBadRestart;
    if (substr == f.out_sub && maxm + 1 != f.channels) return kBadRestart;
    s.min_ch = (int8_t)minc; s.max_ch = (int8_t)maxc; s.max_mat = (int8_t)maxm;
    s.noise_shift = (int8_t)br.get(4);
    s.seed = br.get(23);
    br.get(19);
    s.data_check = (int8_t)br.get(1);
    const uint32_t lossless = br.get(8);
    br.get(16);
    for (int c = 0; c < kMaxCh; ++c) s.assign[c] = 0;
    for (int c = 0; c <= maxm; ++c) {
        const int code = (int)br.get(6);
        const int out = code < kMaxCh ? f.code_to_out[substr][code] : -1;
        if (out < 0 || out > maxm) return kBadRestart;
        s.assign[out] = (int8_t)c;
    }
    const uint32_t sum = restart_checksum(sbuf, br.pos - start);
    if (br.get(8) != sum) return kBadRestartCrc;
    if (br.over()) return kOverrun;
    // the previous run's lossless check (of the output substream)
    if (substr == f.out_sub) {
        if (s.restarted && s.check != kNoCheck && xor8(s.check) != lossless) return kLossless;
        if (!s.restarted) s.stored_check = lossless;
    }
    s.restarted = 1;
    s.presence = (int8_t)0xFF;
    s.n_mat = 0;
    s.blocksize = 8;
    s.check = 0;
    for (int c = 0; c < kMaxCh; ++c) { s.out_shift[c] = 0; s.quant[c] = 0; }
    for (int c = minc; c <= maxc; ++c) {
        Chan& ch = s.ch[c];
        ch.fir_order = ch.iir_order = 0; ch.fir_shift = ch.iir_shift = 0;
        ch.huff_offset = 0; ch.sho = -(1 << 23); ch.codebook = 0; ch.huff_lsbs = 24;
    }
    return kOk;
}

SBT_HD int filter_params(Bits& br, Chan& ch, bool iir, int8_t* changed) {
    if ((*changed)++ > 1) return kBadParams;
    const int order = (int)br.get(4);
    if (order > (iir ? 4 : 8)) return kBadParams;
    if (iir) ch.iir_order = (int8_t)order; else ch.fir_order = (int8_t)order;
    if (order > 0) {
        const int shift = (int)br.get(4);
        if (iir) ch.iir_shift = (int8_t)shift; else ch.fir_shift = (int8_t)shift;
        const int cbits = (int)br.get(5), cshift = (int)br.get(3);
        if (cbits < 1 || cbits > 16 || cbits + cshift > 16) return kBadParams;
        for (int i = 0; i < order; ++i) {
            const int32_t v = br.sget(cbits) * (1 << cshift);
            if (iir) ch.iir_coeff[i] = v; else ch.fir_coeff[i] = v;
        }
        if (br.get(1)) {
            if (!iir) return kBadParams;
            const int sbits = (int)br.get(4), sshift = (int)br.get(4);
            for (int i = 0; i < order; ++i) ch.iir_hist[i] = sbits ? br.sget(sbits) * (1 << sshift) : 0;
            if (ch.known_iir < order) ch.known_iir = (int8_t)order;
        }
    }
    return kOk;
}

// decoding parameters of a block
SBT_HD int decoding_params(Bits& br, const Format& f, Sub& s, int8_t (*fchanged)[2], int* mchanged) {
    if (s.presence & 0x01)
        if (br.get(1)) s.presence = (int8_t)br.get(8);
    const int pres = s.presence & 0xFF;
    if (pres & 0x80)
        if (br.get(1)) {
            s.blocksize = (int16_t)br.get(9);
            if (s.blocksize < 8 || s.blocksize > f.spa) return kBadParams;
        }
    if (pres & 0x40)
        if (br.get(1)) {
            if ((*mchanged)++ > 1) return kBadParams;
            s.n_mat = (int8_t)br.get(4);
            if (s.n_mat > 8) return kBadParams;
            for (int m = 0; m < s.n_mat; ++m) {
                s.mat_out[m] = (int8_t)br.get(4);
                const int frac = (int)br.get(4);
                s.bypass[m] = (int8_t)br.get(1);
                if (s.mat_out[m] > s.max_mat || frac > 14) return kBadParams;
                const int maxc = s.max_mat + (s.noise_type ? 0 : 2);
                for (int c = 0; c <= maxc; ++c) s.coeff[m][c] = br.get(1) ? br.sget(frac + 2) * (1 << (14 - frac)) : 0;
                for (int c = maxc + 1; c < kMaxCh + 2; ++c) s.coeff[m][c] = 0;
                s.mat_noise[m] = s.noise_type ? (int8_t)br.get(4) : 0;
                if (s.mat_noise[m]) return kBadParams;              // noise of type 1 is not decoded here
            }
        }
    if (pres & 0x20)
        if (br.get(1))
            for (int c = 0; c <= s.max_mat; ++c) {
                const int v = br.sget(4);
                if (v < 0) return kBadParams;
                s.out_shift[c] = (int8_t)v;
            }
    unsigned recompute = 0;
    if (pres & 0x10)
        if (br.get(1))
            for (int c = 0; c <= s.max_ch; ++c) { s.quant[c] = (int8_t)br.get(4); recompute |= 1u << c; }
    for (int c = s.min_ch; c <= s.max_ch; ++c)
        if (br.get(1)) {
            recompute |= 1u << c;
            Chan& ch = s.ch[c];
            int rc;
            if (pres & 0x08)
                if (br.get(1) && (rc = filter_params(br, ch, false, &fchanged[c][0])) != kOk) return rc;
            if (pres & 0x04)
                if (br.get(1) && (rc = filter_params(br, ch, true, &fchanged[c][1])) != kOk) return rc;
            if (ch.fir_order + ch.iir_order > 8) return kBadParams;
            if (ch.fir_order && ch.iir_order && ch.fir_shift != ch.iir_shift) return kBadParams;
            if (!ch.fir_order && ch.iir_order) ch.fir_shift = ch.iir_shift;
            if (pres & 0x02)
                if (br.get(1)) ch.huff_offset = br.sget(15);
            ch.codebook = (int8_t)br.get(2);
            ch.huff_lsbs = (int8_t)br.get(5);
            if (ch.huff_lsbs > 24) return kBadParams;
        }
    for (int c = 0; c <= s.max_ch; ++c)
        if (recompute & (1u << c)) {
            Chan& ch = s.ch[c];
            // FFmpeg refuses this for codebooks 1-3 only; with codebook 0 it would read a negative LSB count
            if (ch.huff_lsbs < s.quant[c]) return kBadParams;
            sign_huff(ch, s.quant[c]);
        }
    return br.over() ? kOverrun : kOk;
}

SBT_HD int block_data(Bits& br, const Format& f, Sub& s, State& st) {
    int64_t expect = 0;
    if (s.data_check) { expect = br.pos; expect += br.get(16); }
    if (s.blockpos + s.blocksize > f.spa) return kBadParams;
    const int bp = s.blockpos, n = s.blocksize;
    for (int i = 0; i < n; ++i) {
        for (int m = 0; m < 8; ++m) st.byp[bp + i][m] = 0;
        for (int m = 0; m < s.n_mat; ++m)
            if (s.bypass[m]) st.byp[bp + i][m] = (uint8_t)br.get(1);
        for (int c = s.min_ch; c <= s.max_ch; ++c) {
            const Chan& ch = s.ch[c];
            const int q = s.quant[c];
            const int lsb = ch.huff_lsbs - q;
            int32_t v = 0;
            if (ch.codebook > 0) {
                v = huff_decode(br, ch.codebook);
                if (v < 0) return kBadHuffman;
            }
            if (lsb > 0) v = (int32_t)(((uint32_t)v << lsb) + br.get(lsb));
            v += ch.sho;
            st.buf[bp + i][c] = (int32_t)((uint32_t)v << q);
        }
        if (br.over()) return kOverrun;
    }
    // FIR / IIR prediction
    for (int c = s.min_ch; c <= s.max_ch; ++c) {
        Chan& ch = s.ch[c];
        const int32_t mask = (int32_t)(0u - (1u << s.quant[c]));
        for (int i = 0; i < n; ++i) {
            if (ch.fir_order > ch.known || ch.iir_order > ch.known_iir) return kHistory;
            int64_t acc = 0;
            for (int k = 0; k < ch.fir_order; ++k) acc += (int64_t)ch.fir_hist[k] * ch.fir_coeff[k];
            for (int k = 0; k < ch.iir_order; ++k) acc += (int64_t)ch.iir_hist[k] * ch.iir_coeff[k];
            acc >>= ch.fir_shift;
            const int32_t res = (int32_t)((acc + st.buf[bp + i][c]) & (int64_t)mask);
            for (int k = 7; k > 0; --k) ch.fir_hist[k] = ch.fir_hist[k - 1];
            for (int k = 3; k > 0; --k) ch.iir_hist[k] = ch.iir_hist[k - 1];
            ch.fir_hist[0] = res;
            ch.iir_hist[0] = (int32_t)(res - acc);
            st.buf[bp + i][c] = res;
            if (ch.known < 8) ++ch.known;
            if (ch.known_iir < 4) ++ch.known_iir;
        }
    }
    s.blockpos = (int16_t)(bp + n);
    if (s.data_check) {
        if (br.pos != expect) return kOverrun;
        br.get(8);
    }
    return kOk;
}

// one substream of one AU
SBT_HD int decode_substream(const uint8_t* sbuf, int64_t len, bool parity, const Format& f, int substr, State& st) {
    Sub& s = st.sub[substr];
    Bits br;
    br.init(sbuf, len);
    int8_t fchanged[kMaxCh][2];
    for (int c = 0; c < kMaxCh; ++c) fchanged[c][0] = fchanged[c][1] = 0;
    int mchanged = 0;
    s.blockpos = 0;
    int rc;
    do {
        if (br.get(1)) {
            if (br.get(1)) {
                if ((rc = restart_header(br, sbuf, f, substr, s)) != kOk) return rc;
                s.restart_seen = 1;
            }
            if (!s.restart_seen) return kNoRestart;
            if ((rc = decoding_params(br, f, s, fchanged, &mchanged)) != kOk) return rc;
        }
        if (!s.restart_seen) return kNoRestart;
        if ((rc = block_data(br, f, s, st)) != kOk) return rc;
        if (br.pos >= len * 8) return kOverrun;
    } while (!br.get(1));
    br.pos += (-br.pos) & 15;
    s.eos = 0;
    if (len * 8 - br.pos >= 32) {
        if (br.get(16) != 0xD234) return kBadEnd;
        const int shorten = (int)br.get(16);
        if (shorten & 0x2000) s.blockpos = (int16_t)(s.blockpos - ((shorten & 0x1FFF) < s.blockpos ? (shorten & 0x1FFF) : s.blockpos));
        s.eos = 1;
    }
    if (parity) {
        if (len * 8 - br.pos != 16) return kBadEnd;
        const uint32_t p = br.get(8), c = br.get(8);
        if ((p ^ xor_bytes(sbuf, len - 2)) != 0xA9) return kBadParity;
        if (c != checksum8(sbuf, len - 2)) return kBadCrc;
    }
    if (br.pos != len * 8) return kBadEnd;
    return kOk;
}

// rematrix and pack the output substream of an AU into out[i * channels + out_ch]; the lossless check accumulates
SBT_HD void output(const Format& f, State& st, int16_t* out) {
    Sub& s = st.sub[f.out_sub];
    const int n = s.blockpos;
    int maxc = s.max_mat;
    if (!s.noise_type) {
        uint32_t seed = s.seed;
        for (int i = 0; i < n; ++i) {
            const uint32_t s7 = (seed >> 7) & 0xFFFF;
            st.buf[i][maxc + 1] = (int32_t)(int8_t)(seed >> 15) * (1 << s.noise_shift);
            st.buf[i][maxc + 2] = (int32_t)(int8_t)s7 * (1 << s.noise_shift);
            seed = (seed << 16) ^ s7 ^ (s7 << 5);
        }
        s.seed = seed;
        maxc += 2;
    }
    for (int m = 0; m < s.n_mat; ++m) {
        const int d = s.mat_out[m];
        const int32_t mask = (int32_t)(0u - (1u << s.quant[d]));
        for (int i = 0; i < n; ++i) {
            int64_t acc = 0;
            for (int c = 0; c <= maxc; ++c) acc += (int64_t)st.buf[i][c] * s.coeff[m][c];
            st.buf[i][d] = (int32_t)(((acc >> 14) & mask) + st.byp[i][m]);
        }
    }
    uint32_t check = s.check;
    for (int i = 0; i < n; ++i)
        for (int o = 0; o <= s.max_mat; ++o) {
            const int mc = s.assign[o];
            const int32_t v = (int32_t)((uint32_t)st.buf[i][mc] << s.out_shift[mc]);
            check ^= ((uint32_t)v & 0xFFFFFF) << mc;
            out[(int64_t)i * f.channels + o] = (int16_t)(v >> 8);
        }
    s.check = check;
}

// ---- one AU --------------------------------------------------------------------------------------------------------
// The AU at buf[off, limit): header, optional major sync, directory, the decoded substreams, then the output.
// *nsamp receives the samples it outputs; *eos whether it ends the stream.
SBT_HD int decode_au(const uint8_t* buf, int64_t off, int64_t limit, const Format& f, State& st, bool seg_start,
                     int16_t* out, int* nsamp, int* eos) {
    *nsamp = 0; *eos = 0;
    if (limit - off < 4) return kTruncated;
    const uint8_t* au = buf + off;
    const int64_t length = (int64_t)(((au[0] << 8) | au[1]) & 0xFFF) * 2;
    if (length < 4 || off + length > limit) return kBadLength;
    int64_t at = 4;
    bool sync = false;
    if (length >= 32 && (rb32(au + 4) >> 1) == (0xF8726FBAu >> 1)) {
        if (au[7] == 0xBB) return kMlp;
        const int ms = sync_size(au + 4);
        if (4 + ms > length) return kBadLength;
        if (checksum16(au + 4, ms - 2) != ((uint32_t)au[4 + ms - 2] << 8 | au[4 + ms - 1])) return kBadSyncCrc;
        for (int i = 0; i < 4; ++i)
            if (au[8 + i] != f.fmt[i]) return kFormatChange;
        if ((au[20] >> 4) != f.n_sub) return kFormatChange;
        at += ms;
        sync = true;
        for (int k = 0; k < kMaxSub; ++k) st.sub[k].restart_seen = 0;
    }
    if (seg_start && !sync) return kNoRestart;
    const int64_t dir = at;
    int64_t start[4], end[4];
    bool par[4];
    int64_t prev = 0;
    for (int k = 0; k < f.n_sub; ++k) {
        if (at + 2 > length) return kBadDirectory;
        const uint32_t w = (uint32_t)au[at] << 8 | au[at + 1];
        at += 2;
        if (w & 0x8000) { if (at + 2 > length) return kBadDirectory; at += 2; }
        if (!(((w >> 14) & 1) ^ (sync ? 1 : 0))) return kBadDirectory;
        par[k] = (w >> 13) & 1;
        end[k] = (int64_t)(w & 0xFFF) * 2;
        start[k] = prev;
        if (end[k] < prev) return kBadDirectory;
        prev = end[k];
    }
    const uint8_t p = xor_bytes(au, 4) ^ xor_bytes(au + dir, at - dir);
    if ((((p >> 4) ^ p) & 0xF) != 0xF) return kBadNibble;
    if (at + end[f.n_sub - 1] > length) return kBadDirectory;
    for (int k = 0; k <= f.out_sub; ++k) {
        const int rc = decode_substream(au + at + start[k], end[k] - start[k], par[k], f, k, st);
        if (rc != kOk) return rc;
    }
    output(f, st, out);
    Sub& top = st.sub[f.out_sub];
    *nsamp = top.blockpos;
    *eos = top.eos;
    if (top.eos) top.check = kNoCheck;
    return kOk;
}

// ---- segments ------------------------------------------------------------------------------------------------------
// One restart segment: AUs [first_au, first_au + n_au) from byte `offset`.  blocks[0..n_blocks) are the byte offsets
// where the container's blocks start (one block for a raw stream): an AU must end inside its block, and the next AU
// starts where it ends or, at a block end, at the next block.
struct Segment { int64_t offset, first_au, n_au, next_offset; };
struct SegStatus {
    int64_t au;             // failing AU (code != kOk)
    int32_t code, last_samples;   // last_samples: samples of the segment's last AU
    uint32_t check;         // the segment's lossless check (XOR of its output), kNoCheck after an end-of-stream
    uint32_t stored;        // check byte of the segment's first restart header (checks the previous segment)
    int32_t eos, pad;
};

SBT_HD int64_t block_end(const int64_t* blocks, int64_t n_blocks, int64_t nbytes, int64_t off) {
    int64_t lo = 0, hi = n_blocks;                // first block starting after off
    while (lo < hi) { const int64_t mid = (lo + hi) / 2; if (blocks[mid] <= off) lo = mid + 1; else hi = mid; }
    return lo < n_blocks ? blocks[lo] : nbytes;
}

SBT_HD SegStatus decode_segment(const uint8_t* buf, int64_t nbytes, const int64_t* blocks, int64_t n_blocks,
                                const Format& f, const Segment& g, bool first_segment, State& st, int16_t* seg_pcm) {
    SegStatus r;
    r.au = g.first_au; r.code = kOk; r.last_samples = 0; r.check = kNoCheck; r.stored = 0; r.eos = 0; r.pad = 0;
    for (int k = 0; k < kMaxSub; ++k) {
        Sub& s = st.sub[k];
        s.restart_seen = 0; s.restarted = 0; s.check = kNoCheck; s.eos = 0;
        for (int c = 0; c < kMaxCh; ++c) {
            Chan& ch = s.ch[c];
            for (int j = 0; j < 8; ++j) ch.fir_hist[j] = 0;
            for (int j = 0; j < 4; ++j) ch.iir_hist[j] = 0;
            ch.known = first_segment ? 8 : 0;
            ch.known_iir = first_segment ? 4 : 0;
        }
    }
    int64_t off = g.offset;
    for (int64_t a = 0; a < g.n_au; ++a) {
        r.au = g.first_au + a;
        if (r.eos) { r.code = kAfterEnd; return r; }
        const int64_t lim = block_end(blocks, n_blocks, nbytes, off);
        int ns = 0, eos = 0;
        const int rc = decode_au(buf, off, lim, f, st, a == 0, seg_pcm + a * f.spa * (int64_t)f.channels,
                                 &ns, &eos);
        if (rc != kOk) { r.code = rc; return r; }
        if (a == 0) r.stored = st.sub[f.out_sub].stored_check;
        if (ns != f.spa && !eos) { r.code = kShortAu; return r; }
        r.last_samples = ns;
        r.eos = eos;
        const int64_t length = (int64_t)(((buf[off] << 8) | buf[off + 1]) & 0xFFF) * 2;
        off += length;
    }
    if (off != g.next_offset) { r.code = kBadChain; return r; }
    r.check = st.sub[f.out_sub].check;
    return r;
}

// ---- the chain (host) ----------------------------------------------------------------------------------------------
// Walk the AU lengths from the start: every AU must fit its block, the first one and every AU holding a major-sync
// pattern must be a listed candidate (a major sync whose CRC passes and whose decoded substreams open with restart
// headers: `cand` sorted, `cand_ok` per candidate).  Each such AU starts a segment.  `where(off)` names the byte offset
// of the block holding buffer offset off in messages.
struct Candidate { int64_t offset; int32_t code; int32_t restart; };

template <class Where>
bool chain(const uint8_t* buf, int64_t nbytes, const int64_t* blocks, int64_t n_blocks, const std::vector<Candidate>& cand,
           Where where, std::vector<Segment>& segs, int64_t* n_au_out, char* msg, size_t msg_len) {
    segs.clear();
    int64_t off = n_blocks ? blocks[0] : 0, au = 0;
    size_t ci = 0;
    while (off < nbytes) {
        const int64_t lim = block_end(blocks, n_blocks, nbytes, off);
        if (lim - off < 4) {
            snprintf(msg, msg_len, "TrueHD access unit %lld at byte offset %lld: %s", (long long)au, (long long)where(off),
                     error_text(kTruncated));
            return false;
        }
        const int64_t length = (int64_t)(((buf[off] << 8) | buf[off + 1]) & 0xFFF) * 2;
        if (length < 4 || off + length > lim) {
            snprintf(msg, msg_len, "TrueHD access unit %lld at byte offset %lld: %s", (long long)au, (long long)where(off),
                     error_text(kBadLength));
            return false;
        }
        const bool pattern = length >= 32 && (rb32(buf + off + 4) >> 1) == (0xF8726FBAu >> 1);
        while (ci < cand.size() && cand[ci].offset < off) ++ci;
        const bool listed = ci < cand.size() && cand[ci].offset == off;
        if (pattern || au == 0) {
            int code = kOk;
            if (!pattern) code = kNoRestart;
            else if (!listed) code = buf[off + 7] == 0xBB ? kMlp : kBadSyncCrc;
            else if (cand[ci].code != kOk) code = cand[ci].code;
            else if (!cand[ci].restart) code = kNoRestart;
            if (code != kOk) {
                snprintf(msg, msg_len, "TrueHD access unit %lld at byte offset %lld: %s", (long long)au,
                         (long long)where(off), error_text(code));
                return false;
            }
            if (!segs.empty()) segs.back().next_offset = off;
            Segment g; g.offset = off; g.first_au = au; g.n_au = 0; g.next_offset = nbytes;
            segs.push_back(g);
        }
        ++segs.back().n_au;
        ++au;
        off += length;
    }
    if (!segs.empty()) segs.back().next_offset = off;
    *n_au_out = au;
    return true;
}

// Every segment decoded, and each segment's lossless check equals the byte the next segment's restart header carries;
// only the last AU of the stream may be short.  Returns the sample count, or -1 with a message.
template <class Where>
int64_t check_segments(const std::vector<Segment>& segs, const SegStatus* st, const Format& f, Where where_au, char* msg,
                       size_t msg_len) {
    const int64_t ns = (int64_t)segs.size();
    for (int64_t k = 0; k < ns; ++k) {
        if (st[k].code != kOk) {
            snprintf(msg, msg_len, "TrueHD access unit %lld at byte offset %lld: %s", (long long)st[k].au,
                     (long long)where_au(k, st[k].au), error_text(st[k].code));
            return -1;
        }
    }
    for (int64_t k = 0; k < ns; ++k) {
        if (k + 1 < ns) {
            if (st[k].eos) {
                snprintf(msg, msg_len, "TrueHD access unit %lld at byte offset %lld: %s", (long long)segs[k + 1].first_au,
                         (long long)where_au(k + 1, segs[k + 1].first_au), error_text(kAfterEnd));
                return -1;
            }
            if (st[k].check != kNoCheck && xor8(st[k].check) != st[k + 1].stored) {
                snprintf(msg, msg_len, "TrueHD access unit %lld at byte offset %lld: %s", (long long)segs[k + 1].first_au,
                         (long long)where_au(k + 1, segs[k + 1].first_au), error_text(kLossless));
                return -1;
            }
        }
    }
    if (!ns) return 0;
    const Segment& last = segs[ns - 1];
    return (last.first_au + last.n_au - 1) * f.spa + st[ns - 1].last_samples;
}

// The candidate at a byte offset: a major sync pattern whose CRC passes; whether every decoded substream's data opens
// with a restart header (the two flag bits set and the restart sync word)
SBT_HD Candidate candidate(const uint8_t* buf, int64_t nbytes, int64_t off, const Format& f) {
    Candidate c; c.offset = off; c.code = kBadSyncCrc; c.restart = 0;
    if (nbytes - off < 36) return c;
    const uint8_t* au = buf + off;
    const int64_t length = (int64_t)(((au[0] << 8) | au[1]) & 0xFFF) * 2;
    if ((rb32(au + 4) >> 1) != (0xF8726FBAu >> 1)) return c;
    const int ms = sync_size(au + 4);
    if (4 + ms > nbytes - off || checksum16(au + 4, ms - 2) != ((uint32_t)au[4 + ms - 2] << 8 | au[4 + ms - 1])) return c;
    c.code = au[7] == 0xBB ? kMlp : kOk;
    if (c.code != kOk) return c;
    for (int i = 0; i < 4; ++i)
        if (au[8 + i] != f.fmt[i]) c.code = kFormatChange;
    if ((au[20] >> 4) != f.n_sub) c.code = kFormatChange;
    int64_t at = 4 + ms, prev = 0;
    const int64_t data = at + 2 * f.n_sub;                     // extra words are counted below
    int64_t extra = 0;
    int64_t starts[4];
    int k = 0;
    for (; k < f.n_sub && at + 2 <= length && off + at + 2 <= nbytes; ++k) {
        const uint32_t w = (uint32_t)au[at] << 8 | au[at + 1];
        at += 2;
        if (w & 0x8000) { at += 2; extra += 2; }
        starts[k] = prev;
        prev = (int64_t)(w & 0xFFF) * 2;
    }
    c.restart = k == f.n_sub;
    for (k = 0; c.restart && k <= f.out_sub; ++k) {
        const int64_t p = off + data + extra + starts[k];
        if (p + 3 > nbytes) { c.restart = 0; break; }
        const uint32_t v = (uint32_t)buf[p] << 16 | (uint32_t)buf[p + 1] << 8 | buf[p + 2];
        // bits: 1 (parameters), 1 (restart header), then the 13-bit sync 0x18F5
        if ((v >> 22) != 3 || ((v >> 9) & 0x1FFF) != (0x31EA >> 1)) { c.restart = 0; break; }
    }
    return c;
}

}  // namespace sbthd

namespace sbthd {

// ---- the stream format from the first AU (host) --------------------------------------------------------------------
// FFmpeg's channel bit of each channel of the 13 arrangement groups, and the order restart headers count channels in
inline uint64_t layout_mask(int arrangement) {
    static const uint64_t groups[13] = {0x3ull, 0x4ull, 0x8ull, 0x600ull, 0x5000ull, 0xC0ull, 0x30ull, 0x100ull, 0x800ull,
                                        0x600000000ull, 0x180000000ull, 0x2000ull, 0x800000000ull};
    uint64_t m = 0;
    for (int i = 0; i < 13; ++i)
        if (arrangement >> i & 1) m |= groups[i];
    return m;
}
inline void channel_codes(uint64_t mask, int8_t* code_to_out) {
    static const int order[20] = {0, 1, 2, 3, 9, 10, 12, 14, 6, 7, 4, 5, 8, 11, 33, 34, 31, 32, 13, 35};
    for (int k = 0; k < kMaxCh; ++k) code_to_out[k] = -1;
    int k = 0;
    for (int i = 0; i < 20 && k < kMaxCh; ++i) {
        if (!(mask >> order[i] & 1)) continue;
        int native = 0;
        for (int b = 0; b < order[i]; ++b) native += (int)(mask >> b & 1);
        code_to_out[k++] = (int8_t)native;
    }
}
inline int popcount64(uint64_t m) { int n = 0; for (; m; m &= m - 1) ++n; return n; }

// Parse the major sync of the AU at buf[off]: false with a message when it is missing, damaged, MLP or a layout the
// decoder does not take
inline bool parse_format(const uint8_t* buf, int64_t nbytes, int64_t off, Format* f, char* msg, size_t msg_len) {
    memset(f, 0, sizeof(*f));
    const uint8_t* au = buf + off;
    if (nbytes - off < 36 || (rb32(au + 4) >> 1) != (0xF8726FBAu >> 1)) {
        snprintf(msg, msg_len, "TrueHD access unit 0 at byte offset %%lld: the stream does not start with a major sync");
        return false;
    }
    if (au[7] == 0xBB) { snprintf(msg, msg_len, "MLP (DVD-Audio) is not supported, only TrueHD"); return false; }
    const int ms = sync_size(au + 4);
    if (nbytes - off < 4 + ms || checksum16(au + 4, ms - 2) != ((uint32_t)au[4 + ms - 2] << 8 | au[4 + ms - 1])) {
        snprintf(msg, msg_len, "TrueHD access unit 0 at byte offset %%lld: %s", error_text(kBadSyncCrc));
        return false;
    }
    const uint8_t* s = au + 4;
    for (int i = 0; i < 4; ++i) f->fmt[i] = s[4 + i];
    const int code = s[4] >> 4;
    f->rate = rate_of(code);
    f->spa = 40 << (code & 7);
    f->n_sub = s[16] >> 4;
    const int arr1 = ((s[5] & 0xF) << 1) | (s[6] >> 7);                     // after 4 + 4 + 2 + 2 bits
    const int arr2 = ((s[6] & 0x1F) << 8) | s[7];                          // after 2 more bits
    if (!f->rate || f->spa > kMaxAu) { snprintf(msg, msg_len, "TrueHD sample rate code %d is not supported", code); return false; }
    if (f->n_sub < 1 || f->n_sub > 4) { snprintf(msg, msg_len, "TrueHD with %d substreams is not supported", f->n_sub); return false; }
    f->out_sub = std::min(f->n_sub - 1, 2);
    const uint64_t out_mask = layout_mask(arr2);
    f->channels = popcount64(out_mask);
    if (!arr2 || f->channels > kMaxCh) {
        snprintf(msg, msg_len, "TrueHD channel arrangement 0x%04x is not supported (1 to 8 channels)", arr2);
        return false;
    }
    for (int k = 0; k <= f->out_sub; ++k) {
        const uint64_t m = k == f->out_sub ? out_mask : k == 0 ? 0x3ull : layout_mask(arr1);
        channel_codes(m, f->code_to_out[k]);
    }
    return true;
}

}  // namespace sbthd
