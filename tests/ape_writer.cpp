// The encoder side of a Monkey's Audio 3.99 frame, for tests/ape_cases.py (compiled with g++ by that module).  Each
// stage is the mirror of the decoder stage it feeds, written from the format and not from the library's sb_ape.cuh:
//   the inter-channel decorrelation (Y = right - left, X = left + Y / 2),
//   the 3950 predictor run forward (the residual is the target minus the prediction),
//   the NN filter cascade run forward, last filter first (each filter's input is its output minus its dot product),
//   the 3990 range coder (Schindler's carry-propagating coder as Monkey's Audio writes it) with the adaptive sum,
// and the frame's CRC-32 over the little-endian output bytes.
#include <stdint.h>
#include <string.h>
#include <vector>

namespace {

const uint16_t kCounts[22] = {0,     19578, 36160, 48417, 56323, 60899, 63265, 64435, 64971, 65232, 65351,
                              65416, 65447, 65466, 65476, 65482, 65485, 65488, 65490, 65491, 65492, 65493};
const int kOrders[5][3] = {{0, 0, 0}, {16, 0, 0}, {64, 0, 0}, {32, 256, 0}, {16, 256, 1280}};
const int kFracbits[5][3] = {{0, 0, 0}, {11, 0, 0}, {11, 0, 0}, {10, 13, 0}, {11, 13, 15}};

int sgn(int64_t x) { return (x < 0) - (x > 0); }      // APESIGN: the sign, negated

struct Stats {
    int64_t escapes = 0, max_overflow = 0, max_pivot = 0, saturated = 0, big_pivots = 0, min_pivot = 1 << 30;
};

struct Coder {
    std::vector<uint8_t> out;
    uint32_t low = 0, range = 1u << 31, buffer = 0, help = 0;
    void normalize() {
        while (range <= (1u << 23)) {
            if (low < (0xFFu << 23)) {
                out.push_back((uint8_t)buffer);
                for (; help; --help) out.push_back(0xFF);
                buffer = low >> 23;
            } else if (low & (1u << 31)) {
                out.push_back((uint8_t)(buffer + 1));
                for (; help; --help) out.push_back(0);
                buffer = low >> 23;
            } else {
                ++help;
            }
            low = (low << 8) & ((1u << 31) - 1);
            range <<= 8;
        }
    }
    void shift(uint32_t width, uint32_t start, int bits) {     // decoded by range_decode_culshift(bits)
        normalize();
        const uint32_t t = range >> bits;
        range = t * width;
        low += t * start;
    }
    void freq(uint32_t value, uint32_t total) {               // decoded by range_decode_culfreq(total)
        normalize();
        const uint32_t t = range / total;
        range = t;
        low += t * value;
    }
    void finish() {
        normalize();
        const uint32_t t = (low >> 23) + 1;
        if (t > 0xFF) {
            out.push_back((uint8_t)(buffer + 1));
            for (; help; --help) out.push_back(0);
        } else {
            out.push_back((uint8_t)buffer);
            for (; help; --help) out.push_back(0xFF);
        }
        out.push_back((uint8_t)t);
        out.push_back(0);
        out.push_back(0);
        out.push_back(0);
    }
};

// ksum: the channel's adaptive sum, which sets the pivot (the Rice parameter k that FFmpeg keeps beside it changes no
// output in version 3990)
void encode_value(Coder& c, uint32_t& ksum, int32_t v, int force_escape, Stats& st) {
    const uint32_t base = v > 0 ? 2u * (uint32_t)v - 1u : 0u - 2u * (uint32_t)v;
    uint32_t pivot = ksum >> 5;
    if (pivot == 0) pivot = 1;
    if (pivot < (uint32_t)st.min_pivot) st.min_pivot = pivot;
    const uint32_t overflow = base / pivot, rest = base % pivot;
    if (overflow > (uint32_t)st.max_overflow) st.max_overflow = overflow;
    if (pivot > (uint32_t)st.max_pivot) st.max_pivot = pivot;
    if (overflow >= 63 || force_escape) {
        ++st.escapes;
        c.shift(1, 65535, 16);
        c.shift(1, overflow >> 16, 16);
        c.shift(1, overflow & 0xFFFF, 16);
    } else if (overflow <= 20) {
        c.shift(kCounts[overflow + 1] - kCounts[overflow], kCounts[overflow], 16);
    } else {
        c.shift(1, overflow + 65472, 16);
    }
    if (pivot < 0x10000) {
        c.freq(rest, pivot);
    } else {
        ++st.big_pivots;
        int bbits = 0;
        uint32_t hi = pivot;
        while (hi & ~0xFFFFu) {
            hi >>= 1;
            ++bbits;
        }
        c.freq(rest >> bbits, hi + 1);
        c.freq(rest & ((1u << bbits) - 1), 1u << bbits);
    }
    ksum += (base + 1) / 2 - ((ksum + 16) >> 5);
}

// One NN filter, run forward: given the filter's output, its input.
struct NN {
    int order, frac;
    std::vector<int16_t> w, hist, adapt;     // weights; the saturated outputs and adapt values, oldest first
    int32_t avg = 0;
    NN(int o, int f) : order(o), frac(f), w(o, 0), hist(o, 0), adapt(o, 0) {}
    int32_t input_for(int32_t out, Stats& st) {
        uint32_t dot = 0;
        for (int i = 0; i < order; ++i) dot += (uint32_t)((int32_t)w[i] * hist[i]);
        const int32_t pred = (int32_t)(((int64_t)(int32_t)dot + (1ll << (frac - 1))) >> frac);
        const int32_t in = (int32_t)((uint32_t)out - (uint32_t)pred);
        const int s = sgn(in);
        for (int i = 0; i < order; ++i) w[i] = (int16_t)(w[i] + s * adapt[i]);
        // age the adapt values: the one 1, 2 and 8 samples back halve (FFmpeg's [-1], [-2], [-8] after the write)
        const int32_t sat = out > 32767 ? 32767 : out < -32768 ? -32768 : out;
        if (sat != out) ++st.saturated;
        const uint32_t a = out < 0 ? 0u - (uint32_t)out : (uint32_t)out;
        int16_t na = 0;
        if (a) na = (int16_t)(sgn(out) * (8 << ((a > (int64_t)avg * 3) + (a > (uint32_t)(avg + avg / 3)))));
        avg += (int32_t)(a - (uint32_t)avg) / 16;
        memmove(&hist[0], &hist[1], sizeof(int16_t) * (order - 1));
        memmove(&adapt[0], &adapt[1], sizeof(int16_t) * (order - 1));
        hist[order - 1] = (int16_t)sat;
        adapt[order - 1] = na;
        if (order >= 2) adapt[order - 2] >>= 1;
        if (order >= 3) adapt[order - 3] >>= 1;
        if (order >= 9) adapt[order - 9] >>= 1;
        return in;
    }
};

// The 3950 predictor's state, in FFmpeg's 64-bit layout, run forward: for channel f (0 = Y, 1 = X) and the sample it
// must output, the value the NN filters must deliver.
struct Predictor {
    int64_t dA[2][4] = {}, aA[2][4] = {}, dB[2][5] = {}, aB[2][5] = {};
    int64_t cA[2][4], cB[2][5] = {};
    int64_t lastA[2] = {}, filterA[2] = {}, filterB[2] = {};
    Predictor() {
        const int64_t init[4] = {360, 317, -109, 98};
        for (int f = 0; f < 2; ++f)
            for (int i = 0; i < 4; ++i) cA[f][i] = init[i];
    }
    int32_t stereo(int f, int32_t target) {
        // history slots: d[0] newest
        for (int i = 3; i > 0; --i) { dA[f][i] = dA[f][i - 1]; aA[f][i] = aA[f][i - 1]; }
        const int64_t prevA = dA[f][1];
        dA[f][0] = lastA[f];
        aA[f][0] = sgn(dA[f][0]);
        dA[f][1] = dA[f][0] - prevA;
        aA[f][1] = sgn(dA[f][1]);
        int64_t pa = 0;
        for (int i = 0; i < 4; ++i) pa += dA[f][i] * cA[f][i];
        for (int i = 4; i > 0; --i) { dB[f][i] = dB[f][i - 1]; aB[f][i] = aB[f][i - 1]; }
        const int64_t prevB = dB[f][1];
        dB[f][0] = filterA[f ^ 1] - ((filterB[f] * 31) >> 5);
        aB[f][0] = sgn(dB[f][0]);
        dB[f][1] = dB[f][0] - prevB;
        aB[f][1] = sgn(dB[f][1]);
        filterB[f] = filterA[f ^ 1];
        int64_t pb = 0;
        for (int i = 0; i < 5; ++i) pb += dB[f][i] * cB[f][i];
        const int32_t p = (int32_t)((int64_t)(int32_t)pa + ((int64_t)(int32_t)pb >> 1));
        const int32_t want_last = (int32_t)((int64_t)target - ((filterA[f] * 31) >> 5));
        const int32_t in = (int32_t)((uint32_t)want_last - (uint32_t)(p >> 10));
        lastA[f] = (int32_t)((uint32_t)in + (uint32_t)(p >> 10));
        filterA[f] = lastA[f] + ((filterA[f] * 31) >> 5);
        const int s = sgn(in);
        for (int i = 0; i < 4; ++i) cA[f][i] += aA[f][i] * s;
        for (int i = 0; i < 5; ++i) cB[f][i] += aB[f][i] * s;
        return in;
    }
    int32_t mono(int32_t target) {
        for (int i = 3; i > 0; --i) { dA[0][i] = dA[0][i - 1]; aA[0][i] = aA[0][i - 1]; }
        const int64_t prevA = dA[0][1];
        dA[0][0] = lastA[0];
        dA[0][1] = dA[0][0] - prevA;
        int64_t pa = 0;
        for (int i = 0; i < 4; ++i) pa += dA[0][i] * cA[0][i];
        const int32_t p = (int32_t)pa;
        const int32_t want_last = (int32_t)((int64_t)target - ((filterA[0] * 31) >> 5));
        const int32_t in = (int32_t)((uint32_t)want_last - (uint32_t)(p >> 10));
        lastA[0] = want_last;
        aA[0][0] = sgn(dA[0][0]);
        aA[0][1] = sgn(dA[0][1]);
        const int s = sgn(in);
        for (int i = 0; i < 4; ++i) cA[0][i] += aA[0][i] * s;
        filterA[0] = lastA[0] + ((filterA[0] * 31) >> 5);
        return in;
    }
};

uint32_t crc_update(uint32_t c, const uint8_t* p, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        c ^= p[i];
        for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
    }
    return c;
}

}  // namespace

extern "C" {

// Encode one frame of `blocks` samples.  pcm: interleaved int32 (channels of them per block), the samples the decoder
// must output.  mode: 0 coded (mono or stereo as the stream), 1 pseudo-stereo (both channels equal, coded once),
// 2 silence (all zero).  flags_word: 1 to write the flags word even when the flags are 0.  escape_every: when > 0,
// every escape_every-th value takes the overflow escape whatever its size.  Writes the frame's bytes (CRC, flags,
// range coder) to out and returns their count, or -1 when cap is too small.  stats: escapes, largest overflow, largest
// pivot, saturated NN outputs, values coded with a pivot of 2^16 or more, the smallest pivot.
int64_t ape_encode_frame(const int32_t* pcm, int64_t blocks, int channels, int bits, int level, int mode, int flags_word,
                         int escape_every, uint8_t* out, int64_t cap, int64_t* stats) {
    Stats st;
    uint32_t crc = 0xFFFFFFFFu;
    for (int64_t i = 0; i < blocks; ++i)
        for (int ch = 0; ch < channels; ++ch) {
            const uint32_t v = (uint32_t)pcm[i * channels + ch];
            const uint8_t b[3] = {(uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16)};
            crc = crc_update(crc, b, bits / 8);
        }
    uint32_t flags = 0;
    if (mode == 2) flags = channels == 2 ? 3 : 1;
    else if (mode == 1) flags = 4;
    Coder c;
    const int fset = level / 1000 - 1;
    if (mode != 2) {
        const int coded = (channels == 2 && mode == 0) ? 2 : 1;
        std::vector<int32_t> res((size_t)(blocks * coded));
        Predictor p;
        std::vector<NN> filters[2];
        for (int ch = 0; ch < coded; ++ch)
            for (int l = 0; l < 3 && kOrders[fset][l]; ++l) filters[ch].emplace_back(kOrders[fset][l], kFracbits[fset][l]);
        for (int64_t i = 0; i < blocks; ++i) {
            int32_t d[2];
            if (coded == 2) {
                const int32_t left = pcm[i * 2], right = pcm[i * 2 + 1];
                const int32_t y = (int32_t)((uint32_t)right - (uint32_t)left);
                const int32_t x = (int32_t)((uint32_t)left + (uint32_t)(y / 2));
                d[0] = p.stereo(0, y);
                d[1] = p.stereo(1, x);
            } else {
                d[0] = p.mono(pcm[i * channels]);
            }
            for (int ch = 0; ch < coded; ++ch) {
                int32_t v = d[ch];
                for (int l = (int)filters[ch].size() - 1; l >= 0; --l) v = filters[ch][(size_t)l].input_for(v, st);
                res[(size_t)(i * coded + ch)] = v;
            }
        }
        uint32_t ksum[2] = {16u << 10, 16u << 10};
        int64_t n = 0;
        for (int64_t i = 0; i < blocks; ++i)
            for (int ch = 0; ch < coded; ++ch, ++n)
                encode_value(c, ksum[ch], res[(size_t)(i * coded + ch)], escape_every > 0 && n % escape_every == 0, st);
    }
    c.finish();
    std::vector<uint8_t> frame;
    const uint32_t word = ((~crc) >> 1) | ((flags || flags_word) ? 0x80000000u : 0u);
    for (int s = 24; s >= 0; s -= 8) frame.push_back((uint8_t)(word >> s));
    if (flags || flags_word)
        for (int s = 24; s >= 0; s -= 8) frame.push_back((uint8_t)(flags >> s));
    frame.insert(frame.end(), c.out.begin(), c.out.end());
    if ((int64_t)frame.size() > cap) return -1;
    memcpy(out, frame.data(), frame.size());
    stats[0] = st.escapes; stats[1] = st.max_overflow; stats[2] = st.max_pivot; stats[3] = st.saturated;
    stats[4] = st.big_pivots; stats[5] = st.min_pivot;
    return (int64_t)frame.size();
}

}  // extern "C"
