// The conversion the ffmpeg command line runs for `-ac 1 -ar <rate> -acodec pcm_s16le` on S16 audio: libswresample's
// downmix to mono and its resampler with every option at its default, written once for the kernels of sb_swr.cu and for
// the CPU (tests/emu/emu_swr_driver.cpp compiles this header with g++).  Pinned against libswresample 6.1.100 on its
// x86-64 FMA3 path (tests/test_swr_cases.py holds it there bit for bit through tests/ref_swr.py).
//
// What libswresample does, as established by calling it:
//   - No resampling (equal rates): the integer S16P path.  The mono row of swr_build_matrix2 in Q15: a row of one or
//     two non-zero coefficients is quantised with error diffusion and mixed as (sum c*x + 16384) >> 15 (clipped when
//     the coefficients add up to more than 32768), a longer row is lrint(c * 32768) and its sum is truncated to 16
//     bits.  A mono input is passed through.
//   - Resampling: float.  Every channel is converted (x * 2^-15, exact) and resampled first, then remixed in float in
//     channel order (v = 0; v += y * c, each operation rounded), then lrintf(v * 32768) clipped to int16.
//   - The resampler: a Kaiser-windowed sinc (beta 9, cutoff 0.97, 32 taps at the input rate widened by the decimation
//     factor, even lengths) in 1024 phases, or in out/gcd phases when that ratio needs no more; an inexact ratio
//     interpolates linearly between neighbouring phases.  The FMA3 kernel accumulates taps i = j mod 8 in lane j
//     with fused multiply-adds over the bank row zero-padded to a multiple of 8, then sums
//     (l0+l4)+(l2+l6) + (l1+l5)+(l3+l7); the linear kernel interpolates the four half sums before the last two
//     additions.
//   - The edges: the signal the filter sees starts with its first (taps - 1) / 2 samples mirrored about sample 0, and
//     at the flush (min(left, taps) + 1) / 2 samples mirrored about the last sample are appended, `left` being the
//     input the filter had not yet stepped over.  Outputs run while the whole filter fits.  The result does not depend
//     on how the input is chunked, so the whole buffer is one pass here.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <vector>

#if defined(__CUDACC__)
#define SBS_HD __host__ __device__ __forceinline__
#else
#define SBS_HD inline
#endif

namespace sbswr {

constexpr int kMaxChannels = 8;
constexpr int kLanes = 8;                            // floats per AVX register
constexpr int kFilterSize = 32, kPhaseShift = 10;    // libswresample's filter_size and phase_shift defaults
constexpr double kCutoff = 0.97, kKaiserBeta = 9.0;

// FFmpeg's AV_CH_* bits this stage mixes; any other bit in a layout is refused
enum : uint64_t {
    FL = 0x1, FR = 0x2, FC = 0x4, LFE = 0x8, BL = 0x10, BR = 0x20, FLC = 0x40, FRC = 0x80, BC = 0x100, SL = 0x200,
    SR = 0x400, kKnown = 0x7ff
};

// ---- arithmetic that must not be contracted into FMAs ---------------------------------------------------------------
SBS_HD float fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
SBS_HD float fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
SBS_HD float fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}

// ---- the mono row of the remix matrix -------------------------------------------------------------------------------
struct Mix {
    int channels;
    int count;                       // non-zero coefficients, in channel order
    int index[kMaxChannels];         // their channels
    float flt[kMaxChannels];         // float coefficient of each channel (0 for a channel not in the row)
    int32_t q15[kMaxChannels];       // lrint(c * 32768): rows of three or more coefficients
    int32_t native[kMaxChannels];    // error-diffused Q15: rows of one or two coefficients
    int unity;                       // one coefficient of exactly 1.0: a copy
    int clip;                        // the native coefficients add up to more than 32768
};

// swr_build_matrix2's row for a front-centre output, defaults as ffmpeg passes them: centre and surround levels are
// the float options' -3 dB, the LFE is muted, and the row is scaled down to an absolute sum of 1 when it exceeds it.
// row[k] is channel k of `layout` (in mask order).  Returns false, with the reason in msg, for a layout libswresample
// refuses or this stage does not mix.
inline bool mono_row(uint64_t layout, double* row, char* msg, int msg_len) {
    const double sqrt1_2 = 0.70710678118654752440;
    const double clev = (double)(float)sqrt1_2, slev = (double)(float)sqrt1_2, lfe = 0.0;
    const int n = __builtin_popcountll(layout);
    auto pair_ok = [&](uint64_t m) { const uint64_t s = layout & m; return !s || (s & (s - 1)); };
    if (n < 1 || n > kMaxChannels || (layout & ~(uint64_t)kKnown) || !(layout & (FL | FR | FC)) ||
        !pair_ok(FL | FR) || !pair_ok(SL | SR) || !pair_ok(BL | BR) || !pair_ok(FLC | FRC)) {
        snprintf(msg, msg_len, "channel layout 0x%llx cannot be mixed to mono", (unsigned long long)layout);
        return false;
    }
    double m[11] = {0};                      // by bit
    if (layout & FC) m[2] = 1.0;
    const uint64_t un = layout & ~(uint64_t)FC;
    if (un & (FL | FR)) {
        m[0] += sqrt1_2; m[1] += sqrt1_2;
        if (layout & FC) m[2] = clev * sqrt(2.0);
    }
    if (un & BC) m[8] += slev * sqrt1_2;
    if (un & BL) { m[4] += slev * sqrt1_2; m[5] += slev * sqrt1_2; }
    if (un & SL) { m[9] += slev * sqrt1_2; m[10] += slev * sqrt1_2; }
    if (un & FLC) { m[6] += sqrt1_2; m[7] += sqrt1_2; }
    if (un & LFE) m[3] += lfe;
    double sum = 0;
    int k = 0;
    for (int b = 0; b < 11; ++b)
        if (layout & (1ull << b)) { row[k] = m[b]; sum += fabs(row[k]); ++k; }
    if (sum > 1.0)
        for (int i = 0; i < k; ++i) row[i] /= sum;
    return true;
}

inline bool make_mix(uint64_t layout, Mix* x, char* msg, int msg_len) {
    double row[kMaxChannels];
    if (!mono_row(layout, row, msg, msg_len)) return false;
    *x = Mix{};
    x->channels = __builtin_popcountll(layout);
    double rem = 0;
    int sum = 0;
    for (int j = 0; j < x->channels; ++j) {
        x->flt[j] = (float)row[j];
        x->q15[j] = (int32_t)lrint(row[j] * 32768);
        const double target = row[j] * 32768 + rem;
        x->native[j] = (int32_t)lrintf((float)target);
        rem += target - x->native[j];
        sum += x->native[j] < 0 ? -x->native[j] : x->native[j];
        if (row[j] != 0) x->index[x->count++] = j;
    }
    x->unity = x->count == 1 && row[x->index[0]] == 1.0;
    x->clip = sum > 32768;
    return true;
}

SBS_HD int16_t clip16(int v) { return (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }

// One frame of interleaved S16 through the integer S16P remix
SBS_HD int16_t mix_int(const int16_t* f, const Mix& x) {
    if (x.count == 1) {
        const int i = x.index[0];
        if (x.unity) return f[i];
        const int v = (x.native[i] * f[i] + 16384) >> 15;
        return x.clip ? clip16(v) : (int16_t)v;
    }
    if (x.count == 2) {
        const int i = x.index[0], j = x.index[1];
        const int v = (x.native[i] * f[i] + x.native[j] * f[j] + 16384) >> 15;
        return x.clip ? clip16(v) : (int16_t)v;
    }
    int v = 0;
    for (int k = 0; k < x.count; ++k) v += f[x.index[k]] * x.q15[x.index[k]];
    return (int16_t)((v + 16384) >> 15);
}

// The float remix of one output: y[c] is channel c resampled
SBS_HD float mix_float(const float* y, const Mix& x) {
    float v = 0.f;
    for (int k = 0; k < x.count; ++k) v = fadd(v, fmul(y[x.index[k]], x.flt[x.index[k]]));
    return v;
}

// float -> S16 as libswresample's output conversion does it
SBS_HD int16_t to_s16(float v) {
#if defined(__CUDA_ARCH__)
    const float s = __fmul_rn(v, 32768.f);
    return s >= 32767.f ? (int16_t)32767 : s <= -32768.f ? (int16_t)-32768 : (int16_t)__float2int_rn(s);
#else
    const float s = v * 32768.f;
    return s >= 32767.f ? (int16_t)32767 : s <= -32768.f ? (int16_t)-32768 : (int16_t)lrintf(s);
#endif
}

// ---- the resampler ----------------------------------------------------------------------------------------------------
struct Resampler {
    int filter_length;               // taps
    int filter_alloc;                // taps rounded up to 8: the row stride of the bank, zero-padded
    int phase_count;
    int linear;                      // inexact ratio: interpolate between phases
    int64_t src_incr, dst_incr;      // an output advances dst_incr / src_incr phases
    float inv_src_incr;              // 1.0f / src_incr, as the linear kernel computes it
    double factor;                   // cutoff relative to the input rate, at most 1
};

// Where output t reads: the first of its filter_length samples, its phase, and (linear) the fraction toward the next
SBS_HD void position(const Resampler& r, int64_t t, int64_t* sample, int* phase, int64_t* frac) {
    const int64_t p = t * r.dst_incr;
    const int64_t index = p / r.src_incr;
    *frac = p - index * r.src_incr;
    *sample = index / r.phase_count;
    *phase = (int)(index - *sample * r.phase_count);
}

inline int64_t gcd64(int64_t a, int64_t b) { while (b) { const int64_t t = a % b; a = b; b = t; } return a; }

inline bool make_resampler(int in_rate, int out_rate, Resampler* r, char* msg, int msg_len) {
    if (in_rate < 1 || out_rate < 1) {
        snprintf(msg, msg_len, "bad sample rates %d -> %d", in_rate, out_rate);
        return false;
    }
    *r = Resampler{};
    r->factor = out_rate * kCutoff / in_rate;
    if (r->factor > 1.0) r->factor = 1.0;
    int pc = 1 << kPhaseShift;
    int len = (int)ceil(kFilterSize / r->factor);
    if (len < 1) len = 1;
    if (len > 1) len = (len + 1) & ~1;
    const int64_t g = gcd64(out_rate, in_rate);
    if (out_rate / g <= pc) pc = (int)(out_rate / g);
    r->filter_length = len;
    r->filter_alloc = (len + 7) & ~7;
    r->phase_count = pc;
    const int64_t den = (int64_t)in_rate * pc, g2 = gcd64(out_rate, den);
    int64_t src = out_rate / g2, dst = den / g2;
    if (src > INT32_MAX / 2 || dst > INT32_MAX / 2 || len > 4096) {
        snprintf(msg, msg_len, "sample rates %d -> %d are not supported", in_rate, out_rate);
        return false;
    }
    while (dst < (1 << 20) && src < (1 << 20)) { dst *= 2; src *= 2; }
    r->src_incr = src;
    r->dst_incr = dst;
    r->linear = (dst % src) != 0;
    r->inv_src_incr = 1.0f / (float)src;
    return true;
}

// The zeroth-order modified Bessel function as libswresample's Kaiser window evaluates it (FFmpeg's av_bessel_i0:
// Blair and Edwards' minimax rational approximations, Horner from the highest coefficient)
inline double eval_poly(const double* c, int n, double x) {
    double s = c[n - 1];
    for (int i = n - 2; i >= 0; --i) { s *= x; s += c[i]; }
    return s;
}
inline double bessel_i0(double x) {
    static const double p1[] = {
        -2.2335582639474375249e+15, -5.5050369673018427753e+14, -3.2940087627407749166e+13,
        -8.4925101247114157499e+11, -1.1912746104985237192e+10, -1.0313066708737980747e+08,
        -5.9545626019847898221e+05, -2.4125195876041896775e+03, -7.0935347449210549190e+00,
        -1.5453977791786851041e-02, -2.5172644670688975051e-05, -3.0517226450451067446e-08,
        -2.6843448573468483278e-11, -1.5982226675653184646e-14, -5.2487866627945699800e-18,
    };
    static const double q1[] = {
        -2.2335582639474375245e+15, 7.8858692566751002988e+12, -1.2207067397808979846e+10,
        1.0377081058062166144e+07, -4.8527560179962773045e+03, 1.0,
    };
    static const double p2[] = {
        -2.2210262233306573296e-04, 1.3067392038106924055e-02, -4.4700805721174453923e-01,
        5.5674518371240761397e+00, -2.3517945679239481621e+01, 3.1611322818701131207e+01,
        -9.6090021968656180000e+00,
    };
    static const double q2[] = {
        -5.5194330231005480228e-04, 3.2547697594819615062e-02, -1.1151759188741312645e+00,
        1.3982595353892851542e+01, -6.0228002066743340583e+01, 8.5539563258012929600e+01,
        -3.1446690275135491500e+01, 1.0,
    };
    if (x == 0) return 1.0;
    x = fabs(x);
    if (x <= 15) {
        const double y = x * x;
        return eval_poly(p1, 15, y) / eval_poly(q1, 6, y);
    }
    const double y = 1 / x - 1.0 / 15;
    const double r = eval_poly(p2, 7, y) / eval_poly(q2, 8, y);
    return exp(x) / sqrt(x) * r;
}

// The float bank: (phase_count + 1) rows of filter_alloc floats.  Row phase_count is row 0 one sample later, for the
// linear interpolation of the last phase.
inline void float_bank(const Resampler& r, std::vector<float>& bank) {
    const int L = r.filter_length, alloc = r.filter_alloc, pc = r.phase_count;
    const double factor = r.factor;
    bank.assign((size_t)alloc * (pc + 1), 0.f);
    float* f = bank.data();
    const int ph_nb = pc % 2 ? pc : pc / 2 + 1;
    const int center = (L - 1) / 2;
    std::vector<double> tab(L + 1), sin_lut(ph_nb);
    double norm = 0;
    if (factor == 1.0)
        for (int ph = 0; ph < ph_nb; ++ph) sin_lut[ph] = sin(M_PI * ph / pc) * (center & 1 ? 1 : -1);
    for (int ph = 0; ph < ph_nb; ++ph) {
        double s = sin_lut[ph];
        for (int i = 0; i < L; ++i) {
            const double x = M_PI * ((double)(i - center) - (double)ph / pc) * factor;
            double y;
            if (x == 0) y = 1.0;
            else if (factor == 1.0) y = s / x;
            else y = sin(x) / x;
            const double w = 2.0 * x / (factor * L * M_PI);
            const double a = 1 - w * w;
            y *= bessel_i0(kKaiserBeta * sqrt(a > 0 ? a : 0));
            tab[i] = y;
            s = -s;
            if (!ph) norm += y;
        }
        for (int i = 0; i < L; ++i) f[ph * alloc + i] = (float)(tab[i] * 1 / norm);
        if (pc % 2) continue;
        for (int i = 0; i < L; ++i) f[(pc - ph) * alloc + L - 1 - i] = f[ph * alloc + i];
    }
    f[(size_t)alloc * pc] = f[alloc - 1];
    for (int i = 1; i < alloc; ++i) f[(size_t)alloc * pc + i] = f[i - 1];
}

// The dot product of one bank row with the window w[0 .. filter_alloc) in the FMA3 kernel's lanes and order
SBS_HD void lanes(const float* row, const float* w, int alloc, float* q) {
    float a[kLanes];
    for (int j = 0; j < kLanes; ++j) a[j] = 0.f;
    for (int i = 0; i < alloc; i += kLanes)
        for (int j = 0; j < kLanes; ++j) a[j] = fmaf(row[i + j], w[i + j], a[j]);
    for (int j = 0; j < 4; ++j) q[j] = fadd(a[j], a[j + 4]);
}
SBS_HD float hsum4(const float* q) { return fadd(fadd(q[0], q[2]), fadd(q[1], q[3])); }

// One output of one channel: w is the window starting at the output's first sample
SBS_HD float resample_one(const Resampler& r, const float* bank, const float* w, int phase, int64_t frac) {
    const float* row = bank + (int64_t)phase * r.filter_alloc;
    float q[4];
    lanes(row, w, r.filter_alloc, q);
    if (r.linear) {
        float q2[4];
        lanes(row + r.filter_alloc, w, r.filter_alloc, q2);
        const float t = fmul((float)frac, r.inv_src_incr);
        for (int j = 0; j < 4; ++j) q[j] = fmaf(fsub(q2[j], q[j]), t, q[j]);
    }
    return hsum4(q);
}

// ---- the whole conversion -------------------------------------------------------------------------------------------
struct Plan {
    int channels, in_rate, out_rate;
    int64_t in_frames, out_frames;
    int resample;                    // the rates differ
    int64_t lead;                    // (taps - 1) / 2: samples mirrored before sample 0
    int64_t tail;                    // samples mirrored after the last one
    Mix mix;
    Resampler rs;
};

// Input frame that sample j of the filter's signal is (-1: past its end, read as 0)
SBS_HD int64_t source_frame(const Plan& p, int64_t j) {
    int64_t m = j - p.lead;
    if (m < 0) m = -m;
    if (m < p.in_frames) return m;
    m -= p.in_frames;
    return m < p.tail ? p.in_frames - 1 - m : -1;
}

// Outputs t >= 0 whose first sample is at most `limit`
inline int64_t outputs_upto(const Resampler& r, int64_t limit) {
    if (limit < 0) return 0;
    const unsigned __int128 num = (unsigned __int128)(limit + 1) * r.phase_count * r.src_incr;
    return (int64_t)((num + r.dst_incr - 1) / r.dst_incr);
}

inline bool make_plan(uint64_t layout, int channels, int in_rate, int out_rate, int64_t frames, Plan* p, char* msg,
                      int msg_len) {
    *p = Plan{};
    if (channels != __builtin_popcountll(layout)) {
        snprintf(msg, msg_len, "channel layout 0x%llx does not have %d channels", (unsigned long long)layout, channels);
        return false;
    }
    if (!make_mix(layout, &p->mix, msg, msg_len)) return false;
    if (frames < 0 || out_rate < 1 || in_rate < 1) {
        snprintf(msg, msg_len, "bad geometry");
        return false;
    }
    p->channels = channels;
    p->in_rate = in_rate;
    p->out_rate = out_rate;
    p->in_frames = frames;
    p->resample = in_rate != out_rate;
    if (!p->resample) {
        p->out_frames = frames;
        return true;
    }
    Resampler& r = p->rs;
    if (!make_resampler(in_rate, out_rate, &r, msg, msg_len)) return false;
    const int64_t L = r.filter_length;
    p->lead = (L - 1) / 2;
    if (frames <= L) {
        // nothing comes out before the flush; after it the filter needs L + 1 samples to start
        p->tail = (frames + 1) / 2;
        if (frames + p->tail < L + 1) { p->out_frames = 0; return true; }
    } else {
        const int64_t v1 = p->lead + frames;
        const int64_t m1 = outputs_upto(r, v1 - L);
        int64_t s; int ph; int64_t fr;
        position(r, m1, &s, &ph, &fr);
        const int64_t left = v1 - s;
        p->tail = ((left < L ? left : L) + 1) / 2;
    }
    p->out_frames = outputs_upto(r, p->lead + frames + p->tail - L);
    return true;
}

// The resample kernel's launch shape: the widest tile of 256, 128, 64 or 32 outputs whose input window fits in
// max_bytes of shared memory, and that window's width in floats.  A tile of `tile` outputs starting at any t0 reads
// samples s(t0) .. s(t0 + tile - 1) + filter_alloc - 1.  With X = (tile - 1) * dst_incr / src_incr (integer division)
// the phase index p * phase_count + r (r < phase_count) of t0 advances by at most X + 1 over the tile, so
// s(t0 + tile - 1) - s(t0) <= (r + X + 1) / phase_count <= X / phase_count + 1 = span - 1: the window has one float to
// spare.  Returns false when even 32 outputs need a wider window (no rate pair make_resampler accepts does:
// tests/test_swr_cases.py sweeps them).
inline bool tile_shape(const Resampler& r, int max_bytes, int* tile, int* width) {
    for (int t = 256; t >= 32; t /= 2) {
        const int64_t span = ((int64_t)(t - 1) * r.dst_incr / r.src_incr) / r.phase_count + 2;
        if ((span + r.filter_alloc) * (int64_t)sizeof(float) <= max_bytes) {
            *tile = t;
            *width = (int)(span + r.filter_alloc);
            return true;
        }
    }
    return false;
}

}  // namespace sbswr
