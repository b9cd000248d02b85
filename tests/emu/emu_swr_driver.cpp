// CPU build of the mono downmix and resampler: sushi_b200/csrc/sb_swr.cuh compiled with g++
// (tests/test_swr_cases.py).  The plan, the matrix, the bank and the launch shape are the functions sb_pcm_swr calls.
// emu_swr_convert is one loop over the outputs, each reading the whole filter signal instead of a staged window;
// emu_swr_convert_tiled walks the tiles and windows of k_swr_resample, and emu_swr_tiles measures those windows.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "sb_swr.cuh"

extern "C" {

// geometry[0..5]: output frames, taps, bank row stride, phases, linear, samples mirrored at the end
int emu_swr_plan(uint64_t layout, int channels, int in_rate, int out_rate, int64_t frames, int64_t* geometry, char* msg,
                 int msg_len) {
    sbswr::Plan p;
    if (!sbswr::make_plan(layout, channels, in_rate, out_rate, frames, &p, msg, msg_len)) return -1;
    geometry[0] = p.out_frames;
    geometry[1] = p.rs.filter_length;
    geometry[2] = p.rs.filter_alloc;
    geometry[3] = p.rs.phase_count;
    geometry[4] = p.rs.linear;
    geometry[5] = p.tail;
    return 0;
}

// pcm: frames x channels interleaved S16 -> out: the mono S16 output (emu_swr_plan's frame count).  mix_first remixes
// before resampling instead of after (libswresample does not; kept to show that the order matters).
int emu_swr_convert(const int16_t* pcm, int64_t frames, int channels, uint64_t layout, int in_rate, int out_rate,
                    int mix_first, int16_t* out, char* msg, int msg_len) {
    sbswr::Plan p;
    if (!sbswr::make_plan(layout, channels, in_rate, out_rate, frames, &p, msg, msg_len)) return -1;
    if (!p.resample) {
        for (int64_t i = 0; i < frames; ++i) out[i] = sbswr::mix_int(pcm + i * channels, p.mix);
        return 0;
    }
    const sbswr::Resampler& r = p.rs;
    std::vector<float> bank;
    sbswr::float_bank(r, bank);
    const int64_t n = p.lead + frames + p.tail + r.filter_alloc;
    const int planes = mix_first ? 1 : channels;
    std::vector<std::vector<float>> sig(planes, std::vector<float>((size_t)n, 0.f));
    for (int64_t j = 0; j < n; ++j) {
        const int64_t f = sbswr::source_frame(p, j);
        if (f < 0) continue;
        float x[sbswr::kMaxChannels];
        for (int c = 0; c < channels; ++c) x[c] = pcm[f * channels + c] * (1.0f / 32768);
        if (mix_first) sig[0][(size_t)j] = sbswr::mix_float(x, p.mix);
        else for (int c = 0; c < channels; ++c) sig[c][(size_t)j] = x[c];
    }
    for (int64_t t = 0; t < p.out_frames; ++t) {
        int64_t s, frac;
        int phase;
        sbswr::position(r, t, &s, &phase, &frac);
        float y[sbswr::kMaxChannels];
        for (int c = 0; c < planes; ++c) y[c] = sbswr::resample_one(r, bank.data(), sig[c].data() + s, phase, frac);
        out[t] = sbswr::to_s16(mix_first ? y[0] : sbswr::mix_float(y, p.mix));
    }
    return 0;
}

// The resample kernel's launch shape for a rate pair and how much of its window the outputs use.  tiles[0..4]: the
// tile, the window width in floats (sbswr::tile_shape with max_bytes of shared memory), the largest
// s(t) - s(t0) + filter_alloc over every output t of every tile t0 = tile * (t / tile), the outputs walked, and the
// period of the position pattern in outputs (after it, s advances by a whole number and phase and fraction repeat).
// Tiles start at multiples of `tile`, so the windows repeat only after lcm(period, tile) outputs: the walk covers
// exactly that many, every tile start against every phase of the pattern.  Returns -1 for a pair make_resampler
// refuses, -2 for one no tile fits, -3 when lcm(period, tile) exceeds `cap` (the message says which).
int emu_swr_tiles(int in_rate, int out_rate, int max_bytes, int64_t cap, int64_t* tiles, char* msg, int msg_len) {
    sbswr::Resampler r;
    if (!sbswr::make_resampler(in_rate, out_rate, &r, msg, msg_len)) return -1;
    int tile = 0, width = 0;
    if (!sbswr::tile_shape(r, max_bytes, &tile, &width)) {
        snprintf(msg, msg_len, "sample rates %d -> %d need too wide a filter window", in_rate, out_rate);
        return -2;
    }
    const int64_t den = r.src_incr * r.phase_count;
    const int64_t period = den / sbswr::gcd64(r.dst_incr, den);
    const int64_t n = period / sbswr::gcd64(period, tile) * tile;
    if (n > cap) {
        snprintf(msg, msg_len, "sample rates %d -> %d: %lld outputs to walk, more than %lld", in_rate, out_rate,
                 (long long)n, (long long)cap);
        return -3;
    }
    int64_t need = 0, s0 = 0, s, frac;
    int phase;
    for (int64_t t = 0; t < n; ++t) {
        sbswr::position(r, t, &s, &phase, &frac);
        if (t % tile == 0) s0 = s;
        if (s - s0 + r.filter_alloc > need) need = s - s0 + r.filter_alloc;
    }
    tiles[0] = tile;
    tiles[1] = width;
    tiles[2] = need;
    tiles[3] = n;
    tiles[4] = period;
    return 0;
}

// emu_swr_convert as k_swr_resample computes it, in its order: per tile of outputs and per channel of the mono row,
// the tile's window of s(last) - s(t0) + filter_alloc floats is staged with sbswr::source_frame into a buffer of the
// launch's `width` floats (the rest NaN), each output is filtered from win + (s - s0), and the remix accumulates across
// the channels.  Staging past `width` or reading past what was staged is returned as -2 with the tile, channel and
// index.  Equal rates take the integer path, as in emu_swr_convert.
int emu_swr_convert_tiled(const int16_t* pcm, int64_t frames, int channels, uint64_t layout, int in_rate,
                          int out_rate, int max_bytes, int16_t* out, char* msg, int msg_len) {
    sbswr::Plan p;
    if (!sbswr::make_plan(layout, channels, in_rate, out_rate, frames, &p, msg, msg_len)) return -1;
    if (!p.resample) {
        for (int64_t i = 0; i < frames; ++i) out[i] = sbswr::mix_int(pcm + i * channels, p.mix);
        return 0;
    }
    const sbswr::Resampler& r = p.rs;
    int tile = 0, width = 0;
    if (!sbswr::tile_shape(r, max_bytes, &tile, &width)) {
        snprintf(msg, msg_len, "sample rates %d -> %d need too wide a filter window", in_rate, out_rate);
        return -1;
    }
    std::vector<float> bank;
    sbswr::float_bank(r, bank);
    std::vector<float> win((size_t)width);
    std::vector<float> v((size_t)tile);
    for (int64_t t0 = 0; t0 < p.out_frames; t0 += tile) {
        const int64_t last = (t0 + tile < p.out_frames ? t0 + tile : p.out_frames) - 1;
        int64_t s0, s1, s, frac;
        int phase;
        sbswr::position(r, t0, &s0, &phase, &frac);
        sbswr::position(r, last, &s1, &phase, &frac);
        const int64_t staged = s1 - s0 + r.filter_alloc;
        for (int64_t t = t0; t <= last; ++t) v[(size_t)(t - t0)] = 0.f;
        for (int k = 0; k < p.mix.count; ++k) {
            const int c = p.mix.index[k];
            if (staged > width) {
                snprintf(msg, msg_len, "tile at %lld channel %d stages %lld floats into a window of %d",
                         (long long)t0, c, (long long)staged, width);
                return -2;
            }
            for (int i = 0; i < width; ++i) win[(size_t)i] = NAN;
            for (int64_t i = 0; i < staged; ++i) {
                const int64_t f = sbswr::source_frame(p, s0 + i);
                win[(size_t)i] = f < 0 ? 0.f : (float)pcm[f * channels + c] * (1.0f / 32768);
            }
            for (int64_t t = t0; t <= last; ++t) {
                sbswr::position(r, t, &s, &phase, &frac);
                if (s < s0 || s - s0 + r.filter_alloc > staged) {
                    snprintf(msg, msg_len,
                             "output %lld of the tile at %lld channel %d reads [%lld, %lld) of %lld staged",
                             (long long)t, (long long)t0, c, (long long)(s - s0), (long long)(s - s0 + r.filter_alloc),
                             (long long)staged);
                    return -2;
                }
                const float y = sbswr::resample_one(r, bank.data(), win.data() + (s - s0), phase, frac);
                float& acc = v[(size_t)(t - t0)];
                acc = sbswr::fadd(acc, sbswr::fmul(y, p.mix.flt[c]));
            }
        }
        for (int64_t t = t0; t <= last; ++t) out[t] = sbswr::to_s16(v[(size_t)(t - t0)]);
    }
    return 0;
}

// The float bank of a conversion, (phases + 1) x stride floats
int emu_swr_bank(int in_rate, int out_rate, float* bank, char* msg, int msg_len) {
    sbswr::Resampler r;
    if (!sbswr::make_resampler(in_rate, out_rate, &r, msg, msg_len)) return -1;
    std::vector<float> b;
    sbswr::float_bank(r, b);
    memcpy(bank, b.data(), sizeof(float) * b.size());
    return 0;
}

int emu_swr_row(uint64_t layout, double* row, char* msg, int msg_len) {
    return sbswr::mono_row(layout, row, msg, msg_len) ? 0 : -1;
}

double emu_swr_bessel(double x) { return sbswr::bessel_i0(x); }

}  // extern "C"
