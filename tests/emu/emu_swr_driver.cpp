// CPU build of the mono downmix and resampler: sushi_b200/csrc/sb_swr.cuh compiled with g++
// (tests/test_swr_cases.py).  The plan, the matrix and the bank are the functions sb_pcm_swr calls; in place of the
// kernels, one loop over the outputs, each reading the whole filter signal instead of a staged window.
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
