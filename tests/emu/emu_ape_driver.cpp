// CPU build of the APE decoder: sushi_b200/csrc/sb_ape.cuh compiled with g++ (tests/test_kernel_emulation_ape.py).
// The config and the frame table go through the functions sb_ape_decode_frames calls; in place of the kernels, each
// stage as a loop: entropy_frame per frame; per (frame, coded channel) every NN filter with the 32 lanes' lane_step run
// one after another on their own weights and their partial dot products summed in 32-bit wrap-around, as the warp
// reduction sums them; predictor_frame per frame; and the CRC as 32 slices joined by crc_combine in the kernel's order.
#include <stdint.h>
#include <algorithm>
#include <vector>

#include "sb_ape.cuh"
#include "emu_guard.h"

namespace {

template <int T>
void nn_filter(int32_t* d, int64_t stride, int32_t blocks, int order, int frac) {
    std::vector<int16_t> hist(sbape::kRing, 0), adapt(sbape::kRing, 0);
    sbape::NnShared s{hist.data(), adapt.data()};
    std::vector<std::vector<int32_t>> w(32, std::vector<int32_t>(T, 0));
    int32_t avg = 0;
    for (int64_t t = 0; t < blocks; ++t) {
        const int32_t in = d[t * stride];
        uint32_t dot = 0;
        for (int lane = 0; lane < 32; ++lane) {
            int32_t(&wl)[T] = *reinterpret_cast<int32_t(*)[T]>(w[(size_t)lane].data());
            dot += sbape::lane_step<T>(wl, lane, order, s, t, sbape::sign_neg(in));
        }
        int16_t h, a;
        d[t * stride] = sbape::finish(dot, frac, in, avg, h, a);
        hist[(size_t)(t & (sbape::kRing - 1))] = h;
        adapt[(size_t)(t & (sbape::kRing - 1))] = a;
    }
}

void nn_channel(int32_t* d, int64_t stride, int32_t blocks, int fset) {
    for (int l = 0; l < sbape::kLevels; ++l) {
        const int order = sbape::filter_order(fset, l), frac = sbape::filter_frac(fset, l);
        if (!order) break;
        switch (order) {
        case 16: case 32: nn_filter<1>(d, stride, blocks, order, frac); break;
        case 64: nn_filter<2>(d, stride, blocks, order, frac); break;
        case 256: nn_filter<8>(d, stride, blocks, order, frac); break;
        default: nn_filter<40>(d, stride, blocks, order, frac); break;
        }
    }
}

uint32_t frame_crc(const int32_t* s, int64_t total, int bits, const uint32_t* table) {
    const int64_t per = (total + 31) / 32;
    uint32_t crc[32];
    int64_t len[32];
    for (int lane = 0; lane < 32; ++lane) {
        const int64_t lo = std::min(total, per * lane), hi = std::min(total, lo + per);
        crc[lane] = sbape::crc_bytes(s, lo, hi, bits, table);
        len[lane] = (hi - lo) * (bits / 8);
    }
    for (int step = 1; step < 32; step <<= 1)
        for (int lane = 0; lane + step < 32; lane += 2 * step) {
            if (len[lane + step]) crc[lane] = sbape::crc_combine(crc[lane], crc[lane + step], len[lane + step]);
            len[lane] += len[lane + step];
        }
    return crc[0];
}

}  // namespace

extern "C" {

// Decode the n frames at offsets[f] of buf (nbytes bytes).  config: channels, bits, rate, compression level, blocks
// per frame, last frame's blocks.  pcm receives the interleaved int16 samples.  Returns 0, or -1 with the message
// (naming the frame and file_offsets[f]) in msg.
int emu_ape_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                   const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    sbape::Config c;
    int32_t rate = 0;
    if (!sbape::parse_config(config, &c, &rate, msg, msg_len)) return -1;
    std::vector<sbape::Frame> frames;
    int64_t samples = 0;
    if (!sbape::frame_table(offsets, file_offsets, n, nbytes, c, frames, &samples, msg, msg_len)) return -1;
    std::vector<int32_t> scratch((size_t)(samples * c.channels), 0), kind((size_t)n), status((size_t)n);
    std::vector<uint32_t> stored((size_t)n), table(256);
    for (uint32_t i = 0; i < 256; ++i) table[i] = sbape::crc_entry(i);
    for (int64_t f = 0; f < n; ++f) {
        int32_t kd;
        uint32_t w = 0;
        status[(size_t)f] = sbape::entropy_frame(buf, frames[(size_t)f], c, scratch.data(), &kd, &w);
        kind[(size_t)f] = kd;
        stored[(size_t)f] = w;
    }
    for (int64_t f = 0; f < n; ++f) {
        if (status[(size_t)f] || kind[(size_t)f] == sbape::kSilence) continue;
        const sbape::Frame& fr = frames[(size_t)f];
        const int coded = kind[(size_t)f] == sbape::kStereo ? 2 : 1;
        for (int ch = 0; ch < coded; ++ch)
            nn_channel(scratch.data() + fr.sample * c.channels + ch, c.channels, fr.blocks, c.fset);
    }
    for (int64_t f = 0; f < n; ++f)
        if (!status[(size_t)f])
            status[(size_t)f] = sbape::predictor_frame(frames[(size_t)f], c, kind[(size_t)f], scratch.data(), pcm);
    for (int64_t f = 0; f < n; ++f) {
        if (status[(size_t)f]) continue;
        const sbape::Frame& fr = frames[(size_t)f];
        const uint32_t crc = frame_crc(scratch.data() + fr.sample * c.channels, (int64_t)fr.blocks * c.channels, c.bits,
                                       table.data());
        status[(size_t)f] = sbape::check_crc(crc, stored[(size_t)f]);
    }
    return sbframes::first_failure(status.data(), n, "APE frame", file_offsets, 1, sbape::error_text, msg, msg_len) ? 0
                                                                                                                 : -1;
}

// emu_ape_decode with the data placed so that its last byte is the last readable one (no padding): the next page is
// inaccessible, so a read past the frames faults.
int emu_ape_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets,
                           int64_t n, const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    return emu_guarded(data, nbytes, 0, [&](const uint8_t* buf) {
        return emu_ape_decode(buf, nbytes, offsets, file_offsets, n, config, pcm, msg, msg_len);
    });
}

}  // extern "C"
