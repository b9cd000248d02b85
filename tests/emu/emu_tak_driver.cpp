// CPU build of the TAK decoder: sushi_b200/csrc/sb_tak.cuh compiled with g++ (tests/test_kernel_emulation_tak.py).
// The config and the frame table go through the functions sb_tak_decode_file calls; in place of the kernels, each stage
// as a loop: the sync test at every byte; entropy_frame per frame; per (frame, channel) each filtered subframe with the
// recurrence's pair steps and the 32 lanes' lane_part run one after another, their partial dot products summed in
// 32-bit wrap-around as the warp reduction sums them; per frame the decorrelation sample by sample and the lpc modes as
// k_tak_finish's chunked block scan (256 chunks, their sums carried across); and the CRC as 32 slices joined by
// crc_combine in the kernel's order.
#include <stdint.h>
#include <algorithm>
#include <random>
#include <vector>

#include "sb_tak.cuh"
#include "emu_guard.h"

namespace {

constexpr int kFinishThreads = 256;

struct Warp {
    std::vector<int16_t> ring = std::vector<int16_t>(sbtak::kRing), filter = std::vector<int16_t>(sbtak::kMaxOrder),
                         pred = std::vector<int16_t>(sbtak::kMaxOrder);
    std::vector<int32_t> t = std::vector<int32_t>(sbtak::kMaxOrder);
};

// k_tak_filter's filter_sub once the parameters are read: the recurrence and the lane-split filter
void filter_warp(int32_t* d, int hist, int order, int count, int quant, int dshift, Warp& s) {
    if (order > 0) s.t[0] = s.pred[0] * 64;
    for (int i = 1; i < order; ++i) {
        for (int lane = 0; lane < 32; ++lane)
            for (int j = lane; j < (i + 1) / 2; j += 32) sbtak::taps_pair(s.t.data(), i, j, s.pred[(size_t)i]);
        s.t[(size_t)i] = s.pred[(size_t)i] * 64;
    }
    for (int k = 0; k < order; ++k) s.filter[(size_t)k] = sbtak::tap(s.t.data(), order, quant, k);
    for (int k = 0; k < order; ++k) s.ring[(size_t)k] = (int16_t)(d[hist + k] >> dshift);
    int32_t* out = d + hist + order;
    for (int64_t t = 0; t < count; ++t) {
        uint32_t dot = 0;
        for (int lane = 0; lane < 32; ++lane) dot += sbtak::lane_part(s.ring.data(), s.filter.data(), order, t, lane);
        const int32_t v = sbtak::finish_sample(dot, quant, dshift, out[t]);
        s.ring[(size_t)((t + order) & (sbtak::kRing - 1))] = (int16_t)(v >> dshift);
        out[t] = v;
    }
}

// k_tak_finish's block_scan: 256 chunks of d[lo, hi), each chunk's sum carried into the later ones
void block_scan(int32_t* d, int lo, int hi) {
    const int len = hi - lo, per = (len + kFinishThreads - 1) / kFinishThreads;
    std::vector<uint32_t> sums(kFinishThreads, 0);
    for (int tid = 0; tid < kFinishThreads; ++tid) {
        const int a = std::min(hi, lo + tid * per), b = std::min(hi, a + per);
        for (int i = a; i < b; ++i) sums[(size_t)tid] += (uint32_t)d[i];
    }
    uint32_t acc = 0;
    for (int tid = 0; tid < kFinishThreads; ++tid) {
        const int a = std::min(hi, lo + tid * per), b = std::min(hi, a + per);
        uint32_t run = acc;
        for (int i = a; i < b; ++i) {
            run += (uint32_t)d[i];
            d[i] = (int32_t)run;
        }
        acc += sums[(size_t)tid];
    }
}

uint32_t frame_crc(const uint8_t* buf, int64_t lo0, int64_t hi0, const uint32_t* table) {
    const int64_t total = hi0 - lo0, per = (total + 31) / 32;
    uint32_t crc[32];
    int64_t len[32];
    for (int lane = 0; lane < 32; ++lane) {
        const int64_t lo = lo0 + std::min(total, per * lane), hi = std::min(hi0, lo + per);
        crc[lane] = sbtak::crc_bytes(buf, lo, hi, lane == 0 ? sbtak::kCrcInit : 0u, table);
        len[lane] = hi - lo;
    }
    for (int step = 1; step < 32; step <<= 1)
        for (int lane = 0; lane + step < 32; lane += 2 * step) {
            if (len[lane + step]) crc[lane] = sbtak::crc_combine(crc[lane], crc[lane + step], len[lane + step]);
            len[lane] += len[lane + step];
        }
    return crc[0];
}

// the sync stage and the frame table
bool table(const uint8_t* buf, int64_t audio_start, int64_t audio_end, const sbtak::Config& c,
           std::vector<sbtak::Frame>& frames, int64_t* samples, char* msg, int msg_len) {
    std::vector<sbtak::Candidate> cand;
    for (int64_t i = audio_start; i < audio_end; ++i) {
        sbtak::Candidate h;
        if (buf[i] == 0xFF && sbtak::parse_header(buf, audio_end, i, c, &h)) cand.push_back(h);
    }
    return sbtak::frame_table(cand.data(), (int64_t)cand.size(), audio_start, audio_end, c, frames, samples, msg,
                              (size_t)msg_len);
}

}  // namespace

extern "C" {

// The frame table of the file: n_out frames, frame f spanning [start[f], end[f]).  Returns 0, or -1 with the message.
int emu_tak_frames(const uint8_t* buf, int64_t nbytes, int64_t audio_start, int64_t audio_end, const int32_t* config,
                   int64_t* start, int64_t* end, int64_t cap, int64_t* n_out, char* msg, int msg_len) {
    sbtak::Config c;
    if (!sbtak::parse_config(config, &c, msg, (size_t)msg_len)) return -1;
    std::vector<sbtak::Frame> frames;
    int64_t samples = 0;
    (void)nbytes;
    if (!table(buf, audio_start, audio_end, c, frames, &samples, msg, msg_len)) return -1;
    *n_out = (int64_t)frames.size();
    for (int64_t f = 0; f < (int64_t)frames.size() && f < cap; ++f) {
        start[f] = frames[(size_t)f].start;
        end[f] = frames[(size_t)f].end;
    }
    return 0;
}

// Decode the file (nbytes bytes, audio in [audio_start, audio_end)).  config: as sb_tak_decode_file's.  pcm receives
// the interleaved int16 samples (room for the stream info's total).  Returns 0, or -1 with the message in msg.
int emu_tak_decode(const uint8_t* buf, int64_t nbytes, int64_t audio_start, int64_t audio_end, const int32_t* config,
                   int16_t* pcm, char* msg, int msg_len) {
    sbtak::Config c;
    if (!sbtak::parse_config(config, &c, msg, (size_t)msg_len)) return -1;
    if (nbytes < 1 || audio_start < 0 || audio_end <= audio_start || audio_end > nbytes) {
        snprintf(msg, (size_t)msg_len, "sb_tak_decode_file: bad stream parameters");
        return -1;
    }
    std::vector<sbtak::Frame> frames;
    int64_t samples = 0;
    if (!table(buf, audio_start, audio_end, c, frames, &samples, msg, msg_len)) return -1;
    const int64_t n = (int64_t)frames.size();
    std::vector<int32_t> scratch((size_t)(samples * c.channels), 0), status((size_t)n);
    std::vector<sbtak::Sub> subs((size_t)(n * c.channels * sbtak::kMaxSubframes));
    std::vector<sbtak::State> state((size_t)n);
    std::vector<int64_t> where((size_t)n);
    std::vector<uint32_t> crc_table(256);
    for (uint32_t i = 0; i < 256; ++i) crc_table[i] = sbtak::crc_entry(i);
    for (int64_t f = 0; f < n; ++f) {
        where[(size_t)f] = frames[(size_t)f].start;
        status[(size_t)f] = sbtak::entropy_frame(buf, nbytes, frames[(size_t)f], c, scratch.data(),
                                                 subs.data() + f * c.channels * sbtak::kMaxSubframes,
                                                 &state[(size_t)f]);
    }
    Warp w;
    for (int64_t f = 0; f < n; ++f) {
        if (status[(size_t)f]) continue;
        const sbtak::Frame& fr = frames[(size_t)f];
        for (int ch = 0; ch < c.channels; ++ch) {
            int32_t* d = scratch.data() + fr.sample * c.channels + (int64_t)ch * fr.nb;
            const sbtak::Sub* u = subs.data() + (f * c.channels + ch) * sbtak::kMaxSubframes;
            for (int k = 0; k < state[(size_t)f].nsub[ch]; ++k) {
                sbtak::FilterParams p;
                sbtak::read_filter(buf, nbytes, u[k].bits, u[k].order, w.pred.data(), &p);
                filter_warp(d, u[k].hist, u[k].order, u[k].count, p.quant, p.dshift, w);
            }
        }
    }
    for (int64_t f = 0; f < n; ++f) {
        if (status[(size_t)f]) continue;
        const sbtak::Frame& fr = frames[(size_t)f];
        const sbtak::State& s = state[(size_t)f];
        int32_t* base = scratch.data() + fr.sample * c.channels;
        const int nb = fr.nb;
        if (!s.raw) {
            for (int k = 0; k < s.npairs; ++k) {
                sbtak::Decor dec;
                sbtak::read_decor(buf, nbytes, s.pair[k], &dec);
                for (int i = 0; i < nb; ++i)
                    sbtak::decorrelate_sample(dec, base + (int64_t)s.pair[k].c1 * nb, base + (int64_t)s.pair[k].c2 * nb,
                                              nb, i);
            }
            for (int ch = 0; ch < c.channels; ++ch)
                if (nb >= 2)
                    for (int l = 1; l <= s.lpc[ch]; ++l) block_scan(base + (int64_t)ch * nb, s.lpc[ch] - l, nb);
        }
        for (int i = 0; i < nb; ++i)
            for (int ch = 0; ch < c.channels; ++ch)
                pcm[(fr.sample + i) * c.channels + ch] =
                    sbtak::store(base[(int64_t)ch * nb + i], s.raw ? 0 : s.shift[ch], c.bits);
        const int64_t hi = s.data_end - 3;
        if (frame_crc(buf, fr.start + fr.hsize, hi, crc_table.data()) != sbtak::stored_crc(buf + hi))
            status[(size_t)f] = sbtak::kCrc;
    }
    return sbframes::first_failure(status.data(), n, "TAK frame", where.data(), 1, sbtak::error_text, msg,
                                   (size_t)msg_len) ? 0 : -1;
}

// emu_tak_decode with the file placed so that its last byte is the last readable one (no padding): the next page is
// inaccessible, so a read past the file faults.
int emu_tak_decode_guarded(const uint8_t* data, int64_t nbytes, int64_t audio_start, int64_t audio_end,
                           const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    return emu_guarded(data, nbytes, 0, [&](const uint8_t* buf) {
        return emu_tak_decode(buf, nbytes, audio_start, audio_end, config, pcm, msg, msg_len);
    });
}

// The warp-split filter (recurrence pair steps across lanes, lane-split dot product over the ring) against FFmpeg's
// loop as it writes it, on seeded predictors, history and residuals: 0 when they agree.
int emu_tak_filter_check(int order, int count, int quant, int dshift, uint64_t seed) {
    std::mt19937_64 rng(seed);
    Warp w;
    for (int i = 0; i < order; ++i) w.pred[(size_t)i] = (int16_t)((int)(rng() % 1024) - 512);
    std::vector<int32_t> a((size_t)(order + count)), b;
    for (auto& v : a) v = (int32_t)(rng() >> 32);
    b = a;
    filter_warp(a.data(), 0, order, count, quant, dshift, w);
    std::vector<int32_t> t((size_t)std::max(order, 1));
    std::vector<int16_t> filter((size_t)std::max(order, 1));
    sbtak::filter_taps_serial(w.pred.data(), order, quant, t.data(), filter.data());
    sbtak::filter_serial(b.data(), order, count, quant, dshift, filter.data());
    return a == b ? 0 : -1;
}

// The chunked block scans of an lpc mode against the plain serial prefix sums, on seeded values: 0 when they agree.
int emu_tak_scan_check(int mode, int n, uint64_t seed) {
    std::mt19937_64 rng(seed);
    std::vector<int32_t> a((size_t)n), b;
    for (auto& v : a) v = (int32_t)(rng() >> 32);
    b = a;
    for (int l = 1; l <= mode; ++l) block_scan(a.data(), mode - l, n);
    sbtak::lpc_serial(b.data(), mode, n);
    return a == b ? 0 : -1;
}

}  // extern "C"
