// CPU build of the MP2 decoder: sushi_b200/csrc/sb_mp2.cuh compiled with g++ (tests/test_mp2_cases.py).  The frame
// table goes through the function sb_mp2_decode_frames calls; in place of the kernels, unpack_frame per frame, dct32
// per slot and window_sum per output, with the rounding remainder carried from output to output in FFmpeg's order
// where the GPU scans it.
#include <stdint.h>
#include <algorithm>
#include <vector>

#include "sb_mp2.cuh"

extern "C" {

// Decode buf[0, nbytes), the payloads of n blocks back to back (block k starts at offsets[k] and is at file offset
// file_offsets[k]).  *frames: the frames decoded; pcm (room for cap sample frames) the interleaved int16 samples;
// info: channels, rate, 1 when the stream ends inside a frame.  Returns 0, or -1 with the message in msg.
int emu_mp2_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                   int16_t* pcm, int64_t cap, int64_t* frames_out, int32_t* info, char* msg, int msg_len) {
    auto where = [&](int64_t b) {
        const int64_t k = std::upper_bound(offsets, offsets + n, b) - offsets - 1;
        return file_offsets[k] + (b - offsets[k]);
    };
    std::vector<sbmp2::Frame> frames;
    sbmp2::Stream s;
    if (!sbmp2::frame_table(buf, nbytes, where, frames, &s, msg, msg_len)) return -1;
    const int64_t F = (int64_t)frames.size();
    *frames_out = F;
    info[0] = s.channels; info[1] = s.rate; info[2] = s.cut;
    if (F * sbmp2::kFrameSamples > cap) { snprintf(msg, msg_len, "emu_mp2_decode: output too small"); return -1; }
    const sbmp2::Scales sc = sbmp2::make_scales();
    std::vector<int32_t> sb((size_t)(F * s.channels * sbmp2::kFrameSamples));
    for (int64_t f = 0; f < F; ++f) {
        const int code = sbmp2::unpack_frame(buf, nbytes, frames[(size_t)f], f, F, sc, sb.data());
        if (code) {
            sbframes::refuse(msg, msg_len, "MP2 frame", f, where(frames[(size_t)f].offset), sbmp2::error_text(code));
            return -1;
        }
    }
    for (int64_t r = 0; r < F * s.channels * sbmp2::kSlots; ++r) sbmp2::dct32(&sb[(size_t)r * 32], &sb[(size_t)r * 32]);
    uint32_t rem = 0;
    for (int64_t f = 0; f < F; ++f)
        for (int c = 0; c < s.channels; ++c) {
            const int32_t* base = sb.data() + (size_t)c * F * sbmp2::kFrameSamples;
            auto v = [&](int64_t t, int m) -> int32_t { return t < 0 ? 0 : base[t * 32 + m]; };
            for (int slot = 0; slot < sbmp2::kSlots; ++slot) {
                const int64_t t = f * sbmp2::kSlots + slot;
                for (int pos = 0; pos < 32; ++pos) {
                    const int j = sbmp2::emitted(pos);
                    const int64_t sum = sbmp2::window_sum(v, t, j);
                    pcm[(t * 32 + j) * s.channels + c] = sbmp2::round_sample(rem, sum);
                    rem = (uint32_t)((int64_t)(rem & 0xFFFFFF) + sum) & 0xFFFFFFu;
                }
            }
        }
    return 0;
}

// the window entry i and the DCT of one row, for the table probes
int32_t emu_mp2_window(int i) { return sbmp2::window_at(i); }
void emu_mp2_dct(const int32_t* in, int32_t* out) { sbmp2::dct32(out, in); }

}  // extern "C"
