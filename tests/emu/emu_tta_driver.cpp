// CPU build of the TTA decoder: sushi_b200/csrc/sb_tta.cuh compiled with g++ (tests/test_kernel_emulation_tta.py).
// The config and the frame table go through the functions sb_tta_decode_frames calls; in place of the kernel, one
// decode_frame per frame, with the channel state in a plain array (stride 1) where the kernel uses a column of shared
// memory.
#include <stdint.h>
#include <vector>

#include "sb_tta.cuh"
#include "emu_guard.h"

extern "C" {

// Decode the n frames listed in buf (nbytes bytes): frame f starts at offsets[f] and ends where frame f + 1 starts,
// the last at nbytes.  config: channels, bits, rate, frame length, last frame length.  pcm receives the interleaved
// int16 samples.  Returns 0, or -1 with the message (naming the frame and file_offsets[f]) in msg.
int emu_tta_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                   const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    sbtta::Config c;
    int32_t rate = 0;
    if (!sbtta::parse_config(config, &c, &rate, msg, msg_len)) return -1;
    std::vector<sbtta::Frame> frames;
    int64_t samples = 0;
    if (!sbtta::frame_table(offsets, file_offsets, n, nbytes, c, frames, &samples, msg, msg_len)) return -1;
    std::vector<int32_t> state(sbtta::kMaxChannels * sbtta::kStateWords);
    std::vector<uint32_t> crc(sbtta::kCrcWords);
    for (int i = 0; i < sbtta::kCrcWords; ++i) sbtta::crc_table_entry(crc.data(), i);
    sbtta::State s;
    s.p = state.data();
    s.stride = 1;
    std::vector<int32_t> status((size_t)n);
    for (int64_t f = 0; f < n; ++f) status[(size_t)f] = sbtta::decode_frame(buf, frames[(size_t)f], c, s, crc.data(), pcm);
    return sbframes::first_failure(status.data(), n, "TTA frame", file_offsets, 1, sbtta::error_text, msg, msg_len) ? 0 : -1;
}

// emu_tta_decode with the data placed so that its last byte is the last readable one (no padding): the next page is
// inaccessible, so a read past the frames faults.
int emu_tta_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets,
                           int64_t n, const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    return emu_guarded(data, nbytes, 0, [&](const uint8_t* buf) {
        return emu_tta_decode(buf, nbytes, offsets, file_offsets, n, config, pcm, msg, msg_len);
    });
}

}  // extern "C"
