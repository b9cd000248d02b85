// CPU build of the ALAC decoder: sushi_b200/csrc/sb_alac.cuh compiled with g++ (tests/test_kernel_emulation_alac.py).
// The config, the offsets and the frame table go through the functions sb_alac_decode_frames calls; in place of the
// kernels, each listed frame's first element gives its sample count (k_alac_frames) and each frame is decoded from its
// own scratch (k_alac_decode).
#include <stdint.h>
#include <string.h>
#include <vector>

#include "sb_alac.cuh"
#include "emu_guard.h"

extern "C" {

// Decode the frames at offsets[0..n) of buf (nbytes bytes plus at least 8 readable zero bytes; where[]: each frame's
// file offset, for messages).  pcm receives the interleaved int16 frames (at most cap; NULL: count only).  Returns the
// sample count per channel, or -1 with the message in msg.
int64_t emu_alac_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* where, int64_t n,
                        const int32_t* config, int16_t* pcm, int64_t cap, char* msg, int msg_len) {
    sbalac::Config c;
    if (!sbalac::parse_config(config, &c, msg, msg_len)) return -1;
    if (!sbalac::check_offsets(offsets, where, n, nbytes, msg, msg_len)) return -1;
    std::vector<sbalac::Listed> listed((size_t)n);
    for (int64_t f = 0; f < n; ++f)
        listed[(size_t)f] = sbalac::first_element(buf, offsets[f], f + 1 < n ? offsets[f + 1] : nbytes, c);
    std::vector<sbalac::FrameDesc> frames;
    int64_t total = 0;
    if (!sbalac::frame_table(listed.data(), offsets, where, n, nbytes, frames, &total, msg, msg_len)) return -1;
    std::vector<int16_t> out((size_t)(total * c.channels + 1));
    std::vector<int32_t> scratch((size_t)(2 * c.frame_length));
    std::vector<int32_t> status((size_t)n);
    for (int64_t f = 0; f < n; ++f) {
        const sbalac::FrameDesc& d = frames[(size_t)f];
        status[(size_t)f] = sbalac::decode_frame(buf, d.offset, d.limit, c, listed[(size_t)f].samples, scratch.data(),
                                                 out.data() + d.sample * c.channels);
    }
    if (!sbframes::first_failure(status.data(), n, "ALAC frame", where, 1, sbalac::error_text, msg, msg_len)) return -1;
    if (pcm) memcpy(pcm, out.data(), sizeof(int16_t) * (size_t)(total < cap ? total : cap) * c.channels);
    return total;
}

// emu_alac_decode with the frames placed so that the 8 bytes of padding the library guarantees end exactly at an
// inaccessible page: a read further past the last frame faults.  Returns what emu_alac_decode returns.
int64_t emu_alac_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* offsets, const int64_t* where,
                                int64_t n, const int32_t* config, char* msg, int msg_len) {
    return emu_guarded(data, nbytes, 8, [&](const uint8_t* buf) {
        return emu_alac_decode(buf, nbytes, offsets, where, n, config, nullptr, 0, msg, msg_len);
    });
}

}  // extern "C"
