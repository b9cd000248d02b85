// CPU build of the FLAC decoder: sushi_b200/csrc/sb_flac.cuh compiled with g++, driven the way sb_flac.cu drives it
// (tests/test_kernel_emulation_flac.py).  Every byte position is tried as a frame header (k_flac_sync), the frames are
// chained, every frame is decoded into the planar buffer and checked (k_flac_decode), and the channels are decorrelated
// into interleaved int16 (k_flac_decorrelate).  The chain and the checks are the library's own functions.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "sb_flac.cuh"

extern "C" {

// Index: the decoded samples per channel, or -1 with the message in msg.
int64_t emu_flac_index(const uint8_t* file, int64_t nbytes, int64_t first, int channels, int bits, int rate,
                       char* msg, int msg_len) {
    std::vector<sbflac::Candidate> cand;
    for (int64_t i = first; i + 1 < nbytes; ++i) {
        if (file[i] != 0xFF || (file[i + 1] & 0xFE) != 0xF8) continue;
        sbflac::Header h;
        if (sbflac::parse_header(file + i, nbytes - i, channels, bits, rate, &h) != sbflac::kOk) continue;
        sbflac::Candidate c;
        c.offset = i; c.number = h.number; c.block_size = h.block_size;
        c.assignment = (int16_t)h.assignment; c.variable = (int16_t)h.variable;
        cand.push_back(c);
    }
    std::vector<sbflac::FrameDesc> frames;
    int64_t samples = 0;
    if (!sbflac::chain(cand, first, nbytes, channels, bits, rate, file + first, frames, &samples, msg, msg_len)) return -1;
    return samples;
}

// Decode into pcm[samples * channels] (int16, interleaved).  Returns 0, or -1 with the message in msg.
int emu_flac_decode(const uint8_t* file, int64_t nbytes, int64_t first, int channels, int bits, int rate, int16_t* pcm,
                    char* msg, int msg_len) {
    std::vector<sbflac::Candidate> cand;
    for (int64_t i = first; i + 1 < nbytes; ++i) {
        if (file[i] != 0xFF || (file[i + 1] & 0xFE) != 0xF8) continue;
        sbflac::Header h;
        if (sbflac::parse_header(file + i, nbytes - i, channels, bits, rate, &h) != sbflac::kOk) continue;
        sbflac::Candidate c;
        c.offset = i; c.number = h.number; c.block_size = h.block_size;
        c.assignment = (int16_t)h.assignment; c.variable = (int16_t)h.variable;
        cand.push_back(c);
    }
    std::vector<sbflac::FrameDesc> frames;
    int64_t samples = 0;
    if (!sbflac::chain(cand, first, nbytes, channels, bits, rate, file + first, frames, &samples, msg, msg_len)) return -1;
    uint16_t table[256];
    for (int i = 0; i < 256; ++i) table[i] = sbflac::crc16_entry(i);
    std::vector<int32_t> planar((size_t)samples * channels + 1);
    std::vector<sbflac::FrameStatus> status(frames.size());
    for (size_t f = 0; f < frames.size(); ++f) {
        const sbflac::FrameDesc& d = frames[f];
        status[f].pad = 0;
        status[f].code = sbflac::decode_frame(file, d.offset, d.limit, channels, bits, rate, table,
                                              planar.data() + d.sample * channels, &status[f].end);
    }
    auto bytes_at = [&](int64_t off, uint8_t* buf) {
        if (off < nbytes) memcpy(buf, file + off, (size_t)(nbytes - off < 16 ? nbytes - off : 16));
    };
    if (!sbflac::check_frames(frames, status.data(), nbytes, channels, bits, rate, bytes_at, msg, msg_len)) return -1;
    for (const sbflac::FrameDesc& d : frames)
        for (int j = 0; j < d.block_size; ++j)
            sbflac::decorrelate(planar.data() + d.sample * channels, d.block_size, j, channels, d.assignment, bits,
                                pcm + (d.sample + j) * channels);
    return 0;
}

}  // extern "C"
