// CPU build of the listed-frame path of the FLAC decoder: sushi_b200/csrc/sb_flac.cuh compiled with g++, driven the way
// sb_flac_decode_frames drives it (tests/test_kernel_emulation_mkv_flac.py).  Each listed frame's
// header is checked at its offset (k_flac_frames), the frame table is built from the block sizes, every frame is
// decoded and checked against its lace end (k_flac_decode), and the channels are decorrelated (k_flac_decorrelate).
// For comparison, emu_flac_chain_table builds the table sb_flac_decode_file builds from a whole FLAC file.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "sb_flac.cuh"

namespace {

void put_table(const std::vector<sbflac::FrameDesc>& frames, int64_t* table) {
    for (size_t f = 0; f < frames.size(); ++f) {
        const sbflac::FrameDesc& d = frames[f];
        table[5 * f + 0] = d.offset; table[5 * f + 1] = d.limit; table[5 * f + 2] = d.sample;
        table[5 * f + 3] = d.block_size; table[5 * f + 4] = d.assignment;
    }
}

bool listed(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* where, int64_t n, int channels,
            int bits, int rate, std::vector<sbflac::FrameDesc>& frames, int64_t* samples, char* msg, int msg_len) {
    std::vector<sbflac::ListedFrame> out((size_t)n);
    for (int64_t f = 0; f < n; ++f) out[f] = sbflac::listed_frame(buf, nbytes, offsets, n, f, channels, bits, rate);
    return sbflac::list_frames(out.data(), offsets, where, n, nbytes, frames, samples, msg, msg_len);
}

}  // namespace

extern "C" {

// The table of listed frames into table[n * 5] (offset, limit, sample, block size, assignment).  Returns the samples
// per channel, or -1 with the message in msg.
int64_t emu_flac_frames(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* where, int64_t n,
                        int channels, int bits, int rate, int64_t* table, char* msg, int msg_len) {
    std::vector<sbflac::FrameDesc> frames;
    int64_t samples = 0;
    if (!listed(buf, nbytes, offsets, where, n, channels, bits, rate, frames, &samples, msg, msg_len)) return -1;
    put_table(frames, table);
    return samples;
}

// sb_flac_decode_file's chained table of a whole FLAC file (frames found by their sync codes and coded numbers).  Returns
// the frame count (table filled when it fits in `cap` frames), or -1 with the message in msg.
int64_t emu_flac_chain_table(const uint8_t* file, int64_t nbytes, int64_t first, int channels, int bits, int rate,
                             int64_t* table, int64_t cap, char* msg, int msg_len) {
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
    if ((int64_t)frames.size() <= cap) put_table(frames, table);
    return (int64_t)frames.size();
}

// Decode the listed frames into pcm[samples * channels] (int16, interleaved).  Returns 0, or -1 with the message.
int emu_flac_frames_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* where, int64_t n,
                           int channels, int bits, int rate, int16_t* pcm, char* msg, int msg_len) {
    std::vector<sbflac::FrameDesc> frames;
    int64_t samples = 0;
    if (!listed(buf, nbytes, offsets, where, n, channels, bits, rate, frames, &samples, msg, msg_len)) return -1;
    uint16_t crc[256];
    for (int i = 0; i < 256; ++i) crc[i] = sbflac::crc16_entry(i);
    std::vector<int32_t> planar((size_t)samples * channels + 1);
    std::vector<sbflac::FrameStatus> status(frames.size());
    for (size_t f = 0; f < frames.size(); ++f) {
        const sbflac::FrameDesc& d = frames[f];
        status[f].pad = 0;
        status[f].code = sbflac::decode_frame(buf, d.offset, d.limit, channels, bits, rate, crc,
                                              planar.data() + d.sample * channels, &status[f].end);
    }
    auto bytes_at = [&](int64_t off, uint8_t* out) {
        if (off < nbytes) memcpy(out, buf + off, (size_t)(nbytes - off < 16 ? nbytes - off : 16));
    };
    if (!sbflac::check_frames(frames, status.data(), nbytes, channels, bits, rate, bytes_at, msg, msg_len, where)) return -1;
    for (const sbflac::FrameDesc& d : frames)
        for (int j = 0; j < d.block_size; ++j)
            sbflac::decorrelate(planar.data() + d.sample * channels, d.block_size, j, channels, d.assignment, bits,
                                pcm + (d.sample + j) * channels);
    return 0;
}

}  // extern "C"
