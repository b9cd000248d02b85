// CPU build of the WavPack decoder: sushi_b200/csrc/sb_wavpack.cuh compiled with g++
// (tests/test_kernel_emulation_wavpack.py).  The block table goes through the function sb_wavpack_decode_blocks calls;
// in place of the kernel, one decode_block per block, with the term state in a plain array (stride 1) where the kernel
// uses a column of shared memory.
#include <stdint.h>
#include <stdio.h>
#include <vector>

#include "sb_wavpack.cuh"
#include "emu_guard.h"

extern "C" {

// Decode the n blocks of table (8 int64 per block: offset, size, samples, flags, crc, sample, channel, file offset) from
// buf (nbytes bytes plus at least 8 readable bytes).  pcm has room for `frames` interleaved int16 frames of `channels`
// channels.  Returns 0, or -1 with the message in msg.
int emu_wavpack_decode(const uint8_t* buf, int64_t nbytes, const int64_t* table, int64_t n, int channels,
                       int64_t frames, int16_t* pcm, char* msg, int msg_len) {
    std::vector<sbwv::Block> blocks;
    int64_t samples = 0;
    if (!sbwv::block_table(table, n, nbytes, channels, blocks, &samples, msg, msg_len)) return -1;
    if (samples > frames) {
        snprintf(msg, msg_len, "the blocks hold %lld frames, pcm has room for %lld", (long long)samples, (long long)frames);
        return -1;
    }
    std::vector<int32_t> state(sbwv::kMaxTerms * sbwv::kTermWords);
    sbwv::Terms ts;
    ts.p = state.data();
    ts.stride = 1;
    std::vector<int32_t> status((size_t)n);
    for (int64_t i = 0; i < n; ++i) status[(size_t)i] = sbwv::decode_block(buf, blocks[(size_t)i], channels, ts, pcm);
    return sbframes::first_failure(status.data(), n, "WavPack block", table + 7, 8, sbwv::error_text, msg, msg_len) ? 0 : -1;
}

// emu_wavpack_decode with the data placed so that the 8 bytes of padding the library guarantees end exactly at an
// inaccessible page: a read further past the last block faults.
int emu_wavpack_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* table, int64_t n, int channels,
                               int64_t frames, int16_t* pcm, char* msg, int msg_len) {
    return emu_guarded(data, nbytes, 8, [&](const uint8_t* buf) {
        return emu_wavpack_decode(buf, nbytes, table, n, channels, frames, pcm, msg, msg_len);
    });
}

}  // extern "C"
