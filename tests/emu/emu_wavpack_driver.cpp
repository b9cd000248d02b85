// CPU build of the WavPack decoder: sushi_b200/csrc/sb_wavpack.cuh compiled with g++, driven the way sb_wavpack.cu
// drives it (tests/test_kernel_emulation_wavpack.py): one decode_block per row of the host's block table, with the term
// state in a plain array (stride 1) where the kernel uses a column of shared memory.
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "sb_wavpack.cuh"

extern "C" {

// Decode the n blocks of table (8 int64 per block: offset, size, samples, flags, crc, sample, channel, file offset) from
// buf (nbytes bytes plus at least 8 readable bytes).  pcm receives `frames` interleaved int16 frames of `channels`
// channels.  Returns 0, or -1 with the message in msg.
int emu_wavpack_decode(const uint8_t* buf, int64_t nbytes, const int64_t* table, int64_t n, int channels,
                       int64_t frames, int16_t* pcm, char* msg, int msg_len) {
    std::vector<int32_t> state(sbwv::kMaxTerms * sbwv::kTermWords);
    sbwv::Terms ts;
    ts.p = state.data();
    ts.stride = 1;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t* r = table + 8 * i;
        sbwv::Block b;
        b.offset = r[0]; b.size = r[1]; b.samples = (int32_t)r[2]; b.flags = (uint32_t)r[3]; b.crc = (uint32_t)r[4];
        b.sample = r[5]; b.channel = (int32_t)r[6];
        const int width = (b.flags & sbwv::kMono) ? 1 : 2;
        if (r[0] < 0 || r[1] < 0 || r[0] > nbytes - r[1] || r[2] < 1 || r[5] + r[2] > frames || r[6] + width > channels) {
            snprintf(msg, msg_len, "WavPack block %lld at byte offset %lld: block table entry out of range",
                     (long long)i, (long long)r[7]);
            return -1;
        }
        const int code = sbwv::decode_block(buf, b, channels, ts, pcm);
        if (code != sbwv::kOk) {
            snprintf(msg, msg_len, "WavPack block %lld at byte offset %lld: %s", (long long)i, (long long)r[7],
                     sbwv::error_text(code));
            return -1;
        }
    }
    return 0;
}

}  // extern "C"

#include <sys/mman.h>
#include <unistd.h>

extern "C" {

// emu_wavpack_decode with the data placed so that the 8 bytes of padding the library guarantees end exactly at an
// inaccessible page: a read further past the last block faults.
int emu_wavpack_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* table, int64_t n, int channels,
                               int64_t frames, int16_t* pcm, char* msg, int msg_len) {
    const int64_t page = sysconf(_SC_PAGESIZE);
    const int64_t body = (nbytes + 8 + page - 1) / page * page;
    uint8_t* base = (uint8_t*)mmap(nullptr, body + page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (base == MAP_FAILED) return -2;
    mprotect(base + body, page, PROT_NONE);
    uint8_t* buf = base + body - 8 - nbytes;
    memcpy(buf, data, (size_t)nbytes);
    memset(buf + nbytes, 0, 8);
    const int r = emu_wavpack_decode(buf, nbytes, table, n, channels, frames, pcm, msg, msg_len);
    munmap(base, body + page);
    return r;
}

}  // extern "C"
