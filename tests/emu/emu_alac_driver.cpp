// CPU build of the ALAC decoder: sushi_b200/csrc/sb_alac.cuh compiled with g++, driven the way sb_alac.cu drives it
// (tests/test_kernel_emulation_alac.py).  Each listed frame's first element gives its sample count (k_alac_frames),
// sample positions are the prefix sum, and each frame is decoded from its own scratch (k_alac_decode).
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "sb_alac.cuh"

extern "C" {

// Decode the frames at offsets[0..n) of buf (nbytes bytes plus at least 8 readable zero bytes; where[]: each frame's
// file offset, for messages).  pcm receives the interleaved int16 frames (at most cap; NULL: count only).  Returns the
// sample count per channel, or -1 with the message in msg.
int64_t emu_alac_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* where, int64_t n,
                        const int32_t* config, int16_t* pcm, int64_t cap, char* msg, int msg_len) {
    sbalac::Config c;
    c.frame_length = config[0]; c.bit_depth = config[1]; c.pb = config[2]; c.mb = config[3]; c.kb = config[4];
    c.channels = config[5]; c.rate = config[6];
    std::vector<sbalac::Listed> listed((size_t)n);
    std::vector<int64_t> first((size_t)n + 1, 0);
    for (int64_t f = 0; f < n; ++f) {
        const int64_t lim = f + 1 < n ? offsets[f + 1] : nbytes;
        if (lim <= offsets[f]) {
            snprintf(msg, msg_len, "ALAC frame %lld at byte offset %lld: empty frame", (long long)f, (long long)where[f]);
            return -1;
        }
        listed[(size_t)f] = sbalac::first_element(buf, offsets[f], lim, c);
        if (listed[(size_t)f].code != sbalac::kOk) {
            snprintf(msg, msg_len, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)where[f],
                     sbalac::error_text(listed[(size_t)f].code));
            return -1;
        }
        first[(size_t)f + 1] = first[(size_t)f] + listed[(size_t)f].samples;
    }
    const int64_t total = first[(size_t)n];
    std::vector<int16_t> out((size_t)(total * c.channels + 1));
    std::vector<int32_t> scratch((size_t)(2 * c.frame_length));
    for (int64_t f = 0; f < n; ++f) {
        const int64_t lim = f + 1 < n ? offsets[f + 1] : nbytes;
        const int code = sbalac::decode_frame(buf, offsets[f], lim, c, listed[(size_t)f].samples, scratch.data(),
                                              out.data() + first[(size_t)f] * c.channels);
        if (code != sbalac::kOk) {
            snprintf(msg, msg_len, "ALAC frame %lld at byte offset %lld: %s", (long long)f, (long long)where[f],
                     sbalac::error_text(code));
            return -1;
        }
    }
    if (pcm) memcpy(pcm, out.data(), sizeof(int16_t) * (size_t)(total < cap ? total : cap) * c.channels);
    return total;
}

}  // extern "C"

#include <sys/mman.h>
#include <unistd.h>

extern "C" {

// emu_alac_decode with the frames placed so that the 8 bytes of padding the library guarantees end exactly at an
// inaccessible page: a read further past the last frame faults.  Returns what emu_alac_decode returns.
int64_t emu_alac_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* offsets, const int64_t* where,
                                int64_t n, const int32_t* config, char* msg, int msg_len) {
    const int64_t page = sysconf(_SC_PAGESIZE);
    const int64_t body = (nbytes + 8 + page - 1) / page * page;
    uint8_t* base = (uint8_t*)mmap(nullptr, body + page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (base == MAP_FAILED) return -2;
    mprotect(base + body, page, PROT_NONE);
    uint8_t* buf = base + body - 8 - nbytes;
    memcpy(buf, data, (size_t)nbytes);
    memset(buf + nbytes, 0, 8);
    const int64_t r = emu_alac_decode(buf, nbytes, offsets, where, n, config, nullptr, 0, msg, msg_len);
    munmap(base, body + page);
    return r;
}

}  // extern "C"
