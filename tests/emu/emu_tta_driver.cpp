// CPU build of the TTA decoder: sushi_b200/csrc/sb_tta.cuh compiled with g++, driven the way sb_tta.cu drives it
// (tests/test_kernel_emulation_tta.py): one decode_frame per frame of the host's frame table, with the channel state in
// a plain array (stride 1) where the kernel uses a column of shared memory.
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "sb_tta.cuh"

extern "C" {

// Decode the n frames listed in buf (nbytes bytes): frame f starts at offsets[f] and ends where frame f + 1 starts,
// the last at nbytes.  config: channels, bits, rate, frame length, last frame length.  pcm receives the interleaved
// int16 samples.  Returns 0, or -1 with the message (naming the frame and file_offsets[f]) in msg.
int emu_tta_decode(const uint8_t* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                   const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    sbtta::Config c;
    c.channels = config[0]; c.bits = config[1]; c.frame_length = config[3]; c.last_length = config[4];
    std::vector<int32_t> state(sbtta::kMaxChannels * sbtta::kStateWords);
    std::vector<uint32_t> crc(sbtta::kCrcWords);
    for (int i = 0; i < sbtta::kCrcWords; ++i) sbtta::crc_table_entry(crc.data(), i);
    sbtta::State s;
    s.p = state.data();
    s.stride = 1;
    for (int64_t f = 0; f < n; ++f) {
        const int64_t end = f + 1 < n ? offsets[f + 1] : nbytes;
        if (offsets[f] < 0 || offsets[f] >= nbytes || end <= offsets[f] || end > nbytes) {
            snprintf(msg, msg_len, "TTA frame %lld at byte offset %lld: frame outside the buffer", (long long)f,
                     (long long)file_offsets[f]);
            return -1;
        }
        sbtta::Frame d;
        d.offset = offsets[f]; d.size = end - offsets[f]; d.sample = f * (int64_t)c.frame_length; d.last = f + 1 == n;
        d.pad = 0;
        const int code = sbtta::decode_frame(buf, d, c, s, crc.data(), pcm);
        if (code != sbtta::kOk) {
            snprintf(msg, msg_len, "TTA frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                     sbtta::error_text(code));
            return -1;
        }
    }
    return 0;
}

}  // extern "C"

#include <sys/mman.h>
#include <unistd.h>

extern "C" {

// emu_tta_decode with the data placed so that its last byte is the last readable one: the next page is inaccessible,
// so a read past the frames faults.
int emu_tta_decode_guarded(const uint8_t* data, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets,
                           int64_t n, const int32_t* config, int16_t* pcm, char* msg, int msg_len) {
    const int64_t page = sysconf(_SC_PAGESIZE);
    const int64_t body = (nbytes + page - 1) / page * page;
    uint8_t* base = (uint8_t*)mmap(nullptr, body + page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (base == MAP_FAILED) return -2;
    mprotect(base + body, page, PROT_NONE);
    uint8_t* buf = base + body - nbytes;
    memcpy(buf, data, (size_t)nbytes);
    const int r = emu_tta_decode(buf, nbytes, offsets, file_offsets, n, config, pcm, msg, msg_len);
    munmap(base, body + page);
    return r;
}

}  // extern "C"
