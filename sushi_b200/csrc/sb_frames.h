// How a decoder words the refusal of one frame (or block), written once for the library and for the CPU builds of the
// tests: plain C++, no CUDA.  The host halves of sb_alac.cuh, sb_wavpack.cuh and sb_tta.cuh build their frame tables
// with it, and the entry points report the first failing status with it.
#pragma once
#include <stdint.h>
#include <stdio.h>

namespace sbframes {

// "<what> <f> at byte offset <where>: <text>" into msg (`what`: "ALAC frame", "WavPack block", ...); returns false
inline bool refuse(char* msg, size_t msg_len, const char* what, int64_t f, int64_t where, const char* text) {
    snprintf(msg, msg_len, "%s %lld at byte offset %lld: %s", what, (long long)f, (long long)where, text);
    return false;
}

// The statuses a decode kernel left, one per frame: true when all are 0, else false with the first failing frame's
// message.  Frame f is at file offset where[f * stride]; text(code) is the codec's error_text.
template <class Text>
bool first_failure(const int32_t* status, int64_t n, const char* what, const int64_t* where, int64_t stride, Text text,
                   char* msg, size_t msg_len) {
    for (int64_t f = 0; f < n; ++f)
        if (status[f] != 0) return refuse(msg, msg_len, what, f, where[f * stride], text(status[f]));
    return true;
}

}  // namespace sbframes
