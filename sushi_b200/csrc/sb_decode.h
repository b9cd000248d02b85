// What every decoder entry point (sb_flac.cu, sb_alac.cu, sb_truehd.cu, sb_wavpack.cu, sb_tta.cu, sb_ts_finish) does
// around its kernels, written once: host code only, not part of the ABI.  An entry point reads top to bottom as
// arguments checked, table built (the codec's .cuh), input uploaded, kernel launched, statuses collected, first failure
// reported, PCM handed over; the blocks it allocated on the way are freed when it returns, on whichever line.
//
// Every decoder's input is followed by at least 13 zero bytes on the device (upload_padded): the sync kernels read whole
// 32-bit words, so they need zeros up to the next multiple of 4, and the ALAC and WavPack bit readers fetch 5 bytes at
// a time from a position inside the input.
#pragma once
#include "sb_internal.h"
#include <algorithm>
#include <vector>

namespace sb {

// "<who>: library not initialised" / "<who>: NULL argument", the way every entry point opens
inline int entry_check(const char* who, bool args_given) {
    if (!ctx().inited) SB_FAIL(SB_ESTATE, "%s: library not initialised (call sb_init)", who);
    if (!args_given) SB_FAIL(SB_EINVAL, "%s: NULL argument", who);
    return SB_OK;
}

inline int cuda_result(cudaError_t e, const char* who) {
    if (e != cudaSuccess) SB_FAIL(SB_ECUDA, "%s: %s", who, cudaGetErrorString(e));
    return SB_OK;
}

// The pool blocks a scope allocated: all freed when it ends, but for the one take() hands on (the PCM, to pcm_handle)
struct Blocks {
    std::vector<void*> held;
    Blocks() = default;
    Blocks(const Blocks&) = delete;
    Blocks& operator=(const Blocks&) = delete;
    ~Blocks() { for (void* p : held) pool_free(p); }
    // *p: room for `count` T and 16 bytes more.  On failure the message is pool_alloc's.
    template <class T> int alloc(T** p, size_t count) {
        void* q = nullptr;
        SB_TRY(pool_alloc(&q, sizeof(T) * count + 16));
        held.push_back(q);
        *p = static_cast<T*>(q);
        return SB_OK;
    }
    template <class T> T* take(T* p) {
        held.erase(std::remove(held.begin(), held.end(), static_cast<void*>(p)), held.end());
        return p;
    }
};

// *d: the nbytes bytes of `host` on the device, then zeros up to at least 13 bytes past them (16 from nbytes & ~3)
inline int upload_padded(Blocks& blocks, uint8_t** d, const void* host, int64_t nbytes, const char* who) {
    SB_TRY(blocks.alloc(d, (size_t)nbytes));
    cudaStream_t stream = ctx().stream;
    cudaError_t e = cudaMemsetAsync(*d + (nbytes & ~(int64_t)3), 0, 16, stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(*d, host, (size_t)nbytes, cudaMemcpyHostToDevice, stream);
    return cuda_result(e, who);
}

// After the launches whose error state is `e`: n elements of d_src back into host memory, and the stream drained
template <class T> int collect(cudaError_t e, T* host, const T* d_src, int64_t n, const char* who) {
    cudaStream_t stream = ctx().stream;
    if (e == cudaSuccess) e = cudaMemcpyAsync(host, d_src, sizeof(T) * (size_t)n, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    return cuda_result(e, who);
}

// Every position a sync kernel accepts.  launch(d_cand, d_count, cap) enqueues the kernel, which counts every candidate
// in *d_count and stores the first `cap`; when there were more, one more pass has room for all of them.
template <class Cand, class Launch>
int scan_candidates(int64_t cap, const char* prof_name, const char* who, Launch launch, std::vector<Cand>& cand) {
    Ctx& c = ctx();
    for (int pass = 0; pass < 2; ++pass) {
        Blocks blocks;
        Cand* d_cand = nullptr;
        unsigned long long* d_count = nullptr;
        unsigned long long count = 0;
        SB_TRY(blocks.alloc(&d_cand, (size_t)cap));
        SB_TRY(blocks.alloc(&d_count, 1));
        cudaError_t e = cudaMemsetAsync(d_count, 0, sizeof(count), c.stream);
        if (e == cudaSuccess) {
            ProfScope ps(prof_name);
            launch(d_cand, d_count, cap);
            e = cudaGetLastError();
        }
        SB_TRY(collect(e, &count, d_count, 1, who));
        if ((int64_t)count <= cap) {
            cand.resize(count);
            return collect(cudaSuccess, cand.data(), d_cand, (int64_t)count, who);
        }
        cap = (int64_t)count;                                              // rescan with room for every candidate
    }
    return SB_OK;
}

}  // namespace sb
