// What the demultiplexers fed a file in chunks (sb_ts.cu, sb_ps.cu, sb_ogg.cu) share, written once: the device scans
// of per-CTA totals, the chain of variable-length packets by pointer jumping, the device buffers that grow with the
// stream, and the host-side life of a handle (open, feed checks, waiting
// for the last chunk, the refusal of the first failure, destroy).  Host and device code, not part of the ABI; each
// translation unit keeps its own copy.
#pragma once
#include "sb_decode.h"
#include <algorithm>
#include <vector>

namespace {

using namespace sb;

constexpr int kThreads = 256;
constexpr unsigned long long kNoError = ~0ull;

// first failure wins: the byte offset in the high bits, the code in the low 8
__device__ __forceinline__ void fail_at(unsigned long long* err, int64_t file_off, int code) {
    atomicMin(err, ((unsigned long long)file_off << 8) | (unsigned)code);
}

// exclusive prefix of v over the CTA, *total the CTA's sum (every thread of the CTA calls it)
__device__ long long block_exclusive(long long v, long long* total) {
    __shared__ long long warp_sums[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    long long x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[w] = x;
    __syncthreads();
    if (w == 0) {
        long long s = lane < nw ? warp_sums[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xFFFFFFFFu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < nw) warp_sums[lane] = s;
    }
    __syncthreads();
    const long long before = (w > 0 ? warp_sums[w - 1] : 0) + x - v;
    *total = warp_sums[nw - 1];
    __syncthreads();                                  // warp_sums is reused by the next call
    return before;
}

// One CTA: each of the N values interleaved in cta[N * t + k] (t < n_cta) replaced by the exclusive scan of its
// column on top of base[k] (no base: from 0); the running totals go to total[k], which may be base.
template <int N>
__global__ void __launch_bounds__(1024)
k_scan_totals(long long* __restrict__ cta, int64_t n_cta, const long long* base, long long* total) {
    long long run[N];
#pragma unroll
    for (int k = 0; k < N; ++k) run[k] = base ? base[k] : 0;
    for (int64_t t0 = 0; t0 < n_cta; t0 += blockDim.x) {
        const int64_t t = t0 + threadIdx.x;
#pragma unroll
        for (int k = 0; k < N; ++k) {
            long long sum;
            const long long ex = block_exclusive(t < n_cta ? cta[N * t + k] : 0, &sum);
            if (t < n_cta) cta[N * t + k] = run[k] + ex;
            run[k] += sum;
        }
    }
    __syncthreads();                                  // every thread has read base before it is overwritten
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) total[k] = run[k];
    }
}

// ---- the packet chain of a chunk (sb_ps.cu, sb_ogg.cu) ----------------------------------------------------------
// Candidates are the positions pos[0, m) (sorted) where a packet or page may start; each links to the candidate its
// length reaches, or to the sink m where the chain ends.  The chain from candidate 0 is marked by pointer jumping.

// the candidate at position p, or -1
__device__ __forceinline__ int64_t find_cand(const int64_t* __restrict__ pos, int64_t m, int64_t p) {
    int64_t lo = 0, hi = m;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (pos[mid] < p) lo = mid + 1; else hi = mid;
    }
    return lo < m && pos[lo] == p ? lo : -1;
}

// one round: every marked candidate marks the one `span` links on; the links double.  A mark set during the round
// is on the chain too, so reading it early only marks more of the chain sooner.
__global__ void __launch_bounds__(kThreads)
k_chain_jump(const int32_t* __restrict__ jin, int32_t* __restrict__ jout, uint8_t* on, int64_t m) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v > m) return;
    const int32_t j = jin[v];
    if (on[v]) on[j] = 1;
    jout[v] = jin[j];
}

// the rounds of k_chain_jump until 2^r covers the longest chain, m links; jump[0] holds the links (jump[m] == m) and
// on[] the chain's start, and each round is counted as `prof_name`
inline cudaError_t mark_chain(int32_t* const jump[2], uint8_t* on, int64_t m, const char* prof_name, cudaStream_t st) {
    const unsigned j_cta = (unsigned)((m + 1 + kThreads - 1) / kThreads);
    cudaError_t e = cudaSuccess;
    for (int r = 0; e == cudaSuccess && ((int64_t)1 << r) < m; ++r) {
        ProfScope ps(prof_name);
        k_chain_jump<<<j_cta, kThreads, 0, st>>>(jump[r & 1], jump[(r & 1) ^ 1], on, m);
        e = cudaGetLastError();
    }
    return e;
}

// exclusive scan of n int64 values in place: tile sums, one CTA over the tiles, then each tile
__global__ void __launch_bounds__(kThreads)
k_scan_tiles(const int64_t* __restrict__ v, int64_t n, long long* __restrict__ tiles) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    long long total;
    block_exclusive(i < n ? v[i] : 0, &total);
    if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads)
k_scan_apply(int64_t* __restrict__ v, int64_t n, const long long* __restrict__ tiles) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    long long total;
    const long long ex = block_exclusive(i < n ? v[i] : 0, &total);
    if (i < n) v[i] = tiles[blockIdx.x] + ex;
}

// exclusive scan of d_v[0..n) in place on the library stream, its three launches counted as `prof_name`; the sum comes
// back in *total
int scan_i64(int64_t* d_v, int64_t n, int64_t* total, const char* prof_name, const char* who) {
    Ctx& c = ctx();
    const int64_t tiles = (n + kThreads - 1) / kThreads;
    long long* d_tiles = nullptr;
    if (pool_alloc((void**)&d_tiles, sizeof(long long) * (size_t)(tiles + 1)) != SB_OK) SB_FAIL(SB_ENOMEM, "%s: out of device memory", who);
    cudaError_t e = cudaSuccess;
    {
        ProfScope ps(prof_name, 3);
        k_scan_tiles<<<(unsigned)tiles, kThreads, 0, c.stream>>>(d_v, n, d_tiles);
        k_scan_totals<1><<<1, 1024, 0, c.stream>>>(d_tiles, tiles, nullptr, d_tiles + tiles);
        k_scan_apply<<<(unsigned)tiles, kThreads, 0, c.stream>>>(d_v, n, d_tiles);
        e = cudaGetLastError();
    }
    long long t = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&t, d_tiles + tiles, sizeof(t), cudaMemcpyDeviceToHost, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    pool_free(d_tiles);
    SB_TRY(cuda_result(e, who));
    *total = t;
    return SB_OK;
}

// *p: room for `need` T (and 16 bytes more), its first `used` kept
template <class T>
int grow(T** p, int64_t* cap, int64_t used, int64_t need, cudaStream_t st) {
    if (need <= *cap) return SB_OK;
    const int64_t n = std::max(need, *cap + *cap / 2);
    T* q = nullptr;
    if (pool_alloc((void**)&q, sizeof(T) * (size_t)n + 16) != SB_OK) return SB_ENOMEM;
    if (used > 0 && cudaMemcpyAsync(q, *p, sizeof(T) * (size_t)used, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
        pool_free(q);
        return SB_ECUDA;
    }
    pool_free(*p);
    *p = q;
    *cap = n;
    return SB_OK;
}

// The file offset of the record holding stream byte b, in a table sorted by es_off (where each record's bytes start in
// the stream); -1 before the first
template <class Rec>
int64_t file_offset_of(const std::vector<Rec>& tab, int64_t b) {
    const int64_t k = std::upper_bound(tab.begin(), tab.end(), b, [](int64_t v, const Rec& r) { return v < r.es_off; })
                      - tab.begin() - 1;
    return k >= 0 ? tab[(size_t)k].file_off : -1;
}

// The part of a demultiplexer's handle that is not about its format.  `Run` is what the kernels of a chunk leave for
// placing the next one; its pinned copy *h_run is current once `done` has fired (settle).
template <class Run>
struct ChunkedDemux {
    int64_t next_offset = 0;                            // the file offset the next chunk must start at
    unsigned long long* d_err = nullptr;                // the first failure (fail_at), kNoError while there is none
    Run* h_run = nullptr;
    cudaEvent_t done = nullptr;                         // recorded after the copy to *h_run
    bool pending = false, finished = false;

    ChunkedDemux() = default;
    ChunkedDemux(const ChunkedDemux&) = delete;
    ChunkedDemux& operator=(const ChunkedDemux&) = delete;
    ~ChunkedDemux() {
        pool_free(d_err);
        if (h_run) cudaFreeHost(h_run);
        if (done) cudaEventDestroy(done);
    }

    // *h_run zeroed, the event, no failure yet; the caller destroys the handle when this fails
    int open(const char* who) {
        cudaError_t e = cudaMallocHost((void**)&h_run, sizeof(Run));
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&done, cudaEventDisableTiming);
        if (e == cudaSuccess) *h_run = Run{};
        SB_TRY(cuda_result(e, who));
        if (pool_alloc((void**)&d_err, 16) != SB_OK) SB_FAIL(SB_ENOMEM, "%s: out of device memory", who);
        return cuda_result(cudaMemsetAsync(d_err, 0xFF, sizeof(unsigned long long), ctx().stream), who);
    }

    // after entry_check: chunks of whole `align`-byte packets (1: any size), in file order, before finish
    int feed_check(const char* who, int64_t nbytes, int64_t file_offset, int align) const {
        if (finished) SB_FAIL(SB_ESTATE, "%s: the stream is finished", who);
        if (nbytes < 0 || nbytes % align)
            SB_FAIL(SB_EINVAL, align > 1 ? "%s: %lld bytes is not a whole number of %d-byte packets" : "%s: %lld bytes",
                    who, (long long)nbytes, align);
        if (file_offset != next_offset)
            SB_FAIL(SB_EINVAL, "%s: chunk at byte offset %lld, expected %lld", who, (long long)file_offset,
                    (long long)next_offset);
        return SB_OK;
    }

    // after entry_check: a handle is finished once
    int finish_check(const char* who) {
        if (finished) SB_FAIL(SB_ESTATE, "%s: the stream is finished", who);
        finished = true;
        return SB_OK;
    }

    // wait for the kernels of the last chunk: *h_run is then current
    int settle(const char* who) {
        if (!pending) return SB_OK;
        SB_TRY(cuda_result(cudaEventSynchronize(done), who));
        pending = false;
        return SB_OK;
    }

    // SB_OK when the kernels recorded no failure, else the first one refused as "<noun> at byte offset <N>: <text>",
    // noun(code) and text(code) the format's words for it
    template <class Noun, class Text>
    int check_failure(const char* who, Noun noun, Text text) const {
        unsigned long long err = kNoError;
        SB_TRY(collect(cudaSuccess, &err, d_err, 1, who));
        if (err == kNoError) return SB_OK;
        const int k = (int)(err & 0xFF);
        SB_FAIL(SB_EINVAL, "%s at byte offset %lld: %s", noun(k), (long long)(err >> 8), text(k));
    }
};

// In sb_*_finish: the handle's chunk buffers (T::release_demux) go when the scope ends, on whichever line
template <class T>
struct ReleaseDemux {
    T* t;
    ~ReleaseDemux() { t->release_demux(); }
};

// sb_*_destroy: once the last chunk's kernels are done, everything the handle holds
template <class T>
int destroy_demux(T* t) {
    if (!t) return SB_OK;
    if (t->pending) cudaEventSynchronize(t->done);
    delete t;
    return SB_OK;
}

}  // namespace
