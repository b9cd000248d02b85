// Resident streams: upload, running sums (the integral image OpenCV rebuilds on
// every matchTemplate call, reference wav.py:185), and the per-stream block
// spectra that every query against the stream shares.
#include "sb_internal.h"

using namespace sb;

namespace {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;   // 4096 samples per CTA

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Phase A: per-tile totals of x and x^2 in fp64 (exact integers for u8 input).
template <typename T>
__global__ void __launch_bounds__(SCAN_THREADS)
k_tile_totals(const T* __restrict__ x, int64_t n, double* __restrict__ tsum, double* __restrict__ tsq) {
    __shared__ double s_a[SCAN_THREADS / 32], s_b[SCAN_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
    double a = 0.0, b = 0.0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        int64_t j = base + (int64_t)i * SCAN_THREADS + threadIdx.x;   // coalesced
        if (j < n) { double v = (double)x[j]; a += v; b += v * v; }
    }
    a = warp_sum(a); b = warp_sum(b);
    if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = a; s_b[threadIdx.x >> 5] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ta = 0.0, tb = 0.0;
        for (int w = 0; w < SCAN_THREADS / 32; ++w) { ta += s_a[w]; tb += s_b[w]; }
        tsum[blockIdx.x] = ta; tsq[blockIdx.x] = tb;
    }
}

// Phase B: exclusive scan of the tile totals.  One CTA walks them in slabs of 1024 x TOT_ITEMS (a 90-minute
// stream has 15 880 tiles: two slabs).  A slab goes to shared memory with coalesced loads, every thread scans
// TOT_ITEMS consecutive totals there, the threads' totals are scanned across the CTA, and the slab goes back.
constexpr int TOT_ITEMS = 8;
constexpr int TOT_SLAB = 1024 * TOT_ITEMS;
__global__ void __launch_bounds__(1024)
k_scan_tile_totals(double* __restrict__ tsum, double* __restrict__ tsq, int64_t ntiles) {
    extern __shared__ __align__(16) unsigned char tot_smem[];
    double* s_va = reinterpret_cast<double*>(tot_smem);                   // [TOT_SLAB + TOT_SLAB / TOT_ITEMS] padded
    double* s_vb = s_va + TOT_SLAB + TOT_SLAB / TOT_ITEMS;
    __shared__ double s_a[32], s_b[32];
    __shared__ double carry_a, carry_b;
    if (threadIdx.x == 0) { carry_a = 0.0; carry_b = 0.0; }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto slot = [](int e) { return e + e / TOT_ITEMS; };                  // one padding slot per thread's run: conflict-free
    for (int64_t base = 0; base < ntiles; base += TOT_SLAB) {
#pragma unroll
        for (int i = 0; i < TOT_ITEMS; ++i) {
            const int e = i * 1024 + threadIdx.x;
            const int64_t j = base + e;
            s_va[slot(e)] = j < ntiles ? tsum[j] : 0.0;
            s_vb[slot(e)] = j < ntiles ? tsq[j] : 0.0;
        }
        __syncthreads();
        double va[TOT_ITEMS], vb[TOT_ITEMS];
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int i = 0; i < TOT_ITEMS; ++i) {
            va[i] = s_va[slot(threadIdx.x * TOT_ITEMS + i)]; vb[i] = s_vb[slot(threadIdx.x * TOT_ITEMS + i)];
            a += va[i]; b += vb[i];
        }
        double ia = a, ib = b;                          // inclusive warp scan of the threads' totals
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            double ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
            if (lane >= o) { ia += ta; ib += tb; }
        }
        if (lane == 31) { s_a[warp] = ia; s_b[warp] = ib; }
        __syncthreads();
        if (warp == 0) {
            double wa = s_a[lane], wb = s_b[lane];
            double xa = wa, xb = wb;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                double ta = __shfl_up_sync(0xffffffffu, xa, o), tb = __shfl_up_sync(0xffffffffu, xb, o);
                if (lane >= o) { xa += ta; xb += tb; }
            }
            s_a[lane] = xa - wa; s_b[lane] = xb - wb;   // exclusive warp offsets
        }
        __syncthreads();
        double ea = carry_a + s_a[warp] + (ia - a), eb = carry_b + s_b[warp] + (ib - b);
#pragma unroll
        for (int i = 0; i < TOT_ITEMS; ++i) {
            s_va[slot(threadIdx.x * TOT_ITEMS + i)] = ea; s_vb[slot(threadIdx.x * TOT_ITEMS + i)] = eb;
            ea += va[i]; eb += vb[i];
        }
        __syncthreads();
        if (threadIdx.x == 1023) { carry_a = ea; carry_b = eb; }
#pragma unroll
        for (int i = 0; i < TOT_ITEMS; ++i) {
            const int e = i * 1024 + threadIdx.x;
            const int64_t j = base + e;
            if (j < ntiles) { tsum[j] = s_va[slot(e)]; tsq[j] = s_vb[slot(e)]; }
        }
        __syncthreads();
    }
}

// Phase C: in-tile inclusive scan + tile offset -> pfx[i+1] = (sum, sum of squares).
// Thread t scans SCAN_ITEMS consecutive samples; the results go through shared memory so that the
// 16-byte stores to HBM are coalesced (a blocked arrangement would scatter them 256 bytes apart).
template <typename T>
__global__ void __launch_bounds__(SCAN_THREADS)
k_tile_scan(const T* __restrict__ x, int64_t n, const double* __restrict__ osum, const double* __restrict__ osq,
            double2* __restrict__ pfx) {
    __shared__ double s_a[SCAN_THREADS / 32], s_b[SCAN_THREADS / 32];
    extern __shared__ __align__(16) unsigned char scan_smem[];
    double2* s_out = reinterpret_cast<double2*>(scan_smem);             // [SCAN_TILE + SCAN_TILE/16] padded
    const int64_t tile0 = (int64_t)blockIdx.x * SCAN_TILE;
    const int64_t base = tile0 + (int64_t)threadIdx.x * SCAN_ITEMS;
    double va[SCAN_ITEMS], vb[SCAN_ITEMS];
    double a = 0.0, b = 0.0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        int64_t j = base + i;
        double v = j < n ? (double)x[j] : 0.0;
        a += v; b += v * v;
        va[i] = a; vb[i] = b;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        double ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
        if (lane >= o) { ia += ta; ib += tb; }
    }
    if (lane == 31) { s_a[warp] = ia; s_b[warp] = ib; }
    __syncthreads();
    double wa = 0.0, wb = 0.0;
    for (int w = 0; w < warp; ++w) { wa += s_a[w]; wb += s_b[w]; }
    const double offa = osum[blockIdx.x] + wa + (ia - a);
    const double offb = osq[blockIdx.x] + wb + (ib - b);
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        const int e = threadIdx.x * SCAN_ITEMS + i;
        s_out[e + (e >> 4)] = make_double2(offa + va[i], offb + vb[i]);   // +1 slot per 16: conflict-free
    }
    __syncthreads();
#pragma unroll 4
    for (int e = threadIdx.x; e < SCAN_TILE; e += SCAN_THREADS) {
        const int64_t j = tile0 + e;
        if (j < n) pfx[j + 1] = s_out[e + (e >> 4)];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) pfx[0] = make_double2(0.0, 0.0);
}

// ---- uint8 streams: the same three phases on exact integers, written for HBM bandwidth -------------------
// The running sums cost 16 bytes per sample to write against 1 byte to read, so the scan is a store stream:
// phase C below gives every store instruction of a warp 512 contiguous bytes (lane l owns sample 32*it + l,
// the scan across the lanes is five shuffle steps on 32-bit integers -- sums inside a 4096-sample tile fit:
// 4096 * 255^2 < 2^31), with no trip through shared memory and no barrier between loads and stores, so the
// 8 warps of a CTA stream independently.  Phase A reads 16 bytes per lane and sums with dp4a.
// Tile offsets without a serial pass: phase A also adds every tile's totals into the accumulator of its GROUP of
// 128 tiles (exact 64-bit integers); a tile of phase C then sums the accumulators of the groups in front of its
// own (one warp, a few loads per lane) and the totals of the tiles in front of it inside its group (another warp).
constexpr int SCAN_GROUP = 128;

__device__ __forceinline__ uint4 mask_tail16(uint4 v, int keep) {         // zero the bytes from `keep` on (keep < 16)
    unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kb = keep - 4 * k;
        w[k] = kb >= 4 ? w[k] : (kb <= 0 ? 0u : (w[k] & (0xffffffffu >> (8 * (4 - kb)))));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void sums16(uint4 v, unsigned& a, unsigned& b) {
    a = __dp4a(v.x, 0x01010101u, __dp4a(v.y, 0x01010101u, __dp4a(v.z, 0x01010101u, __dp4a(v.w, 0x01010101u, 0u))));
    b = __dp4a(v.x, v.x, __dp4a(v.y, v.y, __dp4a(v.z, v.z, __dp4a(v.w, v.w, 0u))));
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_tile_totals_u8(const uint8_t* __restrict__ x, int64_t n, uint2* __restrict__ tot, unsigned long long* __restrict__ grp) {
    __shared__ unsigned s_a[SCAN_THREADS / 32], s_b[SCAN_THREADS / 32];
    const int64_t j = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * 16;     // stream allocations carry 16 bytes of slack
    unsigned a = 0, b = 0;
    if (j < n) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(x + j));
        if (j + 16 > n) v = mask_tail16(v, (int)(n - j));
        sums16(v, a, b);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
    if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = a; s_b[threadIdx.x >> 5] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned ta = 0, tb = 0;
        for (int w = 0; w < SCAN_THREADS / 32; ++w) { ta += s_a[w]; tb += s_b[w]; }
        tot[blockIdx.x] = make_uint2(ta, tb);
        atomicAdd(grp + 2 * (blockIdx.x / SCAN_GROUP), (unsigned long long)ta);
        atomicAdd(grp + 2 * (blockIdx.x / SCAN_GROUP) + 1, (unsigned long long)tb);
    }
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_tile_scan_u8(const uint8_t* __restrict__ x, int64_t n, const uint2* __restrict__ tot, const unsigned long long* __restrict__ grp,
               double2* __restrict__ pfx) {
    constexpr int NW = SCAN_THREADS / 32, PER_WARP = SCAN_TILE / NW;        // 512 samples per warp
    __shared__ unsigned s_a[NW], s_b[NW];
    __shared__ unsigned long long s_base[4];                                // group part and in-group part of (sum, sum of squares)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile = blockIdx.x, g = tile / SCAN_GROUP;
    const int64_t w0 = (int64_t)tile * SCAN_TILE + (int64_t)warp * PER_WARP;
    if (warp == NW - 1) {                              // groups in front of this tile's group
        unsigned long long a = 0, b = 0;
        for (int i = lane; i < g; i += 32) { a += __ldg(grp + 2 * i); b += __ldg(grp + 2 * i + 1); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
        if (lane == 0) { s_base[0] = a; s_base[1] = b; }
    } else if (warp == NW - 2) {                       // tiles of the same group in front of this tile
        unsigned long long a = 0, b = 0;
        for (int i = g * SCAN_GROUP + lane; i < tile; i += 32) { const uint2 t = __ldg(tot + i); a += t.x; b += t.y; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
        if (lane == 0) { s_base[2] = a; s_base[3] = b; }
    }
    {   // totals of the warps in front of this one inside the tile
        unsigned a = 0, b = 0;
        const int64_t j = w0 + lane * 16;
        if (j < n) {
            uint4 v = __ldg(reinterpret_cast<const uint4*>(x + j));
            if (j + 16 > n) v = mask_tail16(v, (int)(n - j));
            sums16(v, a, b);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
        if (lane == 0) { s_a[warp] = a; s_b[warp] = b; }
    }
    __syncthreads();
    unsigned cs = 0, cq = 0;                           // integer carry inside the tile (exact)
    for (int w = 0; w < warp; ++w) { cs += s_a[w]; cq += s_b[w]; }
    const double bs = (double)(s_base[0] + s_base[2]), bq = (double)(s_base[1] + s_base[3]);     // exact: < 2^53
    if (blockIdx.x == 0 && threadIdx.x == 0) pfx[0] = make_double2(0.0, 0.0);
#pragma unroll 4
    for (int it = 0; it < PER_WARP / 32; ++it) {
        const int64_t j = w0 + it * 32 + lane;
        if (w0 + it * 32 >= n) break;                  // warp-uniform
        const unsigned v = j < n ? (unsigned)__ldg(x + j) : 0u;
        unsigned s = v, q = v * v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned ts = __shfl_up_sync(0xffffffffu, s, o), tq = __shfl_up_sync(0xffffffffu, q, o);
            if (lane >= o) { s += ts; q += tq; }
        }
        if (j < n) pfx[j + 1] = make_double2(bs + (double)(cs + s), bq + (double)(cq + q));
        cs += __shfl_sync(0xffffffffu, s, 31);
        cq += __shfl_sync(0xffffffffu, q, 31);
    }
}

constexpr size_t kTotSmem = 2 * sizeof(double) * (TOT_SLAB + TOT_SLAB / TOT_ITEMS);
int ensure_tot_smem() {
    static bool attr_set = false;
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_scan_tile_totals, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTotSmem));
        attr_set = true;
    }
    return SB_OK;
}

int build_prefix_u8(sb_stream* s) {
    Ctx& c = ctx();
    const int64_t n = s->n;
    const int64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    const int64_t ngroups = (ntiles + SCAN_GROUP - 1) / SCAN_GROUP;
    unsigned char* d_t = nullptr;
    const size_t grp_bytes = sizeof(unsigned long long) * 2 * ngroups;
    SB_TRY(pool_alloc((void**)&d_t, grp_bytes + sizeof(uint2) * ntiles));
    unsigned long long* grp = reinterpret_cast<unsigned long long*>(d_t);
    uint2* tot = reinterpret_cast<uint2*>(d_t + grp_bytes);
    const uint8_t* x = static_cast<const uint8_t*>(s->d_raw);
    SB_CUDA(cudaMemsetAsync(grp, 0, grp_bytes, c.stream));
    {
        ProfScope ps("scan_tile_totals");
        k_tile_totals_u8<<<(unsigned)ntiles, SCAN_THREADS, 0, c.stream>>>(x, n, tot, grp);
    }
    {
        ProfScope ps("scan_tiles");
        k_tile_scan_u8<<<(unsigned)ntiles, SCAN_THREADS, 0, c.stream>>>(x, n, tot, grp, s->d_pfx);
    }
    SB_CUDA(cudaGetLastError());
    pool_free(d_t);            // reused only by later work on the same stream
    return SB_OK;
}

template <typename T>
int build_prefix(sb_stream* s) {
    Ctx& c = ctx();
    const int64_t n = s->n;
    const int64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    double* d_t = nullptr;
    SB_TRY(pool_alloc((void**)&d_t, sizeof(double) * 2 * ntiles));
    double* tsum = d_t; double* tsq = d_t + ntiles;
    const T* x = static_cast<const T*>(s->d_raw);
    {
        ProfScope ps("scan_tile_totals");
        k_tile_totals<T><<<(unsigned)ntiles, SCAN_THREADS, 0, c.stream>>>(x, n, tsum, tsq);
    }
    SB_TRY(ensure_tot_smem());
    {
        ProfScope ps("scan_tile_offsets");
        k_scan_tile_totals<<<1, 1024, kTotSmem, c.stream>>>(tsum, tsq, ntiles);
    }
    {
        ProfScope ps("scan_tiles");
        const size_t smem = sizeof(double2) * (SCAN_TILE + SCAN_TILE / 16);
        static bool attr_set = false;
        if (!attr_set) {
            SB_CUDA(cudaFuncSetAttribute(k_tile_scan<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr_set = true;
        }
        k_tile_scan<T><<<(unsigned)ntiles, SCAN_THREADS, smem, c.stream>>>(x, n, tsum, tsq, s->d_pfx);
    }
    SB_CUDA(cudaGetLastError());
    pool_free(d_t);            // reused only by later work on the same stream
    return SB_OK;
}

int stream_finish(sb_stream* s) {
    SB_TRY(pool_alloc((void**)&s->d_pfx, sizeof(double2) * (s->n + 1)));
    if (s->dtype == SB_U8) return build_prefix_u8(s);
    return build_prefix<float>(s);
}

int stream_alloc(int64_t n, int dtype, sb_stream** out, const char* who) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "%s: library not initialised (call sb_init)", who);
    if (!out) SB_FAIL(SB_EINVAL, "%s: NULL output handle", who);
    if (n < 1) SB_FAIL(SB_EINVAL, "%s: stream length %lld < 1", who, (long long)n);
    if (dtype != SB_U8 && dtype != SB_F32) SB_FAIL(SB_EINVAL, "%s: unknown dtype %d", who, dtype);
    sb_stream* s = new (std::nothrow) sb_stream();
    if (!s) SB_FAIL(SB_ENOMEM, "%s: out of host memory", who);
    s->n = n; s->dtype = dtype;
    const size_t esz = dtype == SB_U8 ? 1 : 4;
    if (pool_alloc(&s->d_raw, esz * n + 16) != SB_OK) { delete s; return SB_ENOMEM; }
    *out = s;
    return SB_OK;
}

}  // namespace

namespace sb {

int stream_finish_public(sb_stream* s) { return stream_finish(s); }

// Block spectra in the quad layout of the packed kernels (sb_fused2.cu): B = 16384, hop B.
// Rows are built on demand: [k_lo, k_hi) is what the batch at hand reads.  A rank of an event-sharded job
// touches only the part of the destination stream its own events' search windows cover, so it transforms
// that part only (the replicated stream preparation is the Amdahl term of strong scaling, SURVEY.md 8e).
int ensure_spectra_quad(sb_stream* s, int64_t k_lo, int64_t k_hi) {
    const int64_t nblk = (s->n + kLagBlock - 1) / kLagBlock;
    if (k_lo < 0) k_lo = 0;
    if (k_hi > nblk) k_hi = nblk;
    if (k_lo >= k_hi) return SB_OK;
    if (!s->d_specq) {
        SB_TRY(pool_alloc((void**)&s->d_specq, sizeof(float2) * (size_t)nblk * kQuadRowF2));
        s->nblkq = nblk; s->specq_lo = s->specq_hi = k_lo;
    }
    auto build = [&](int64_t a, int64_t b) -> int {
        if (a >= b) return SB_OK;
        ProfScope ps("block_spectra");
        return launch_block_spectra_quad(s, a, b - a, s->d_specq + a * (int64_t)kQuadRowF2);
    };
    if (s->specq_lo == s->specq_hi) {                // nothing built yet
        SB_TRY(build(k_lo, k_hi));
        s->specq_lo = k_lo; s->specq_hi = k_hi;
        return SB_OK;
    }
    // keep the built range contiguous: extend it on either side (a gap between an old and a new range is filled)
    if (k_lo < s->specq_lo) { SB_TRY(build(k_lo, s->specq_lo)); s->specq_lo = k_lo; }
    if (k_hi > s->specq_hi) { SB_TRY(build(s->specq_hi, k_hi)); s->specq_hi = k_hi; }
    return SB_OK;
}

// Build (or fetch) the block spectra of `s` in the classic row layout of engine 1's kernels (also behind engines
// 2 / 4 / 5 for the queries routed through the blocked multiply): row k = FFT_2B of samples [kB, kB + 2B).
int ensure_spectra(sb_stream* s) {
    if (s->d_spec) return SB_OK;
    const int64_t nblk = (s->n + kLagBlock - 1) / kLagBlock;
    float2* spec = nullptr;
    SB_TRY(pool_alloc((void**)&spec, sizeof(float2) * (size_t)nblk * (kLagBlock + 1)));
    int rc;
    {
        ProfScope ps("block_spectra");
        rc = launch_block_spectra(s, 0, nblk, spec);
    }
    if (rc != SB_OK) { pool_free(spec); return rc; }
    s->d_spec = spec; s->nblk = nblk;
    return SB_OK;
}

}  // namespace sb

extern "C" {

int sb_stream_create(const void* host_samples, int64_t n, int dtype, sb_stream** out) {
    if (!host_samples) SB_FAIL(SB_EINVAL, "sb_stream_create: NULL samples");
    SB_TRY(stream_alloc(n, dtype, out, "sb_stream_create"));
    sb_stream* s = *out;
    Ctx& c = ctx();
    const size_t esz = dtype == SB_U8 ? 1 : 4;
    cudaError_t e = cudaMemcpyAsync(s->d_raw, host_samples, esz * n, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { sb_stream_destroy(s); *out = nullptr; SB_FAIL(SB_ECUDA, "sb_stream_create: H2D copy: %s", cudaGetErrorString(e)); }
    int rc = stream_finish(s);
    if (rc != SB_OK) { sb_stream_destroy(s); *out = nullptr; }
    return rc;
}

int sb_stream_create_device(const void* dev_samples, int64_t n, int dtype, sb_stream** out) {
    if (!dev_samples) SB_FAIL(SB_EINVAL, "sb_stream_create_device: NULL samples");
    SB_TRY(stream_alloc(n, dtype, out, "sb_stream_create_device"));
    sb_stream* s = *out;
    Ctx& c = ctx();
    const size_t esz = dtype == SB_U8 ? 1 : 4;
    // enqueue only: the caller may have ordered the library stream behind a broadcast that is still in flight
    cudaError_t e = cudaMemcpyAsync(s->d_raw, dev_samples, esz * n, cudaMemcpyDeviceToDevice, c.stream);
    if (e != cudaSuccess) { sb_stream_destroy(s); *out = nullptr; SB_FAIL(SB_ECUDA, "sb_stream_create_device: D2D copy: %s", cudaGetErrorString(e)); }
    int rc = stream_finish(s);
    if (rc != SB_OK) { sb_stream_destroy(s); *out = nullptr; }
    return rc;
}

int sb_stream_destroy(sb_stream* s) {
    if (!s) return SB_OK;
    Ctx& c = ctx();
    (void)c;
    pool_free(s->d_raw); pool_free(s->d_pfx); pool_free(s->d_spec); pool_free(s->d_specq); pool_free(s->d_loadhist);
    delete s;
    return SB_OK;
}

const void* sb_stream_device_ptr(const sb_stream* s) { return s ? s->d_raw : nullptr; }
int64_t sb_stream_length(const sb_stream* s) { return s ? s->n : -1; }
int sb_stream_dtype(const sb_stream* s) { return s ? s->dtype : -1; }

int sb_stream_read(const sb_stream* s, int64_t off, int64_t n, void* host_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_stream_read: library not initialised");
    if (!s || !host_out) SB_FAIL(SB_EINVAL, "sb_stream_read: NULL argument");
    if (off < 0 || n < 0 || off + n > s->n) SB_FAIL(SB_EINVAL, "sb_stream_read: range [%lld,+%lld) outside stream of %lld",
                                                     (long long)off, (long long)n, (long long)s->n);
    const size_t esz = s->dtype == SB_U8 ? 1 : 4;
    SB_CUDA(cudaMemcpyAsync(host_out, static_cast<const char*>(s->d_raw) + esz * off, esz * n,
                            cudaMemcpyDeviceToHost, c.stream));
    SB_CUDA(cudaStreamSynchronize(c.stream));
    return SB_OK;
}

}  // extern "C"
