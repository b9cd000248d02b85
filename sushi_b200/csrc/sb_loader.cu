// Loader kernels: the arithmetic of WavStream.__init__ (reference wav.py:64-91,108-156).
//   K1  sb_load_pcm   int16/int24 decode, channel average, per-chunk nearest-neighbour resample
//                     (cv2.resize INTER_NEAREST index map), edge padding      wav.py:64-91,125-141
//   K2  sb_normalise  3 x median clip, rescale to [0,1], optional uint8 quantisation  wav.py:145-156
// sb_pcm_load runs K1 on a decoder's int16 PCM (an sb_pcm); sb_pcm_from_be makes one from big-endian PCM (k_pcm_be).
// Everything is float32 with explicitly rounded operations (no FMA contraction), in the order the
// reference applies them, so the result is bit-identical to the NumPy/OpenCV loader.
#include "sb_internal.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

using namespace sb;

namespace sb { int stream_finish_public(sb_stream* s); }

namespace {

struct ResampleGeom {
    int64_t frames;        // frames in the file
    int framerate;         // frames per chunk (READ_CHUNK_SIZE = 1 s, wav.py:105,126)
    int64_t nfull;         // number of full chunks
    int len_last;          // frames in the trailing partial chunk (0 if none)
    int out_full;          // output samples of a full chunk   (wav.py:127)
    int out_last;          // output samples of the partial chunk
    int resample;          // downsample_rate != 1 (wav.py:131)
    double ifx_full;       // 1 / (out_full / framerate)   -- OpenCV's inverse scale, fp64
    double ifx_last;
    int64_t padding;       // wav.py:120
    int64_t total;         // wav.py:119
    int64_t written;       // samples produced by the chunk loop (may run past total - padding: see sb_load_pcm)
};

// One frame -> the integer numerator of the reference's float32 sample: int16 values (int24: bytes 1,2,
// wav.py:71-74) summed over the channels.  The reference sums float32 values left to right (wav.py:88-89);
// every partial sum is an integer below 2^24, hence exact, so the float32 sum IS (float)acc.
__device__ __forceinline__ int decode_acc(const unsigned char* __restrict__ pcm, int64_t frame, int channels, int width) {
    const unsigned char* p = pcm + frame * (int64_t)channels * width;
    int acc = 0;
    if (width == 2) {
        const short* q = reinterpret_cast<const short*>(p);            // frames are 2-byte aligned
        for (int c = 0; c < channels; ++c) acc += (int)q[c];
    } else {
        for (int c = 0; c < channels; ++c) {
            const unsigned char* q = p + c * 3 + 1;
            acc += (int)(short)((unsigned short)q[0] | ((unsigned short)q[1] << 8));
        }
    }
    return acc;
}
__device__ __forceinline__ float acc_value(int acc, int channels) {
    return channels == 1 ? (float)acc : __fdiv_rn((float)acc, (float)channels);      // wav.py:90
}

// ---- medians without sorting ---------------------------------------------------------------------
// np.median over {x >= 0} and over {x <= 0} of the PADDED array (wav.py:145-146) needs two order statistics
// each.  Every sample is (float)acc / channels with an integer acc, |acc| <= 32768 * channels, so selection can
// run on integers: a coarse histogram (bins of 32 in sample value = 32 * channels in acc; 2048 bins) is
// accumulated by the decode kernel itself while it writes the samples, and ONE further pass over the float32
// data histograms acc inside the (at most four) coarse bins that hold the wanted ranks.  Two reads of the
// float32 stream in all -- that pass and the normalisation -- where a radix select on float keys took ten.
constexpr int kCoarseBins = 2048, kCoarseZero = 1024, kCoarseWidth = 32, kMaxChannels = 64;
__device__ __forceinline__ int coarse_bin(float v) {
    int b = (int)floorf(v * (1.0f / kCoarseWidth)) + kCoarseZero;       // exact: division by a power of two
    return b < 0 ? 0 : (b > kCoarseBins - 1 ? kCoarseBins - 1 : b);
}

// Work items: [0, n_chunk_items) = (chunk, slab of 1024 output samples); then the head and the tail padding in
// slabs of 1024.  A CTA takes items round robin; its coarse histogram lives in shared memory.
struct LoadItems { int per_full; int per_last; int64_t n_content; int64_t n_head; int64_t n_tail; };

__global__ void __launch_bounds__(256)
k_decode_resample_pad(const unsigned char* __restrict__ pcm, ResampleGeom g, LoadItems li, int channels, int width,
                      float* __restrict__ out, unsigned long long* __restrict__ hist) {
    __shared__ unsigned s_h[kCoarseBins + 1];                            // [kCoarseBins] counts exact zeros
    for (int i = threadIdx.x; i <= kCoarseBins; i += blockDim.x) s_h[i] = 0;
    __syncthreads();
    const int64_t n_items = li.n_content + li.n_head + li.n_tail;
    const int64_t tail0 = g.total - g.padding;
    auto count = [&](float v, int acc) { atomicAdd(&s_h[coarse_bin(v)], 1u); if (acc == 0) atomicAdd(&s_h[kCoarseBins], 1u); };
    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        if (item < li.n_content) {
            int64_t c; int slab, len, outn; double ifx;
            if (item < g.nfull * (int64_t)li.per_full) { c = item / li.per_full; slab = (int)(item - c * li.per_full); len = g.framerate; outn = g.out_full; ifx = g.ifx_full; }
            else { c = g.nfull; slab = (int)(item - g.nfull * (int64_t)li.per_full); len = g.len_last; outn = g.out_last; ifx = g.ifx_last; }
            const int64_t frame0 = c * (int64_t)g.framerate;
            const int64_t o0 = g.padding + c * (int64_t)g.out_full;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int x = slab * 1024 + r * 256 + threadIdx.x;
                if (x < outn && o0 + x < tail0) {                         // what lands in the tail padding is overwritten
                    int sx = x;
                    if (g.resample) { sx = (int)floor((double)x * ifx); if (sx > len - 1) sx = len - 1; }   // OpenCV resizeNN: cvFloor(x * ifx)
                    const int acc = decode_acc(pcm, frame0 + sx, channels, width);
                    const float v = acc_value(acc, channels);
                    out[o0 + x] = v;
                    count(v, acc);
                }
            }
        } else {
            // padding: head repeats the first content sample (wav.py:140), tail repeats data[-padding-1] (wav.py:141);
            // a gap between the last written sample and the tail (np.empty in the reference) reads as zero
            const bool head = item < li.n_content + li.n_head;
            const int64_t slab = head ? item - li.n_content : item - li.n_content - li.n_head;
            const int64_t base = head ? 0 : tail0, limit = head ? g.padding : g.total;
            // head: [0, padding); tail region also covers the gap [padding + written, tail0) first
            int acc = 0;
            if (head) { if (g.written > 0) acc = decode_acc(pcm, 0, channels, width); }
            else {
                const int64_t o = tail0 - 1 - g.padding;            // content index of data[-padding-1]
                if (o >= 0 && o < g.written) {
                    int64_t c; int x, len; double ifx;
                    if (g.out_full > 0 && o < g.nfull * (int64_t)g.out_full) { c = o / g.out_full; x = (int)(o - c * g.out_full); len = g.framerate; ifx = g.ifx_full; }
                    else { c = g.nfull; x = (int)(o - g.nfull * (int64_t)g.out_full); len = g.len_last; ifx = g.ifx_last; }
                    int sx = x;
                    if (g.resample) { sx = (int)floor((double)x * ifx); if (sx > len - 1) sx = len - 1; }
                    acc = decode_acc(pcm, c * (int64_t)g.framerate + sx, channels, width);
                }
            }
            const float v = acc_value(acc, channels);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int64_t i = base + slab * 1024 + r * 256 + threadIdx.x;
                if (i < limit) { out[i] = v; count(v, acc); }
            }
        }
    }
    // the gap between the written content and the tail padding (float rounding of the sample count, wav.py:113-116)
    const int64_t gap0 = g.padding + g.written, gap_n = tail0 - gap0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < gap_n; i += (int64_t)gridDim.x * blockDim.x) {
        out[gap0 + i] = 0.f; count(0.f, 0);
    }
    __syncthreads();
    for (int i = threadIdx.x; i <= kCoarseBins; i += blockDim.x)
        if (s_h[i]) atomicAdd(hist + i, (unsigned long long)s_h[i]);
}

// acc histograms inside up to four coarse bins: fine[t][acc - base[t]], base[t] = (bin[t] - kCoarseZero) * 32 * channels
struct FineTargets { int bin[4]; int base[4]; int n; int width; };     // width = 32 * channels
__global__ void __launch_bounds__(256)
k_select_fine(const float* __restrict__ x, int64_t n, int channels, FineTargets ft, unsigned* __restrict__ fine) {
    extern __shared__ unsigned s_f[];                                     // [ft.n][ft.width]
    for (int i = threadIdx.x; i < ft.n * ft.width; i += blockDim.x) s_f[i] = 0;
    __syncthreads();
    const float fc = (float)channels;
    auto one = [&](float v) {
        const int b = coarse_bin(v);
#pragma unroll
        for (int t = 0; t < 4; ++t)
            if (t < ft.n && b == ft.bin[t]) {
                const int off = __float2int_rn(v * fc) - ft.base[t];      // acc, exactly (|acc| < 2^22)
                if (off >= 0 && off < ft.width) atomicAdd(&s_f[t * ft.width + off], 1u);
                else atomicAdd(fine + 4 * ft.width, 1u);                  // cannot happen for sb_load_pcm data: flagged
            }
    };
    const int64_t n4 = n >> 2;                                            // streams are 256-byte aligned
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        one(v.x); one(v.y); one(v.z); one(v.w);
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 3)) one(x[(n4 << 2) + threadIdx.x]);
    __syncthreads();
    for (int i = threadIdx.x; i < ft.n * ft.width; i += blockDim.x)
        if (s_f[i]) atomicAdd(fine + i, s_f[i]);
}

__global__ void __launch_bounds__(256)
k_normalise(const float* __restrict__ x, int64_t n, float lo, float hi, float* __restrict__ out_f32,
            unsigned char* __restrict__ out_u8) {
    const float den = __fsub_rn(hi, lo);
    auto one = [&](float v) {
        v = fminf(fmaxf(v, lo), hi);                         // np.clip (wav.py:148)
        v = __fsub_rn(v, lo);                                // wav.py:150
        return __fdiv_rn(v, den);                            // wav.py:151 (float32 difference, float32 divide)
    };
    auto quant = [&](float v) {
        v = __fmul_rn(v, 255.0f);                            // wav.py:154
        v = __fadd_rn(v, 0.5f);                              // wav.py:155
        return (unsigned)(unsigned char)(int)v;              // astype('uint8'): truncation (wav.py:156)
    };
    // streams are 256-byte aligned: 16-byte loads, two of them in flight per thread, 8-byte / 16-byte stores
    const int64_t n8 = n >> 3;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + 2 * i), w = __ldg(reinterpret_cast<const float4*>(x) + 2 * i + 1);
        const float a = one(v.x), b = one(v.y), c = one(v.z), d = one(v.w), e = one(w.x), f = one(w.y), g = one(w.z), h = one(w.w);
        if (out_u8) {
            *reinterpret_cast<uint2*>(out_u8 + 8 * i) = make_uint2(quant(a) | (quant(b) << 8) | (quant(c) << 16) | (quant(d) << 24),
                                                                   quant(e) | (quant(f) << 8) | (quant(g) << 16) | (quant(h) << 24));
        } else {
            reinterpret_cast<float4*>(out_f32)[2 * i] = make_float4(a, b, c, d);
            reinterpret_cast<float4*>(out_f32)[2 * i + 1] = make_float4(e, f, g, h);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 7)) {
        const int64_t j = (n8 << 3) + threadIdx.x;
        const float v = one(x[j]);
        if (out_u8) out_u8[j] = (unsigned char)quant(v); else out_f32[j] = v;
    }
}

// Rank r (0-based, ascending) of subset 0 = {x >= 0} or subset 1 = {x <= 0}, located on the coarse histogram:
// `zero` = the value is exactly 0; else (bin, idx) = idx-th smallest non-zero member inside coarse bin `bin`.
struct RankWhere { bool zero; int bin; long long idx; };
RankWhere locate_rank(const unsigned long long* h, int subset, long long r) {
    const long long zeros = (long long)h[kCoarseBins];
    RankWhere w = {false, 0, 0};
    if (subset == 0) {                        // zeros first, then the positives ascending
        if (r < zeros) { w.zero = true; return w; }
        long long left = r - zeros;
        for (int b = kCoarseZero; b < kCoarseBins; ++b) {
            const long long cnt = (long long)h[b] - (b == kCoarseZero ? zeros : 0);
            if (left < cnt) { w.bin = b; w.idx = left; return w; }
            left -= cnt;
        }
    } else {                                  // the negatives ascending, then the zeros
        long long left = r;
        for (int b = 0; b < kCoarseZero; ++b) {
            if (left < (long long)h[b]) { w.bin = b; w.idx = left; return w; }
            left -= (long long)h[b];
        }
        w.zero = true;
    }
    return w;
}

// Both medians (NumPy: middle element, or the float32 mean of the two middle ones) from the coarse histogram
// the decode kernel left behind plus one pass over the data.
int medians_from_histograms(const sb_stream* raw, float* med_pos, float* med_neg) {
    Ctx& c = ctx();
    const int ch = raw->pcm_channels;
    unsigned long long h[kCoarseBins + 1];
    SB_CUDA(cudaMemcpyAsync(h, raw->d_loadhist, sizeof(h), cudaMemcpyDeviceToHost, c.stream));
    SB_CUDA(cudaStreamSynchronize(c.stream));
    const long long zeros = (long long)h[kCoarseBins];
    long long pos = 0, neg = 0;
    for (int b = 0; b < kCoarseZero; ++b) neg += (long long)h[b];
    for (int b = kCoarseZero; b < kCoarseBins; ++b) pos += (long long)h[b];
    const long long count[2] = {pos, neg + zeros};          // bin kCoarseZero holds the zeros: pos already includes them
    RankWhere want[2][2];
    int nwant[2];
    FineTargets ft; ft.n = 0; ft.width = kCoarseWidth * ch;
    for (int s = 0; s < 2; ++s) {
        nwant[s] = count[s] == 0 ? 0 : (count[s] % 2 == 0 ? 2 : 1);
        const long long k = (count[s] - 1) / 2;
        for (int e = 0; e < nwant[s]; ++e) {
            want[s][e] = locate_rank(h, s, k + e);
            if (!want[s][e].zero) {
                bool have = false;
                for (int t = 0; t < ft.n; ++t) have = have || ft.bin[t] == want[s][e].bin;
                if (!have) { ft.bin[ft.n] = want[s][e].bin; ft.base[ft.n] = (want[s][e].bin - kCoarseZero) * ft.width; ++ft.n; }
            }
        }
    }
    std::vector<unsigned> fine((size_t)4 * ft.width + 1, 0u);
    if (ft.n) {
        unsigned* d_fine = nullptr;
        SB_TRY(pool_alloc((void**)&d_fine, fine.size() * sizeof(unsigned)));
        SB_CUDA(cudaMemsetAsync(d_fine, 0, fine.size() * sizeof(unsigned), c.stream));
        {
            ProfScope ps("median_select_fine");
            k_select_fine<<<c.sm_count * 8, 256, (size_t)ft.n * ft.width * sizeof(unsigned), c.stream>>>(
                static_cast<const float*>(raw->d_raw), raw->n, ch, ft, d_fine);
        }
        cudaError_t e = cudaMemcpyAsync(fine.data(), d_fine, fine.size() * sizeof(unsigned), cudaMemcpyDeviceToHost, c.stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        pool_free(d_fine);
        if (e != cudaSuccess) SB_FAIL(SB_ECUDA, "sb_normalise: median selection: %s", cudaGetErrorString(e));
        if (fine[(size_t)4 * ft.width]) SB_FAIL(SB_EINVAL, "sb_normalise: samples are not int16 / channels values (not produced by sb_load_pcm?)");
    }
    float med[2] = {nanf(""), nanf("")};                     // np.median([]) is nan
    for (int s = 0; s < 2; ++s) {
        float v[2] = {0.f, 0.f};
        for (int e = 0; e < nwant[s]; ++e) {
            const RankWhere& w = want[s][e];
            if (w.zero) { v[e] = 0.f; continue; }
            int t = 0;
            while (ft.bin[t] != w.bin) ++t;
            long long left = w.idx;
            int acc = 0; bool found = false;
            for (int o = 0; o < ft.width && !found; ++o) {
                const int a = ft.base[t] + o;
                if (a == 0) continue;                        // zeros are counted apart
                const long long cnt = fine[(size_t)t * ft.width + o];
                if (left < cnt) { acc = a; found = true; } else left -= cnt;
            }
            if (!found) SB_FAIL(SB_ECUDA, "sb_normalise: internal: median rank not found in its histogram bin");
            v[e] = ch == 1 ? (float)acc : (float)acc / (float)ch;
        }
        if (nwant[s] == 1) med[s] = v[0];
        else if (nwant[s] == 2) med[s] = (v[0] + v[1]) * 0.5f;      // np.mean of two float32 values, float32 arithmetic
    }
    *med_pos = med[0]; *med_neg = med[1];
    return SB_OK;
}

int py2_round_pos(double x) { return (int)floor(x + 0.5); }     // round() of Python 2 for x >= 0 (wav.py:127)

// The geometry of one load: the chunk loop of the reference (wav.py:113-137) over `frames` frames, and the kernel's
// work items.  Checks the arguments; `who` prefixes the messages.
int plan_load(int64_t frames, int channels, int sample_width, int framerate, int sample_rate, int64_t padding,
              int64_t total_len, const char* who, ResampleGeom* gout, LoadItems* liout) {
    if (sample_width != 2 && sample_width != 3) SB_FAIL(SB_EINVAL, "Unsupported sample width: %d", sample_width);
    if (frames < 0 || channels < 1 || framerate < 1 || sample_rate < 1 || padding < 0 || total_len < 1)
        SB_FAIL(SB_EINVAL, "%s: bad geometry", who);
    ResampleGeom g;
    g.frames = frames; g.framerate = framerate;
    g.nfull = frames / framerate;
    g.len_last = (int)(frames - g.nfull * framerate);
    const double rate = (double)sample_rate / (double)framerate;          // wav.py:114
    g.resample = rate != 1.0;
    g.out_full = py2_round_pos((double)framerate * rate);
    g.out_last = py2_round_pos((double)g.len_last * rate);
    g.ifx_full = g.out_full > 0 ? 1.0 / ((double)g.out_full / (double)framerate) : 0.0;
    g.ifx_last = (g.out_last > 0 && g.len_last > 0) ? 1.0 / ((double)g.out_last / (double)g.len_last) : 0.0;
    g.padding = padding; g.total = total_len;
    g.written = g.nfull * (int64_t)g.out_full + g.out_last;
    // The reference reads whole seconds from the start of the data chunk (wav.py:125-137), so `frames` may hold more
    // than the total_len - 2 * padding samples the header accounts for (a chunk after the PCM) or fewer (a truncated
    // file).  Samples past the content region are overwritten by the tail padding there and are not written here;
    // samples past the end of the buffer make the reference's copy fail.
    if (g.written > total_len - padding)
        SB_FAIL(SB_EINVAL, "%s: %lld resampled samples run past a buffer of %lld with %lld padding",
                who, (long long)g.written, (long long)total_len, (long long)padding);
    if (channels > kMaxChannels) SB_FAIL(SB_EINVAL, "%s: %d channels (at most %d)", who, channels, kMaxChannels);
    LoadItems li;
    li.per_full = (g.out_full + 1023) / 1024; li.per_last = (g.out_last + 1023) / 1024;
    li.n_content = g.nfull * (int64_t)li.per_full + li.per_last;
    li.n_head = (padding + 1023) / 1024; li.n_tail = (padding + 1023) / 1024;
    *gout = g; *liout = li;
    return SB_OK;
}

// big-endian 16- or 24-bit samples -> the top 16 bits as int16
__global__ void __launch_bounds__(256)
k_pcm_be(const uint8_t* __restrict__ in, int64_t n, int width, int16_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint8_t* p = in + i * width;
        out[i] = (int16_t)(uint16_t)(((unsigned)p[0] << 8) | p[1]);
    }
}

}  // namespace

namespace sb {

// Everything of sb_load_pcm after the PCM is on the device: allocate the float32 stream and its coarse histogram and
// enqueue k_decode_resample_pad on the library stream.  d_pcm must stay valid until that work has run.
int load_pcm_device(const unsigned char* d_pcm, int64_t frames, int channels, int sample_width, int framerate,
                    int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32, const char* who) {
    Ctx& c = ctx();
    ResampleGeom g; LoadItems li;
    SB_TRY(plan_load(frames, channels, sample_width, framerate, sample_rate, padding, total_len, who, &g, &li));
    sb_stream* s = new (std::nothrow) sb_stream();
    if (!s) SB_FAIL(SB_ENOMEM, "%s: out of host memory", who);
    s->n = total_len; s->dtype = SB_F32; s->pcm_channels = channels;
    int rc = pool_alloc(&s->d_raw, sizeof(float) * total_len + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&s->d_loadhist, sizeof(unsigned long long) * (kCoarseBins + 1));
    if (rc != SB_OK) { pool_free(s->d_raw); delete s; return rc; }
    cudaError_t e = cudaMemsetAsync(s->d_loadhist, 0, sizeof(unsigned long long) * (kCoarseBins + 1), c.stream);
    if (e == cudaSuccess) {
        ProfScope ps("decode_resample_pad");
        k_decode_resample_pad<<<c.sm_count * 8, 256, 0, c.stream>>>(
            d_pcm, g, li, channels, sample_width, static_cast<float*>(s->d_raw), s->d_loadhist);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "%s: %s", who, cudaGetErrorString(e)); }
    *out_f32 = s;                 // no running sums yet: only sb_normalise / sb_stream_read accept it
    return SB_OK;
}

int pcm_handle(int16_t* d_pcm, int64_t frames, int channels, int rate, sb_pcm** out) {
    sb_pcm* p = new (std::nothrow) sb_pcm{d_pcm, frames, channels, rate};
    if (!p) { pool_free(d_pcm); SB_FAIL(SB_ENOMEM, "out of host memory for a decoded-PCM handle"); }
    *out = p;
    return SB_OK;
}

}  // namespace sb

extern "C" {

int sb_load_pcm(const void* pcm_host, int64_t frames, int channels, int sample_width,
                int framerate, int sample_rate, int64_t padding, int64_t total_len,
                sb_stream** out_f32) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_load_pcm: library not initialised (call sb_init)");
    if (!pcm_host || !out_f32) SB_FAIL(SB_EINVAL, "sb_load_pcm: NULL argument");
    ResampleGeom g; LoadItems li;
    SB_TRY(plan_load(frames, channels, sample_width, framerate, sample_rate, padding, total_len, "sb_load_pcm", &g, &li));
    unsigned char* d_pcm = nullptr;
    const size_t pcm_bytes = (size_t)frames * channels * sample_width;
    SB_TRY(pool_alloc((void**)&d_pcm, pcm_bytes + 16));
    sb_stream* s = nullptr;
    cudaError_t e = cudaMemcpyAsync(d_pcm, pcm_host, pcm_bytes, cudaMemcpyHostToDevice, c.stream);
    if (e != cudaSuccess) { pool_free(d_pcm); SB_FAIL(SB_ECUDA, "sb_load_pcm: %s", cudaGetErrorString(e)); }
    const int rc = load_pcm_device(d_pcm, frames, channels, sample_width, framerate, sample_rate, padding, total_len, &s,
                                   "sb_load_pcm");
    e = cudaStreamSynchronize(c.stream);                                  // pcm_host may be reused by the caller
    pool_free(d_pcm);
    if (rc != SB_OK) return rc;
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_load_pcm: %s", cudaGetErrorString(e)); }
    *out_f32 = s;
    return SB_OK;
}

int sb_pcm_info(const sb_pcm* pcm, int64_t* frames, int32_t* channels, int32_t* rate) {
    if (!pcm || !frames || !channels || !rate) SB_FAIL(SB_EINVAL, "sb_pcm_info: NULL argument");
    *frames = pcm->frames; *channels = pcm->channels; *rate = pcm->rate;
    return SB_OK;
}

int sb_pcm_load(const sb_pcm* pcm, int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_pcm_load: library not initialised (call sb_init)");
    if (!pcm || !out_f32) SB_FAIL(SB_EINVAL, "sb_pcm_load: NULL argument");
    sb_stream* s = nullptr;
    SB_TRY(load_pcm_device(reinterpret_cast<const unsigned char*>(pcm->d_pcm), pcm->frames, pcm->channels, 2, pcm->rate,
                           sample_rate, padding, total_len, &s, "sb_pcm_load"));
    const cudaError_t e = cudaStreamSynchronize(c.stream);
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_pcm_load: %s", cudaGetErrorString(e)); }
    *out_f32 = s;
    return SB_OK;
}

int sb_pcm_destroy(sb_pcm* pcm) {
    if (!pcm) return SB_OK;
    pool_free(pcm->d_pcm);
    delete pcm;
    return SB_OK;
}

int sb_pcm_from_be(const void* pcm_host, int64_t frames, int channels, int sample_width, int framerate, sb_pcm** out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_pcm_from_be: library not initialised (call sb_init)");
    if (!pcm_host || !out) SB_FAIL(SB_EINVAL, "sb_pcm_from_be: NULL argument");
    if (sample_width != 2 && sample_width != 3) SB_FAIL(SB_EINVAL, "Unsupported sample width: %d", sample_width);
    if (frames < 0 || channels < 1) SB_FAIL(SB_EINVAL, "sb_pcm_from_be: bad geometry");
    const int64_t n = frames * channels;
    unsigned char* d_in = nullptr;
    int16_t* d_pcm = nullptr;
    int rc = pool_alloc((void**)&d_in, (size_t)n * sample_width + 16);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_pcm, sizeof(int16_t) * (size_t)n + 16);
    if (rc != SB_OK) { pool_free(d_in); pool_free(d_pcm); return rc; }
    cudaError_t e = cudaMemcpyAsync(d_in, pcm_host, (size_t)n * sample_width, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && n > 0) {
        ProfScope ps("pcm_be");
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)c.sm_count * 16));
        k_pcm_be<<<grid, 256, 0, c.stream>>>(d_in, n, sample_width, d_pcm);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);             // pcm_host may be reused by the caller
    pool_free(d_in);
    if (e != cudaSuccess) { pool_free(d_pcm); SB_FAIL(SB_ECUDA, "sb_pcm_from_be: %s", cudaGetErrorString(e)); }
    return pcm_handle(d_pcm, frames, channels, framerate, out);
}

int sb_normalise(const sb_stream* raw_f32, int dtype, sb_stream** out, float* min3_out, float* max3_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_normalise: library not initialised (call sb_init)");
    if (!raw_f32 || !out) SB_FAIL(SB_EINVAL, "sb_normalise: NULL argument");
    if (raw_f32->dtype != SB_F32) SB_FAIL(SB_EINVAL, "sb_normalise: input must be a float32 stream from sb_load_pcm");
    if (dtype != SB_U8 && dtype != SB_F32) SB_FAIL(SB_EINVAL, "Unknown sample type of WAV stream, must be uint8 or float32");
    const int64_t n = raw_f32->n;
    const float* x = static_cast<const float*>(raw_f32->d_raw);
    if (!raw_f32->d_loadhist || raw_f32->pcm_channels < 1)
        SB_FAIL(SB_EINVAL, "sb_normalise: input was not produced by sb_load_pcm");
    float med_pos = 0.f, med_neg = 0.f;
    int rc = medians_from_histograms(raw_f32, &med_pos, &med_neg);
    if (rc != SB_OK) return rc;
    const float hi = med_pos * 3.0f, lo = med_neg * 3.0f;               // wav.py:145-146 (float32 products)
    if (min3_out) *min3_out = lo;
    if (max3_out) *max3_out = hi;

    sb_stream* s = new (std::nothrow) sb_stream();
    if (!s) SB_FAIL(SB_ENOMEM, "sb_normalise: out of host memory");
    s->n = n; s->dtype = dtype;
    rc = pool_alloc(&s->d_raw, (dtype == SB_U8 ? 1 : 4) * (size_t)n + 16);
    if (rc != SB_OK) { delete s; return rc; }
    {
        ProfScope ps("normalise_quantise");
        k_normalise<<<c.sm_count * 16, 256, 0, c.stream>>>(
            x, n, lo, hi, dtype == SB_F32 ? static_cast<float*>(s->d_raw) : nullptr,
            dtype == SB_U8 ? static_cast<unsigned char*>(s->d_raw) : nullptr);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { sb_stream_destroy(s); SB_FAIL(SB_ECUDA, "sb_normalise: %s", cudaGetErrorString(e)); }
    rc = stream_finish_public(s);
    if (rc != SB_OK) { sb_stream_destroy(s); return rc; }
    *out = s;
    return SB_OK;
}

}  // extern "C"
