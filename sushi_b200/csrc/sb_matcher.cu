// The matcher: WavStream.find_substream (reference wav.py:177-188), i.e.
// cv2.matchTemplate(TM_SQDIFF_NORMED) + first-index argmin, for batches of
// independent queries against a resident stream.
//
// Formulation (DESIGN.md section 3): uniformly partitioned overlap-save.  The image
// stream is cut into lag blocks of B positions; block spectra X_k = FFT_2B(image[kB
// .. kB+2B) - c) are built once per stream.  A template of n samples is cut into
// P = ceil(n/B) partitions T_p (zero padded to 2B).  For lag block k
//     corr_k = IFFT_2B( sum_p conj(T^_p) * X^_{k+p} )[0 .. B)
// is the centred cross-correlation at positions kB .. kB+B-1; the un-centred
// sum(I*T), the window energy sum(I^2) and sum(T^2) come from exact running sums,
// and OpenCV's normalisation rule + float32 rounding + first-index argmin are
// applied in the same kernel that runs the inverse FFT (sb_fused.cu, sb_fused2.cu).
// Both operands are centred before the fp32 FFTs, which keeps the transform error
// relative to the signal's variation instead of its offset: the image stream on
// a = mean of the whole stream, every template on b = its own mean (rounded to
// integers for uint8 data, so the centred samples stay exact).  The kernels undo
// the centring exactly from the running sums:
//     sum(I*T) = sum(I'T') + b*sum(I_w) + a*sum(T) - n*a*b
#include "sb_internal.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <vector>

namespace sb { int ensure_spectra(sb_stream* s); int ensure_spectra_quad(sb_stream* s, int64_t k_lo, int64_t k_hi); }
using namespace sb;

namespace {

// ---- register-blocked spectral multiply for long templates ------------------------------------
// G = MAC_GROUP consecutive lag blocks of one query share every template row: block g at partition
// step p needs spectrum row k0+g+p, so a ring of G row values slides by one row per step and each
// step costs one template load and ONE new spectrum load per bin for G multiply-accumulates (the
// fused kernel's own multiply loads 2 per multiply-accumulate).  Y[item][bin] goes to a buffer the fused kernel
// then reads instead of multiplying itself.  Rows are requested MACB_AHEAD steps early.
__global__ void k_fill_groups(const QueryDesc* __restrict__ desc, int q_begin, int64_t group_first, int2* __restrict__ groups) {
    const int q = q_begin + blockIdx.x;
    const int64_t base = desc[q].groupBase - group_first;
    const int ng = (desc[q].nk + MAC_GROUP - 1) / MAC_GROUP;
    for (int i = threadIdx.x; i < ng; i += blockDim.x) groups[base + i] = make_int2(q, i * MAC_GROUP);
}

constexpr int MACB_THREADS = 256;
constexpr int MACB_BINS = MACB_THREADS;             // one bin per thread: ~64 registers, 32 warps per SM
constexpr int MACB_AHEAD = 3;                       // spectrum / template rows requested this many steps early
__global__ void __launch_bounds__(MACB_THREADS, 4)
k_mac_blocked(const float2* __restrict__ That, int64_t part_first, const float2* __restrict__ Xhat, int64_t nblk,
              const QueryDesc* __restrict__ desc, const int2* __restrict__ groups, int64_t item_first,
              int B, float2* __restrict__ Y, int chunks_per_group) {
    constexpr int G = MAC_GROUP, D = MACB_AHEAD, RS = G + D;     // ring of RS spectrum values: slot r % RS holds row k0 + r
    const int2 grp = groups[blockIdx.x / chunks_per_group];
    const int chunk = blockIdx.x % chunks_per_group;
    const QueryDesc d = desc[grp.x];
    const int64_t k0 = d.k0 + grp.y;
    const int ng = min(G, d.nk - grp.y);
    const int nb = B + 1;
    const int b0 = chunk * MACB_BINS + threadIdx.x;
    if (b0 >= nb) return;
    const float2 zero = make_float2(0.f, 0.f);
    const float2* tp = That + (d.partBase - part_first) * (int64_t)nb + b0;
    const float2* xp = Xhat + k0 * (int64_t)nb + b0;
    const int P = d.P;
    const int64_t rows_left = nblk - k0;               // rows k0 + r with r >= rows_left are past the stream: zero
    float2 acc[G], x[RS], t[D + 1];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = zero;
#pragma unroll
    for (int r = 0; r < RS - 1; ++r) x[r] = r < rows_left ? __ldg(xp + (int64_t)r * nb) : zero;   // rows 0 .. G+D-2
    x[RS - 1] = zero;
#pragma unroll
    for (int i = 0; i < D; ++i) t[i] = i < P ? __ldg(tp + (int64_t)i * nb) : zero;
    t[D] = zero;
    // steps are unrolled RS*(D+1) at a time so that every ring index is a compile-time constant
    for (int p0 = 0; p0 < P; p0 += RS * (D + 1)) {
#pragma unroll
        for (int s = 0; s < RS * (D + 1); ++s) {
            const int p = p0 + s;
            if (p < P) {                               // uniform over the CTA
                // request what step p + D will need: row p+G+D-1 (into the slot of row p-1, now dead) and T^[p+D]
                const int64_t nr = (int64_t)p + G + D - 1;
                x[(s + G + D - 1) % RS] = nr < rows_left ? __ldg(xp + nr * nb) : zero;
                t[(s + D) % (D + 1)] = p + D < P ? __ldg(tp + (int64_t)(p + D) * nb) : zero;
                const float2 tv = t[s % (D + 1)];
#pragma unroll
                for (int g = 0; g < G; ++g) {          // block g at step p multiplies row k0 + g + p
                    const float2 a = x[(s + g) % RS];
                    acc[g].x += tv.x * a.x + tv.y * a.y;  acc[g].y += tv.x * a.y - tv.y * a.x;
                }
            }
        }
    }
    float2* y = Y + (d.itemBase + grp.y - item_first) * (int64_t)nb + b0;
#pragma unroll
    for (int g = 0; g < G; ++g)
        if (g < ng) y[(int64_t)g * nb] = acc[g];
}

// keys are in processing order; results go back in the caller's order
__global__ void k_unpack_results(const unsigned long long* __restrict__ keys, const QueryDesc* __restrict__ desc,
                                 int64_t count, float* __restrict__ diff, int64_t* __restrict__ idx) {
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q < count) {
        const unsigned long long k = keys[q];
        const int o = desc[q].orig;
        diff[o] = __uint_as_float((unsigned int)(k >> 32));
        idx[o] = (int64_t)(unsigned int)(k & 0xffffffffull);
    }
}

template <typename T>
int grow(T** p, int64_t* cap, int64_t need, bool pinned = false) {
    if (need <= *cap) return SB_OK;
    Ctx& c = ctx();
    cudaStreamSynchronize(c.stream);
    if (*p) { if (pinned) cudaFreeHost(*p); else cudaFree(*p); *p = nullptr; *cap = 0; }
    int64_t ncap = std::max<int64_t>(need, 16);
    cudaError_t e = pinned ? cudaMallocHost((void**)p, sizeof(T) * ncap) : cudaMalloc((void**)p, sizeof(T) * ncap);
    if (e != cudaSuccess) SB_FAIL(SB_ENOMEM, "allocation of %lld bytes failed: %s", (long long)(sizeof(T) * ncap), cudaGetErrorString(e));
    *cap = ncap;
    return SB_OK;
}

// Partition count from which a query goes through k_mac_blocked.  The blocked kernel moves ~5x fewer
// spectrum bytes per lag block, but its products make a round trip through HBM (2 x 131 KB per block)
// before the FFT, so it pays only for long templates.  The threshold was set on an earlier GPU and has not
// been re-measured on the H100.
constexpr int64_t kBlockedFromPartitions = 12;

// The streams of one call.  The single-stream entry points pass {image, tmpl} and no slots; a multi-stream call
// (sb_find_multi) passes its stream table and per-query image / template slots.
struct StreamSet {
    const sb_stream* image1 = nullptr; const sb_stream* tmpl1 = nullptr;                  // single-stream calls
    const sb_stream* const* s = nullptr; int64_t n = 0;                                     // multi-stream calls
    const int32_t* islot = nullptr; const int32_t* tslot = nullptr;
    const sb_stream* image(int64_t q) const { return islot ? s[islot[q]] : image1; }
    const sb_stream* tmpl(int64_t q) const { return tslot ? s[tslot[q]] : tmpl1; }
    bool multi() const { return islot != nullptr; }
};
StreamSet pair_of(const sb_stream* image, const sb_stream* tmpl) { StreamSet ss; ss.image1 = image; ss.tmpl1 = tmpl; return ss; }

// The per-query rules of every matcher entry point (q names the query in the caller's arrays)
int check_query(const sb_stream* image, const sb_stream* tmpl, int64_t q, int64_t o, int64_t n, int64_t s, int64_t L) {
    if (n < 1 || L < 1) SB_FAIL(SB_EINVAL, "query %lld: template length %lld / lag count %lld must be >= 1", (long long)q, (long long)n, (long long)L);
    if (o < 0 || o + n > tmpl->n) SB_FAIL(SB_EINVAL, "query %lld: template [%lld,+%lld) outside template stream of %lld samples", (long long)q, (long long)o, (long long)n, (long long)tmpl->n);
    if (s < 0 || s + L - 1 + n > image->n) SB_FAIL(SB_EINVAL, "query %lld: search span [%lld,+%lld)+%lld outside image stream of %lld samples", (long long)q, (long long)s, (long long)L, (long long)n, (long long)image->n);
    if (L > 0xffffffffll) SB_FAIL(SB_EINVAL, "query %lld: more than 2^32 lags", (long long)q);
    return SB_OK;
}

// Whether a template of n samples takes the register-blocked multiply route (every engine)
bool blocked_class(int64_t n) {
    const Ctx& c = ctx();
    if (c.premac_mode == 1) return false;
    return c.premac_mode == 2 || (n + kLagBlock - 1) / kLagBlock >= kBlockedFromPartitions;
}

// Validate + plan a batch on the host.  Fills c.h_desc[0..count) in PROCESSING order: first the queries
// whose multiply runs inside the fused kernel, then (from *n_direct on) those routed through the
// register-blocked multiply kernel.  The route depends only on the query itself (its partition count),
// never on what else is in the batch, so a given (template, position) always takes the same arithmetic
// path.  QueryDesc::orig maps back to the caller's order; curve offsets follow the caller's order.
int plan_batch(const StreamSet& ss, int64_t count,
               const int64_t* toff, const int64_t* tlen, const int64_t* lag0, const int64_t* nlags,
               int direct_group, int64_t* n_direct_out,
               int64_t* total_items, int64_t* total_parts, int64_t* total_groups, int64_t* max_query_parts) {
    Ctx& c = ctx();
    const int64_t B = kLagBlock;                    // partition length = hop = lags per item
    SB_CUDA(cudaEventSynchronize(c.ev_desc));       // previous batch has finished reading h_desc
    if (c.h_desc_cap < count) {
        if (c.h_desc) { cudaStreamSynchronize(c.stream); cudaFreeHost(c.h_desc); c.h_desc = nullptr; c.h_desc_cap = 0; }
        SB_CUDA(cudaMallocHost((void**)&c.h_desc, sizeof(QueryDesc) * std::max<int64_t>(count, 64)));
        c.h_desc_cap = std::max<int64_t>(count, 64);
    }
    int64_t n_direct = 0;
    for (int64_t q = 0; q < count; ++q) {
        SB_TRY(check_query(ss.image(q), ss.tmpl(q), q, toff[q], tlen[q], lag0[q], nlags[q]));
        if (!blocked_class(tlen[q])) ++n_direct;
    }
    int64_t items = 0, parts = 0, maxp = 0, groups = 0;
    int64_t pos_direct = 0, pos_blocked = n_direct;
    // two passes so that the running totals follow the processing order
    for (int cls = 0; cls < 2; ++cls) {
        int64_t curve_total = 0;
        for (int64_t q = 0; q < count; ++q) {
            const int64_t n = tlen[q], L = nlags[q], s = lag0[q];
            if ((blocked_class(n) ? 1 : 0) == cls) {
                QueryDesc& d = c.h_desc[cls == 0 ? pos_direct++ : pos_blocked++];
                d.toff = toff[q]; d.tlen = n; d.lag0 = s; d.nlags = L;
                d.P = (int32_t)((n + B - 1) / B);
                d.k0 = (int32_t)(s / B);
                d.nk = (int32_t)((s + L - 1) / B - d.k0 + 1);
                d.itemBase = items; d.partBase = parts; d.orig = (int32_t)q; d.curveOff = curve_total; d.groupBase = groups;
                groups += cls == 0 ? (d.nk + direct_group - 1) / direct_group : (d.nk + MAC_GROUP - 1) / MAC_GROUP;
                items += d.nk; parts += d.P;
                maxp = std::max<int64_t>(maxp, d.P);
            }
            curve_total += L;
        }
    }
    *n_direct_out = n_direct;
    *total_items = items; *total_parts = parts; *total_groups = groups; *max_query_parts = maxp;
    return SB_OK;
}

// Rows of the block spectra the queries of a multi-stream call read and that are not built yet, as (slot, row) pairs:
// run_batch builds them for every image stream in ONE launch of the forward kernel.  The bookkeeping per stream is
// ensure_spectra_quad's: the built range [specq_lo, specq_hi) stays contiguous and is extended on either side.
int spectra_rows_multi(const StreamSet& ss, int64_t count, StreamEntry* table, std::vector<int2>& rows) {
    Ctx& c = ctx();
    std::vector<int64_t> lo(ss.n, INT64_MAX), hi(ss.n, 0);
    for (int64_t q = 0; q < count; ++q) {
        const QueryDesc& d = c.h_desc[q];
        const int32_t i = ss.islot[d.orig];
        lo[i] = std::min<int64_t>(lo[i], d.k0);
        hi[i] = std::max<int64_t>(hi[i], (int64_t)d.k0 + d.nk + d.P);
    }
    for (int64_t i = 0; i < ss.n; ++i) {
        if (lo[i] == INT64_MAX) continue;
        sb_stream* s = const_cast<sb_stream*>(ss.s[i]);
        const int64_t nblk = (s->n + kLagBlock - 1) / kLagBlock;
        const int64_t k_lo = std::max<int64_t>(lo[i], 0), k_hi = std::min<int64_t>(hi[i], nblk);
        if (k_lo >= k_hi) continue;
        if (!s->d_specq) {
            SB_TRY(pool_alloc((void**)&s->d_specq, sizeof(float2) * (size_t)nblk * kQuadRowF2));
            s->nblkq = nblk; s->specq_lo = s->specq_hi = k_lo;
        }
        auto add = [&](int64_t a, int64_t b) { for (int64_t k = a; k < b; ++k) rows.push_back(make_int2((int)i, (int)k)); };
        if (s->specq_lo == s->specq_hi) { add(k_lo, k_hi); s->specq_lo = k_lo; s->specq_hi = k_hi; }
        else {
            if (k_lo < s->specq_lo) { add(k_lo, s->specq_lo); s->specq_lo = k_lo; }
            if (k_hi > s->specq_hi) { add(s->specq_hi, k_hi); s->specq_hi = k_hi; }
        }
        table[i].specq = s->d_specq; table[i].nblk = s->nblkq;
    }
    return SB_OK;
}

// Core: descriptors on host (validated here), results to device arrays d_diff/d_idx.
// Multi-stream calls (ss.multi()) run the packed engine's direct class only (sb_find_multi routes everything else
// through single-stream calls); every kernel then reads its query's streams from a table uploaded here.
int run_batch(const StreamSet& ss, int64_t count,
              const int64_t* toff, const int64_t* tlen, const int64_t* lag0, const int64_t* nlags,
              float* d_diff, int64_t* d_idx, float* d_curve) {
    Ctx& c = ctx();
    sb_stream* image = const_cast<sb_stream*>(ss.image(0));
    const sb_stream* tmpl = ss.tmpl(0);
    if (!ss.multi() && image->dtype != tmpl->dtype) SB_FAIL(SB_EINVAL, "image and template streams differ in sample type");
    if (count > 0x7fffffffll) SB_FAIL(SB_EINVAL, "more than 2^31 queries in one batch");
    const int B = kLagBlock;
    // Multiply strategy per query: inside the fused kernel (2 loads per multiply-accumulate, nothing through
    // HBM), or -- for very long templates (kBlockedFromPartitions) -- the register-blocked kernel
    // k_mac_blocked over MAC_GROUP lag blocks, whose products the fused kernel then reads from a chunk buffer.
    // Engine 1 runs the direct class on the fused kernel of sb_fused.cu; engines 2 / 4 / 5 run it on the packed
    // kernels (sb_fused2.cu) over quad-layout spectrum rows.  The blocked class always keeps engine 1's kernels and
    // the classic row layout, so a stream may hold its block spectra in both layouts.
    const bool use_packed = c.engine >= 2;
    const int nb = B + 1;                                    // float2 per classic spectrum row
    int64_t n_direct = 0, total_items = 0, total_parts = 0, total_groups = 0, maxp = 0;
    SB_TRY(plan_batch(ss, count, toff, tlen, lag0, nlags, 2, &n_direct,
                      &total_items, &total_parts, &total_groups, &maxp));
    if (ss.multi() && (!use_packed || n_direct != count)) SB_FAIL(SB_EINVAL, "internal: a multi-stream batch must be packed direct-class only");
    // Packed kernels: one CTA per lag block, or one per pair of consecutive lag blocks of a query (shared template
    // rows, 2P+1 row reads instead of 4P, second product spectrum parked in L2).  Both give bit-identical results;
    // pairs pay from about four partitions per template (H100 SXM at 400 W, 1000 queries at +-120 s on 30-min streams:
    // pair / single time 1.18 at P = 1, 1.05 at P = 3, 1.00 at P = 4, 0.87 at P = 6, 0.75 at P = 11), so engine 2
    // picks per batch by the average partition count; engines 4 / 5 force one or the other.
    bool use_pairs = c.engine == 4;
    if (use_packed && c.engine == 2 && n_direct > 0) {
        double rows = 0.0, blocks = 0.0;
        for (int64_t q = 0; q < n_direct; ++q) { rows += (double)c.h_desc[q].nk * c.h_desc[q].P; blocks += (double)c.h_desc[q].nk; }
        use_pairs = rows >= 4.0 * blocks;
    }
    // multi-stream calls: the stream table (StreamEntry per slot), the slots of every query in processing order and
    // the row list of the block spectra, in one device buffer
    MultiArgs multi{};
    const MultiArgs* mp = nullptr;
    if (ss.multi()) {
        const size_t tb = (sizeof(StreamEntry) * ss.n + 15) & ~(size_t)15, sb = (sizeof(int2) * count + 15) & ~(size_t)15;
        int64_t max_rows = 0;
        for (int64_t i = 0; i < ss.n; ++i) max_rows += (ss.s[i]->n + B - 1) / B;
        SB_TRY(grow(&c.d_multi, &c.multi_cap, (int64_t)(tb + sb + sizeof(int2) * max_rows)));
        std::vector<StreamEntry> table(ss.n);
        for (int64_t i = 0; i < ss.n; ++i) table[i] = {ss.s[i]->d_specq, ss.s[i]->nblkq, ss.s[i]->d_raw, ss.s[i]->n, ss.s[i]->d_pfx};
        multi.d_streams = reinterpret_cast<const StreamEntry*>(c.d_multi);
        multi.d_slots = reinterpret_cast<const int2*>(c.d_multi + tb);
        multi.dtype = image->dtype;
        mp = &multi;
        std::vector<int2> rows, slots(count);
        SB_TRY(spectra_rows_multi(ss, count, table.data(), rows));
        for (int64_t q = 0; q < count; ++q) slots[q] = make_int2(ss.islot[c.h_desc[q].orig], ss.tslot[c.h_desc[q].orig]);
        int2* d_rows = reinterpret_cast<int2*>(c.d_multi + tb + sb);
        SB_CUDA(cudaMemcpyAsync(c.d_multi, table.data(), sizeof(StreamEntry) * ss.n, cudaMemcpyHostToDevice, c.stream));
        SB_CUDA(cudaMemcpyAsync(c.d_multi + tb, slots.data(), sizeof(int2) * count, cudaMemcpyHostToDevice, c.stream));
        if (!rows.empty()) {
            SB_CUDA(cudaMemcpyAsync(d_rows, rows.data(), sizeof(int2) * rows.size(), cudaMemcpyHostToDevice, c.stream));
            ProfScope ps("block_spectra");
            SB_TRY(launch_block_spectra_quad_multi(multi, d_rows, (int64_t)rows.size()));
        }
    } else if (use_packed && n_direct > 0) {
        // spectrum rows the direct class reads: lag block k of a query multiplies rows k .. k+P-1 (a pair: .. k+P)
        int64_t k_lo = INT64_MAX, k_hi = 0;
        for (int64_t q = 0; q < n_direct; ++q) {
            const QueryDesc& d = c.h_desc[q];
            k_lo = std::min<int64_t>(k_lo, d.k0);
            k_hi = std::max<int64_t>(k_hi, (int64_t)d.k0 + d.nk + d.P);
        }
        SB_TRY(ensure_spectra_quad(image, k_lo, k_hi));
    }
    if (!use_packed || n_direct < count) SB_TRY(ensure_spectra(image));

    SB_TRY(grow(&c.d_desc, &c.desc_cap, count));
    SB_TRY(grow(&c.d_keys, &c.keys_cap, count));
    SB_CUDA(cudaMemcpyAsync(c.d_desc, c.h_desc, sizeof(QueryDesc) * count, cudaMemcpyHostToDevice, c.stream));
    SB_CUDA(cudaEventRecord(c.ev_desc, c.stream));
    SB_CUDA(cudaMemsetAsync(c.d_keys, 0xff, sizeof(unsigned long long) * count, c.stream));

    const int64_t parts_cap_want = std::max<int64_t>(std::min<int64_t>(total_parts, c.max_parts), maxp);
    // float2 per template partition row: quad layout or classic
    const int64_t part_row_f2 = use_packed ? kQuadRowF2 : nb;
    SB_TRY(grow(&c.d_parts, &c.parts_cap, parts_cap_want * part_row_f2));
    // lag blocks per product buffer (0.5 GB)
    const int64_t premac_chunk = 4096;

    // the two query classes, each in super-chunks of whole queries whose partition spectra fit the buffer
    for (int cls = 0; cls < 2; ++cls) {
    const int64_t q_lo = cls == 0 ? 0 : n_direct, q_hi = cls == 0 ? n_direct : count;
    const bool premac = cls == 1;
    int64_t qb = q_lo;
    while (qb < q_hi) {
        int64_t qe = qb, np = 0;
        while (qe < q_hi && np + c.h_desc[qe].P <= parts_cap_want) { np += c.h_desc[qe].P; ++qe; }
        if (qe == qb) SB_FAIL(SB_ENOMEM, "internal: partition buffer too small");
        const int64_t part_first = c.h_desc[qb].partBase;
        // 1. template partitions -> spectra
        {
            ProfScope ps("part_spectra");
            if (use_packed && !premac) SB_TRY(launch_part_spectra_quad(tmpl, c.d_desc, (int)qb, (int)qe, part_first, np, c.d_parts, mp));
            else SB_TRY(launch_part_spectra(tmpl, c.d_desc, (int)qb, (int)qe, part_first, np, c.d_parts));
        }
        // 2. items of these queries
        const int64_t item_lo = c.h_desc[qb].itemBase;
        const int64_t item_hi = (qe < count) ? c.h_desc[qe].itemBase : total_items;
        if (use_packed && !premac) {
            ProfScope ps("match_fused");
            if (use_pairs) {
                const int64_t g0 = c.h_desc[qb].groupBase;
                const int64_t g1 = (qe < count) ? c.h_desc[qe].groupBase : total_groups;
                SB_TRY(launch_match_pair(image, tmpl, c.d_parts, part_first, c.d_desc, (int)qb, (int)qe, g0, g1 - g0, c.d_keys, d_curve, mp));
            } else
                SB_TRY(launch_match_packed(image, tmpl, c.d_parts, part_first, c.d_desc, (int)qb, (int)qe,
                                           item_lo, item_hi - item_lo, c.d_keys, d_curve, mp));
        } else if (!premac) {
            ProfScope ps("match_fused");
            SB_TRY(launch_match_fused(image, tmpl, c.d_parts, part_first, nullptr, c.d_desc, (int)qb, (int)qe,
                                      item_lo, item_hi - item_lo, c.d_keys, d_curve));
        } else {
            int64_t qa = qb;
            while (qa < qe) {
                int64_t qz = qa, ni = 0;
                while (qz < qe && (qz == qa || ni + c.h_desc[qz].nk <= premac_chunk)) { ni += c.h_desc[qz].nk; ++qz; }
                const int64_t i0 = c.h_desc[qa].itemBase, g0 = c.h_desc[qa].groupBase;
                const int64_t ngroups = ((qz < count) ? c.h_desc[qz].groupBase : total_groups) - g0;
                SB_TRY(grow(&c.d_items, &c.items_cap, ni * nb));
                SB_TRY(grow(&c.d_groups, &c.groups_cap, ngroups));
                const int gch = (nb + MACB_BINS - 1) / MACB_BINS;
                {
                    ProfScope ps("mac_blocked", 2);
                    k_fill_groups<<<(unsigned)(qz - qa), 128, 0, c.stream>>>(c.d_desc, (int)qa, g0, c.d_groups);
                    k_mac_blocked<<<(unsigned)(ngroups * gch), MACB_THREADS, 0, c.stream>>>(
                        c.d_parts, part_first, image->d_spec, image->nblk, c.d_desc, c.d_groups, i0, B, c.d_items, gch);
                }
                {
                    ProfScope ps("match_fused");
                    SB_TRY(launch_match_fused(image, tmpl, c.d_parts, part_first, c.d_items, c.d_desc, (int)qa, (int)qz,
                                              i0, ni, c.d_keys, d_curve));
                }
                qa = qz;
            }
        }
        qb = qe;
    }
    }
    {
        ProfScope ps("unpack_results");
        k_unpack_results<<<(unsigned)((count + 255) / 256), 256, 0, c.stream>>>(c.d_keys, c.d_desc, count, d_diff, d_idx);
    }
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// Queries of `ss` with results to host arrays (sb_find_batch)
int find_to_host(const StreamSet& ss, int64_t count, const int64_t* tmpl_off, const int64_t* tmpl_len,
                 const int64_t* lag0, const int64_t* nlags, float* diff_out, int64_t* idx_out) {
    Ctx& c = ctx();
    if (c.res_cap < count) {
        cudaStreamSynchronize(c.stream);
        cudaFree(c.d_diff); cudaFree(c.d_idx); c.d_diff = nullptr; c.d_idx = nullptr; c.res_cap = 0;
        SB_CUDA(cudaMalloc(&c.d_diff, sizeof(float) * count));
        SB_CUDA(cudaMalloc(&c.d_idx, sizeof(int64_t) * count));
        c.res_cap = count;
    }
    if (c.h_res_cap < count) {
        cudaFreeHost(c.h_diff); cudaFreeHost(c.h_idx); c.h_diff = nullptr; c.h_idx = nullptr; c.h_res_cap = 0;
        SB_CUDA(cudaMallocHost((void**)&c.h_diff, sizeof(float) * count));
        SB_CUDA(cudaMallocHost((void**)&c.h_idx, sizeof(int64_t) * count));
        c.h_res_cap = count;
    }
    SB_TRY(run_batch(ss, count, tmpl_off, tmpl_len, lag0, nlags, c.d_diff, c.d_idx, nullptr));
    SB_CUDA(cudaMemcpyAsync(c.h_diff, c.d_diff, sizeof(float) * count, cudaMemcpyDeviceToHost, c.stream));
    SB_CUDA(cudaMemcpyAsync(c.h_idx, c.d_idx, sizeof(int64_t) * count, cudaMemcpyDeviceToHost, c.stream));
    SB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(diff_out, c.h_diff, sizeof(float) * count);
    memcpy(idx_out, c.h_idx, sizeof(int64_t) * count);
    return SB_OK;
}

// Whole curves of the queries of `ss`, concatenated in query order, to a host array (sb_match_curves)
int curves_to_host(const StreamSet& ss, int64_t count, const int64_t* tmpl_off, const int64_t* tmpl_len,
                   const int64_t* lag0, const int64_t* nlags, float* curves_out) {
    int64_t total = 0;
    for (int64_t q = 0; q < count; ++q) total += nlags[q];
    Ctx& c = ctx();
    float* d_curve = nullptr; float* d_diff = nullptr; int64_t* d_idx = nullptr;
    SB_TRY(pool_alloc((void**)&d_curve, sizeof(float) * total));
    int rc = pool_alloc((void**)&d_diff, sizeof(float) * count);
    if (rc == SB_OK) rc = pool_alloc((void**)&d_idx, sizeof(int64_t) * count);
    if (rc == SB_OK) rc = run_batch(ss, count, tmpl_off, tmpl_len, lag0, nlags, d_diff, d_idx, d_curve);
    if (rc == SB_OK) {
        cudaError_t e = cudaMemcpyAsync(curves_out, d_curve, sizeof(float) * total, cudaMemcpyDeviceToHost, c.stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        if (e != cudaSuccess) { set_error("sb_match_curves: D2H: %s", cudaGetErrorString(e)); rc = SB_ECUDA; }
    }
    pool_free(d_curve); pool_free(d_diff); pool_free(d_idx);
    return rc;
}

// Multi-stream calls.  The packed engine's direct class (engines 2, 4, 5; templates below the blocked threshold) goes
// out as ONE multi-stream batch, whatever the number of streams.  Everything else -- the blocked class and engine 1 --
// runs as one ordinary single-stream batch per distinct (image, template) pair inside the same call: same results,
// more launches.  Results land in the caller's order.
int run_multi(const char* who, const sb_stream* const* streams, int32_t n_streams, int64_t count,
              const int32_t* image_slot, const int32_t* tmpl_slot, const int64_t* tmpl_off, const int64_t* tmpl_len,
              const int64_t* lag0, const int64_t* nlags, float* diff_out, int64_t* idx_out, float* curves_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "%s: library not initialised (call sb_init)", who);
    if (count < 0) SB_FAIL(SB_EINVAL, "%s: negative count", who);
    if (count == 0) return SB_OK;
    if (!streams || n_streams < 1) SB_FAIL(SB_EINVAL, "%s: no streams", who);
    if (!image_slot || !tmpl_slot || !tmpl_off || !tmpl_len || !lag0 || !nlags || (curves_out ? false : (!diff_out || !idx_out)))
        SB_FAIL(SB_EINVAL, "%s: NULL array", who);
    for (int32_t i = 0; i < n_streams; ++i) {
        if (!streams[i]) SB_FAIL(SB_EINVAL, "%s: stream slot %d is NULL", who, (int)i);
        if (!streams[i]->d_pfx) SB_FAIL(SB_EINVAL, "%s: stream slot %d has no running sums (a raw sb_load_pcm stream must go through sb_normalise)", who, (int)i);
        if (streams[i]->dtype != streams[0]->dtype) SB_FAIL(SB_EINVAL, "%s: stream slot %d differs in sample type from slot 0 (all streams of a call share one)", who, (int)i);
    }
    for (int64_t q = 0; q < count; ++q) {
        if (image_slot[q] < 0 || image_slot[q] >= n_streams) SB_FAIL(SB_EINVAL, "%s: query %lld: image slot %d outside [0, %d)", who, (long long)q, (int)image_slot[q], (int)n_streams);
        if (tmpl_slot[q] < 0 || tmpl_slot[q] >= n_streams) SB_FAIL(SB_EINVAL, "%s: query %lld: template slot %d outside [0, %d)", who, (long long)q, (int)tmpl_slot[q], (int)n_streams);
        SB_TRY(check_query(streams[image_slot[q]], streams[tmpl_slot[q]], q, tmpl_off[q], tmpl_len[q], lag0[q], nlags[q]));
    }
    const bool packed = c.engine >= 2;
    std::vector<int64_t> curve_off(count + 1, 0);
    for (int64_t q = 0; q < count; ++q) curve_off[q + 1] = curve_off[q] + nlags[q];
    // one subset of the queries: descriptor arrays gathered, results scattered back to the caller's positions
    auto run_subset = [&](const std::vector<int64_t>& sel, const StreamSet& ss, std::vector<int32_t>* slots) -> int {
        const int64_t m = (int64_t)sel.size();
        std::vector<int64_t> a(4 * m);
        for (int64_t i = 0; i < m; ++i) {
            const int64_t q = sel[i];
            a[i] = tmpl_off[q]; a[m + i] = tmpl_len[q]; a[2 * m + i] = lag0[q]; a[3 * m + i] = nlags[q];
            if (slots) { slots[0].push_back(image_slot[q]); slots[1].push_back(tmpl_slot[q]); }
        }
        StreamSet s2 = ss;
        if (slots) { s2.islot = slots[0].data(); s2.tslot = slots[1].data(); }
        if (curves_out && m == count) {        // every query, in the caller's order: straight into the caller's array
            SB_TRY(curves_to_host(s2, m, &a[0], &a[m], &a[2 * m], &a[3 * m], curves_out));
        } else if (curves_out) {
            int64_t total = 0;
            for (int64_t i = 0; i < m; ++i) total += a[3 * m + i];
            std::vector<float> cur(total);
            SB_TRY(curves_to_host(s2, m, &a[0], &a[m], &a[2 * m], &a[3 * m], cur.data()));
            for (int64_t i = 0, o = 0; i < m; o += a[3 * m + i], ++i) memcpy(curves_out + curve_off[sel[i]], cur.data() + o, sizeof(float) * a[3 * m + i]);
        } else {
            std::vector<float> d(m);
            std::vector<int64_t> k(m);
            SB_TRY(find_to_host(s2, m, &a[0], &a[m], &a[2 * m], &a[3 * m], d.data(), k.data()));
            for (int64_t i = 0; i < m; ++i) { diff_out[sel[i]] = d[i]; idx_out[sel[i]] = k[i]; }
        }
        return SB_OK;
    };
    std::vector<int64_t> direct;
    std::map<std::pair<int32_t, int32_t>, std::vector<int64_t>> other;
    for (int64_t q = 0; q < count; ++q) {
        if (packed && !blocked_class(tmpl_len[q])) direct.push_back(q);
        else other[{image_slot[q], tmpl_slot[q]}].push_back(q);
    }
    if (!direct.empty()) {
        StreamSet ss; ss.s = streams; ss.n = n_streams;
        std::vector<int32_t> slots[2];
        SB_TRY(run_subset(direct, ss, slots));
    }
    for (const auto& g : other) SB_TRY(run_subset(g.second, pair_of(streams[g.first.first], streams[g.first.second]), nullptr));
    return SB_OK;
}

int check_common(const char* who, const sb_stream* image, const sb_stream* tmpl, int64_t count) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "%s: library not initialised (call sb_init)", who);
    if (!image || !tmpl) SB_FAIL(SB_EINVAL, "%s: NULL stream", who);
    if (!image->d_pfx || !tmpl->d_pfx) SB_FAIL(SB_EINVAL, "%s: stream has no running sums (a raw sb_load_pcm stream must go through sb_normalise)", who);
    if (count < 0) SB_FAIL(SB_EINVAL, "%s: negative count", who);
    return SB_OK;
}

}  // namespace

extern "C" {

int sb_find_batch(const sb_stream* image, const sb_stream* tmpl, int64_t count,
                  const int64_t* tmpl_off, const int64_t* tmpl_len,
                  const int64_t* lag0, const int64_t* nlags,
                  float* diff_out, int64_t* idx_out) {
    SB_TRY(check_common("sb_find_batch", image, tmpl, count));
    if (count == 0) return SB_OK;
    if (!tmpl_off || !tmpl_len || !lag0 || !nlags || !diff_out || !idx_out) SB_FAIL(SB_EINVAL, "sb_find_batch: NULL array");
    return find_to_host(pair_of(image, tmpl), count, tmpl_off, tmpl_len, lag0, nlags, diff_out, idx_out);
}

int sb_find_batch_device(const sb_stream* image, const sb_stream* tmpl, int64_t count,
                         const int64_t* tmpl_off, const int64_t* tmpl_len,
                         const int64_t* lag0, const int64_t* nlags,
                         float* d_diff_out, int64_t* d_idx_out) {
    SB_TRY(check_common("sb_find_batch_device", image, tmpl, count));
    if (count == 0) return SB_OK;
    if (!tmpl_off || !tmpl_len || !lag0 || !nlags || !d_diff_out || !d_idx_out) SB_FAIL(SB_EINVAL, "sb_find_batch_device: NULL array");
    return run_batch(pair_of(image, tmpl), count, tmpl_off, tmpl_len, lag0, nlags, d_diff_out, d_idx_out, nullptr);
}

int sb_find(const sb_stream* image, const void* tmpl_host, int64_t tmpl_len,
            int64_t lag0, int64_t nlags, float* diff_out, int64_t* idx_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_find: library not initialised (call sb_init)");
    if (!image || !tmpl_host) SB_FAIL(SB_EINVAL, "sb_find: NULL argument");
    sb_stream* t = nullptr;
    SB_TRY(sb_stream_create(tmpl_host, tmpl_len, image->dtype, &t));
    const int64_t zero = 0;
    int rc = sb_find_batch(image, t, 1, &zero, &tmpl_len, &lag0, &nlags, diff_out, idx_out);
    sb_stream_destroy(t);
    return rc;
}

int sb_match_curves(const sb_stream* image, const sb_stream* tmpl, int64_t count,
                    const int64_t* tmpl_off, const int64_t* tmpl_len,
                    const int64_t* lag0, const int64_t* nlags, float* curves_out) {
    SB_TRY(check_common("sb_match_curves", image, tmpl, count));
    if (count == 0) return SB_OK;
    if (!tmpl_off || !tmpl_len || !lag0 || !nlags || !curves_out) SB_FAIL(SB_EINVAL, "sb_match_curves: NULL array");
    for (int64_t q = 0; q < count; ++q)
        if (nlags[q] < 1) SB_FAIL(SB_EINVAL, "sb_match_curves: query %lld has nlags < 1", (long long)q);
    return curves_to_host(pair_of(image, tmpl), count, tmpl_off, tmpl_len, lag0, nlags, curves_out);
}

int sb_find_multi(const sb_stream* const* streams, int32_t n_streams, int64_t count,
                  const int32_t* image_slot, const int32_t* tmpl_slot,
                  const int64_t* tmpl_off, const int64_t* tmpl_len,
                  const int64_t* lag0, const int64_t* nlags,
                  float* diff_out, int64_t* idx_out) {
    return run_multi("sb_find_multi", streams, n_streams, count, image_slot, tmpl_slot, tmpl_off, tmpl_len, lag0, nlags,
                     diff_out, idx_out, nullptr);
}

int sb_match_curves_multi(const sb_stream* const* streams, int32_t n_streams, int64_t count,
                          const int32_t* image_slot, const int32_t* tmpl_slot,
                          const int64_t* tmpl_off, const int64_t* tmpl_len,
                          const int64_t* lag0, const int64_t* nlags, float* curves_out) {
    if (!curves_out && count > 0) SB_FAIL(SB_EINVAL, "sb_match_curves_multi: NULL array");
    return run_multi("sb_match_curves_multi", streams, n_streams, count, image_slot, tmpl_slot, tmpl_off, tmpl_len, lag0, nlags,
                     nullptr, nullptr, curves_out);
}

int sb_match_curve(const sb_stream* image, const sb_stream* tmpl,
                   int64_t tmpl_off, int64_t tmpl_len, int64_t lag0, int64_t nlags,
                   float* curve_out) {
    return sb_match_curves(image, tmpl, 1, &tmpl_off, &tmpl_len, &lag0, &nlags, curve_out);
}

}  // extern "C"
