// Internal declarations shared by the translation units of libsushi_b200.so.
// Nothing here is part of the ABI (see include/sushi_b200.h for that).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <map>
#include <functional>

#include "sushi_b200.h"

struct sb_stream;
struct sb_pcm;

namespace sb {

// ---- error plumbing ---------------------------------------------------------
void set_error(const char* fmt, ...);
#define SB_FAIL(code, ...) do { sb::set_error(__VA_ARGS__); return (code); } while (0)
#define SB_CUDA(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
    sb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    return SB_ECUDA; } } while (0)
#define SB_TRY(expr) do { int rc__ = (expr); if (rc__ != SB_OK) return rc__; } while (0)

// ---- per-kernel accounting --------------------------------------------------
struct ProfEntry { double ms = 0.0; int64_t launches = 0; };
struct PendingEvent { int name_id; cudaEvent_t a, b; };

// ---- query descriptor as the kernels see it ----------------------------------
// One query = one find_substream call (reference wav.py:177-188) reduced to
// integer sample offsets.  itemBase / partBase are exclusive prefix sums over the
// batch: item = (query, lag block k), part = (query, template partition p).
struct QueryDesc {
    int64_t toff;      // template start in the template stream
    int64_t tlen;      // template length n
    int64_t lag0;      // first candidate position in the image stream
    int64_t nlags;     // number of candidate positions L
    int64_t itemBase;  // first item of this query in the batch-wide item list
    int64_t partBase;  // first partition spectrum of this query
    int64_t curveOff;  // where this query's curve starts in the curve buffer (curve mode only)
    int64_t groupBase; // first multiply group of this query in the batch: MAC_GROUP consecutive lag blocks (blocked class), pairs of lag blocks (direct class)
    int32_t P;         // ceil(n / B): template partitions of B samples
    int32_t k0;        // lag0 / B: first lag block (B lags per item)
    int32_t nk;        // number of lag blocks touched
    int32_t orig;      // index of this query in the caller's arrays (descriptors are in processing order)
};

constexpr int kLagBlock = 16384;  // B: lags per lag block and samples per template partition (hop B); the FFT size is 2B
constexpr int MAC_GROUP = 8;      // lag blocks per register-blocked multiply group (sb_matcher.cu: k_mac_blocked)

struct Ctx {
    bool inited = false;
    int device = -1;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    int engine = 2;                // 2: packed fused kernels (sb_fused2.cu; default), 4 / 5: always / never pairs of lag blocks, 1: fused lag-block kernel (sb_fused.cu)
    int premac_mode = 0;           // 0: register-blocked multiply kernel for queries whose template spans >= 12 partitions, 1: never, 2: always
    int epilogue = 3;              // body of the packed kernels on uint8 streams: 3 = run-level bounds + k_finish_runs (default), 1 = first version (sb_set_epilogue)
    int64_t max_parts = 16384;     // template partition spectra kept per super-chunk

    // scratch (grown on demand)
    float2* d_parts = nullptr;  int64_t parts_cap = 0;     // [parts][B+1] complex (in-place R2C)
    float2* d_items = nullptr;  int64_t items_cap = 0;     // [items][B+1] complex products of the blocked multiply (k_mac_blocked)
    QueryDesc* d_desc = nullptr; int64_t desc_cap = 0;
    int2* d_groups = nullptr; int64_t groups_cap = 0;      // (query, first local lag block) per multiply group
    unsigned long long* d_keys = nullptr; int64_t keys_cap = 0;
    unsigned char* d_multi = nullptr; int64_t multi_cap = 0;   // multi-stream calls: stream table, per-query slots, spectrum row list
    float* d_diff = nullptr; int64_t* d_idx = nullptr; int64_t res_cap = 0;
    // pinned staging
    QueryDesc* h_desc = nullptr; int64_t h_desc_cap = 0;
    float* h_diff = nullptr; int64_t* h_idx = nullptr; int64_t h_res_cap = 0;

    // timers / profile
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    cudaEvent_t ev_desc = nullptr;   // marks the last H2D copy out of h_desc
    bool prof_on = false;
    std::vector<std::string> prof_names;
    std::vector<ProfEntry> prof;
    std::vector<PendingEvent> pending;
    std::vector<cudaEvent_t> event_pool;
    int64_t launches = 0;
};

Ctx& ctx();
int prof_id(const char* name);
int prof_collect();

// RAII bracket around every kernel class: counts launches, and records CUDA events when profiling is on
struct ProfScope {
    int id; cudaEvent_t a = nullptr, b = nullptr; bool on;
    explicit ProfScope(const char* name, int nlaunch = 1);
    ~ProfScope();
};

// Size-keyed pool of device blocks: streams are created and destroyed per batch by some
// callers; cudaMalloc/cudaFree (which synchronise the device) must not sit on that path.
int pool_alloc(void** out, size_t bytes);
void pool_free(void* p);
void pool_release_all();

// engine 2 (sb_fused2.cu): spectrum rows in the quad layout, kQuadRowF2 float2 per row (128-byte aligned)
constexpr int kQuadRowF2 = 16400;

// One stream of a multi-stream call (sb_find_multi / sb_match_curves_multi), as the packed kernels read it: its
// quad-layout spectrum rows and their count, its raw samples and their count, its running sums.  The table is built
// per call and uploaded next to the descriptors; a second array gives every query (processing order) its image slot
// (.x) and template slot (.y).  All streams of one call share a sample type.
struct StreamEntry {
    float2* specq; int64_t nblk;
    const void* raw; int64_t n;
    const double2* pfx;
};
struct MultiArgs { const StreamEntry* d_streams; const int2* d_slots; int dtype; };

// multi == nullptr: one image and one template stream (the kernels compiled as before); otherwise image / tmpl are
// ignored and every query reads its streams from the table
int launch_match_packed(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first,
                        const QueryDesc* d_desc, int q_begin, int q_end, int64_t item_first, int64_t n_items,
                        unsigned long long* d_keys, float* d_curve, const MultiArgs* multi = nullptr);
int launch_match_pair(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first,
                      const QueryDesc* d_desc, int q_begin, int q_end, int64_t pair_first, int64_t n_pairs,
                      unsigned long long* d_keys, float* d_curve, const MultiArgs* multi = nullptr);
int launch_block_spectra_quad(const sb_stream* s, int64_t k_first, int64_t rows, float2* out);
// block spectra rows of several streams in one launch: row_list[i] = (slot, row)
int launch_block_spectra_quad_multi(const MultiArgs& multi, const int2* d_row_list, int64_t n_rows);
int launch_part_spectra_quad(const sb_stream* tmpl, const QueryDesc* d_desc, int q_begin, int q_end,
                             int64_t part_first, int64_t rows, float2* out, const MultiArgs* multi = nullptr);
void packed_release_tables();

int launch_match_fused(const sb_stream* image, const sb_stream* tmpl, const float2* d_parts, int64_t part_first, const float2* d_premac,
                       const QueryDesc* d_desc, int q_begin, int q_end, int64_t item_first, int64_t n_items,
                       unsigned long long* d_keys, float* d_curve);
int launch_block_spectra(const sb_stream* s, int64_t k_first, int64_t rows, float2* out);
int launch_part_spectra(const sb_stream* tmpl, const QueryDesc* d_desc, int q_begin, int q_end,
                        int64_t part_first, int64_t rows, float2* out);
void fused_release_tables();

// sb_loader.cu: sb_load_pcm after its host-to-device copy (sb_pcm_load feeds it a decoder's int16 PCM on the device)
int load_pcm_device(const unsigned char* d_pcm, int64_t frames, int channels, int sample_width, int framerate,
                    int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32, const char* who);

// sb_loader.cu: a decoded-PCM handle that takes ownership of d_pcm (a pool block); on failure d_pcm is freed
int pcm_handle(int16_t* d_pcm, int64_t frames, int channels, int rate, sb_pcm** out);

// sb_truehd.cu: sb_truehd_decode on a stream already on the device (sb_ts.cu feeds it a transport stream's TrueHD
// payload); where(off) names the file offset of stream byte `off` in messages
int truehd_index_device(const uint8_t* host, const uint8_t* d_buf, int64_t nbytes, const int64_t* offsets,
                        const int64_t* d_blocks, int64_t n, const std::function<int64_t(int64_t)>& where, sb_pcm** out);

}  // namespace sb

// The decoded-PCM handle of the ABI: interleaved int16 PCM on the device, what every decoder produces.
struct sb_pcm {
    int16_t* d_pcm;
    int64_t frames;
    int channels, rate;
};

// The opaque stream handle of the ABI.
struct sb_stream {
    int64_t n = 0;
    int dtype = SB_U8;
    // streams produced by sb_load_pcm: channel count of the PCM they came from and the coarse value histogram the
    // decode kernel accumulated (sb_normalise selects the medians from it)
    int pcm_channels = 0;
    unsigned long long* d_loadhist = nullptr;
    void* d_raw = nullptr;        // n samples (u8 or f32)
    double2* d_pfx = nullptr;     // [n+1] running sums: .x = sum of samples, .y = sum of squares (exact for u8)
    // block spectra in the classic layout of engine 1's kernels: [nblk][B+1] complex64, row k = FFT_2B of samples [kB, kB+2B)
    float2* d_spec = nullptr;
    int64_t nblk = 0;
    // the same rows in the quad layout of the packed kernels: [nblkq][kQuadRowF2] float2
    float2* d_specq = nullptr;
    int64_t nblkq = 0;
    int64_t specq_lo = 0, specq_hi = 0;   // rows [specq_lo, specq_hi) of d_specq are built (on demand, per batch)
};
