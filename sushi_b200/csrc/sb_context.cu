// Library context: device binding, error text, device memory pool, timers and the
// per-kernel-class accounting used by bench.py's roofline block.
#include "sb_internal.h"
#include <cstdarg>
#include <cstdio>
#include <cstring>

namespace sb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

Ctx& ctx() { static Ctx c; return c; }

int prof_id(const char* name) {
    Ctx& c = ctx();
    for (size_t i = 0; i < c.prof_names.size(); ++i)
        if (c.prof_names[i] == name) return (int)i;
    c.prof_names.emplace_back(name);
    c.prof.emplace_back();
    return (int)c.prof_names.size() - 1;
}

static cudaEvent_t pool_get() {
    Ctx& c = ctx();
    if (!c.event_pool.empty()) { cudaEvent_t e = c.event_pool.back(); c.event_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr; cudaEventCreate(&e); return e;
}

ProfScope::ProfScope(const char* name, int nlaunch) {
    Ctx& c = ctx();
    c.launches += nlaunch;
    id = prof_id(name);
    c.prof[id].launches += nlaunch;
    on = c.prof_on;
    if (on) { a = pool_get(); b = pool_get(); cudaEventRecord(a, c.stream); }
}
ProfScope::~ProfScope() {
    if (!on) return;
    Ctx& c = ctx();
    cudaEventRecord(b, c.stream);
    c.pending.push_back({id, a, b});
    if (c.pending.size() > 8192) prof_collect();
}

int prof_collect() {
    Ctx& c = ctx();
    if (c.pending.empty()) return SB_OK;
    SB_CUDA(cudaStreamSynchronize(c.stream));
    for (auto& p : c.pending) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, p.a, p.b);
        c.prof[p.name_id].ms += ms;
        c.event_pool.push_back(p.a); c.event_pool.push_back(p.b);
    }
    c.pending.clear();
    return SB_OK;
}

namespace {
std::multimap<size_t, void*> g_free_blocks;      // cached, not in use
std::map<void*, size_t> g_live_blocks;           // handed out
size_t g_cached_bytes = 0;
const size_t kMaxCachedBytes = (size_t)24 << 30;
}

int pool_alloc(void** out, size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    auto it = g_free_blocks.find(bytes);
    if (it != g_free_blocks.end()) {
        *out = it->second; g_cached_bytes -= bytes; g_free_blocks.erase(it);
        g_live_blocks[*out] = bytes;
        return SB_OK;
    }
    cudaError_t e = cudaMalloc(out, bytes);
    if (e != cudaSuccess) {                         // give cached blocks back and retry once
        pool_release_all();
        e = cudaMalloc(out, bytes);
    }
    if (e != cudaSuccess) { cudaGetLastError(); SB_FAIL(SB_ENOMEM, "device allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e)); }
    g_live_blocks[*out] = bytes;
    return SB_OK;
}

void pool_free(void* p) {
    if (!p) return;
    auto it = g_live_blocks.find(p);
    if (it == g_live_blocks.end()) { cudaFree(p); return; }
    const size_t bytes = it->second;
    g_live_blocks.erase(it);
    if (g_cached_bytes + bytes > kMaxCachedBytes) { cudaFree(p); return; }
    // blocks are only reused by work enqueued later on the same (single) library stream
    g_free_blocks.emplace(bytes, p); g_cached_bytes += bytes;
}

void pool_release_all() {
    Ctx& c = ctx();
    if (c.stream) cudaStreamSynchronize(c.stream);
    for (auto& kv : g_free_blocks) cudaFree(kv.second);
    g_free_blocks.clear(); g_cached_bytes = 0;
}

}  // namespace sb

using namespace sb;

extern "C" {

int sb_abi_version(void) { return SB_ABI_VERSION; }
const char* sb_last_error(void) { return g_err; }

int sb_init(int device) {
    Ctx& c = ctx();
    if (c.inited) {
        if (c.device == device) return SB_OK;
        SB_FAIL(SB_ESTATE, "sb_init: already bound to device %d", c.device);
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        SB_FAIL(SB_ECUDA, "sb_init: no CUDA device visible (%s) -- this library has no CPU path",
                cudaGetErrorString(e));
    if (device < 0 || device >= ndev) SB_FAIL(SB_EINVAL, "sb_init: device %d out of range [0,%d)", device, ndev);
    SB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    SB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        SB_FAIL(SB_ECUDA, "sb_init: device %d is sm_%d%d; this library is built for sm_90a only",
                device, prop.major, prop.minor);
    c.sm_count = prop.multiProcessorCount;
    SB_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    SB_CUDA(cudaEventCreate(&c.t0));
    SB_CUDA(cudaEventCreate(&c.t1));
    SB_CUDA(cudaEventCreateWithFlags(&c.ev_desc, cudaEventDisableTiming));
    c.device = device;
    c.inited = true;
    g_err[0] = 0;
    return SB_OK;
}

int sb_shutdown(void) {
    Ctx& c = ctx();
    if (!c.inited) return SB_OK;
    cudaStreamSynchronize(c.stream);
    prof_collect();
    pool_release_all();
    fused_release_tables();
    packed_release_tables();
    cudaFree(c.d_parts); cudaFree(c.d_items); cudaFree(c.d_desc); cudaFree(c.d_keys); cudaFree(c.d_groups); cudaFree(c.d_multi);
    cudaFree(c.d_diff); cudaFree(c.d_idx);
    cudaFreeHost(c.h_desc); cudaFreeHost(c.h_diff); cudaFreeHost(c.h_idx);
    for (auto e : c.event_pool) cudaEventDestroy(e);
    cudaEventDestroy(c.t0); cudaEventDestroy(c.t1); cudaEventDestroy(c.ev_desc);
    cudaStreamDestroy(c.stream);
    c = Ctx();
    return SB_OK;
}

int sb_sync(void) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_sync: library not initialised");
    SB_CUDA(cudaStreamSynchronize(c.stream));
    return SB_OK;
}

int sb_set_block_size(int block) {
    if (block != kLagBlock) SB_FAIL(SB_EINVAL, "sb_set_block_size: %d is not %d, the only lag-block size", block, kLagBlock);
    return SB_OK;
}
int sb_get_block_size(void) { return kLagBlock; }
int sb_set_engine(int engine) {
    if (engine < 1 || engine > 5 || engine == 3) SB_FAIL(SB_EINVAL, "sb_set_engine: %d is not one of 1 (fused kernel), 2 (packed fused kernels), 4 / 5 (packed kernel always / never over pairs of lag blocks)", engine);
    ctx().engine = engine;
    return SB_OK;
}
int sb_get_engine(void) { return ctx().engine; }
int sb_set_premac_mode(int mode) {
    if (mode < 0 || mode > 2) SB_FAIL(SB_EINVAL, "sb_set_premac_mode: %d is not 0 (by template length), 1 (never) or 2 (always)", mode);
    ctx().premac_mode = mode;
    return SB_OK;
}
int sb_set_hop_mode(int mode) {
    if (mode != 1) SB_FAIL(SB_EINVAL, "sb_set_hop_mode: %d is not 1 (hop B), the only overlap-save geometry", mode);
    return SB_OK;
}
int sb_set_epilogue(int variant) {
    if (variant != 1 && variant != 3) SB_FAIL(SB_EINVAL, "sb_set_epilogue: %d is not 1 (first version) or 3 (run-level bounds + k_finish_runs, the default); 2 was dropped in round 2", variant);
    ctx().epilogue = variant;
    return SB_OK;
}
int sb_get_epilogue(void) { return ctx().epilogue; }
int sb_set_max_parts(int64_t parts) {
    if (parts < 1) SB_FAIL(SB_EINVAL, "sb_set_max_parts: %lld < 1", (long long)parts);
    ctx().max_parts = parts;
    return SB_OK;
}

void* sb_get_stream(void) { return (void*)ctx().stream; }
int sb_pinned_alloc(int64_t bytes, void** out) {
    if (!ctx().inited) SB_FAIL(SB_ESTATE, "sb_pinned_alloc: library not initialised");
    if (!out || bytes < 1) SB_FAIL(SB_EINVAL, "sb_pinned_alloc: bad argument");
    cudaError_t e = cudaMallocHost(out, (size_t)bytes);
    if (e != cudaSuccess) SB_FAIL(SB_ENOMEM, "sb_pinned_alloc(%lld): %s", (long long)bytes, cudaGetErrorString(e));
    return SB_OK;
}
int sb_pinned_free(void* p) { if (p) cudaFreeHost(p); return SB_OK; }

int sb_device_alloc(int64_t bytes, void** out) {
    if (!ctx().inited) SB_FAIL(SB_ESTATE, "sb_device_alloc: library not initialised");
    if (!out || bytes < 1) SB_FAIL(SB_EINVAL, "sb_device_alloc: bad argument");
    cudaError_t e = cudaMalloc(out, (size_t)bytes);
    if (e != cudaSuccess) SB_FAIL(SB_ENOMEM, "sb_device_alloc(%lld): %s", (long long)bytes, cudaGetErrorString(e));
    return SB_OK;
}
int sb_device_free(void* p) { if (p) cudaFree(p); return SB_OK; }
int sb_copy_to_host(void* host_dst, const void* dev_src, int64_t bytes) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_copy_to_host: library not initialised");
    if (!host_dst || !dev_src || bytes < 0) SB_FAIL(SB_EINVAL, "sb_copy_to_host: bad argument");
    SB_CUDA(cudaMemcpyAsync(host_dst, dev_src, (size_t)bytes, cudaMemcpyDeviceToHost, c.stream));
    SB_CUDA(cudaStreamSynchronize(c.stream));
    return SB_OK;
}

int sb_copy_to_device(void* dev_dst, const void* host_src, int64_t bytes) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_copy_to_device: library not initialised");
    if (!dev_dst || !host_src || bytes < 0) SB_FAIL(SB_EINVAL, "sb_copy_to_device: bad argument");
    SB_CUDA(cudaMemcpyAsync(dev_dst, host_src, (size_t)bytes, cudaMemcpyHostToDevice, c.stream));
    SB_CUDA(cudaStreamSynchronize(c.stream));      // the caller may reuse the host buffer
    return SB_OK;
}
int sb_copy_on_device(void* dev_dst, const void* dev_src, int64_t bytes) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_copy_on_device: library not initialised");
    if (!dev_dst || !dev_src || bytes < 0) SB_FAIL(SB_EINVAL, "sb_copy_on_device: bad argument");
    SB_CUDA(cudaMemcpyAsync(dev_dst, dev_src, (size_t)bytes, cudaMemcpyDeviceToDevice, c.stream));
    return SB_OK;
}

int sb_timer_start(void) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_timer_start: library not initialised");
    SB_CUDA(cudaEventRecord(c.t0, c.stream));
    return SB_OK;
}
int sb_timer_stop(float* ms_out) {
    Ctx& c = ctx();
    if (!c.inited) SB_FAIL(SB_ESTATE, "sb_timer_stop: library not initialised");
    if (!ms_out) SB_FAIL(SB_EINVAL, "sb_timer_stop: NULL output");
    SB_CUDA(cudaEventRecord(c.t1, c.stream));
    SB_CUDA(cudaEventSynchronize(c.t1));
    SB_CUDA(cudaEventElapsedTime(ms_out, c.t0, c.t1));
    return SB_OK;
}

int sb_profile_enable(int on) {
    Ctx& c = ctx();
    if (!on && c.inited) SB_TRY(prof_collect());
    c.prof_on = on != 0;
    return SB_OK;
}
int sb_profile_reset(void) {
    Ctx& c = ctx();
    if (c.inited) SB_TRY(prof_collect());
    for (auto& p : c.prof) p = ProfEntry();
    c.launches = 0;
    return SB_OK;
}
int sb_profile_get(const char* name, double* ms_out, int64_t* launches_out) {
    Ctx& c = ctx();
    if (!name) SB_FAIL(SB_EINVAL, "sb_profile_get: NULL name");
    if (c.inited) SB_TRY(prof_collect());
    for (size_t i = 0; i < c.prof_names.size(); ++i) {
        if (c.prof_names[i] == name) {
            if (ms_out) *ms_out = c.prof[i].ms;
            if (launches_out) *launches_out = c.prof[i].launches;
            return SB_OK;
        }
    }
    if (ms_out) *ms_out = 0.0;
    if (launches_out) *launches_out = 0;
    return SB_OK;
}
const char* sb_profile_names(void) {
    static thread_local std::string s;
    s.clear();
    Ctx& c = ctx();
    for (size_t i = 0; i < c.prof_names.size(); ++i) { if (i) s += ","; s += c.prof_names[i]; }
    return s.c_str();
}
int64_t sb_launch_count(void) { return ctx().launches; }

}  // extern "C"
