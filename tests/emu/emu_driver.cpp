// TEST INFRASTRUCTURE ONLY (see emu_cuda.h).  Compiles the match kernels of sushi_b200/csrc/sb_fused2.cu for the
// host and runs CTAs of them, one OS thread per CUDA thread:
//     g++ -std=c++20 -O1 -pthread -DSB_EMULATE -I tests/emu -I sushi_b200/csrc -I include -I /usr/local/cuda/include
//         -shared -fPIC tests/emu/emu_driver.cpp -o tests/emu/_build/libsb_emu.so
#include "emu_cuda.h"
#include "../../sushi_b200/csrc/sb_fused2.cu"

namespace {
alignas(128) unsigned char smem_raw[232 * 1024];      // the kernels' `extern __shared__` array
std::vector<float4> g_park(kParkF4);                  // k_match_pair's park: one slot (CTAs run one after the other)
int g_park_busy = 0;
}

// ---- running the 512 threads of a CTA ---------------------------------------------------------------------
#ifdef SB_EMU_THREADS
namespace emu {
void run_cta(const std::function<void(int)>& body) {
    std::vector<std::thread> th;
    th.reserve(kThreads);
    for (int t = 0; t < kThreads; ++t)
        th.emplace_back([&body, t] { threadIdx = {(unsigned)t, 0, 0}; t_lane = t & 31; t_warp = t >> 5; body(t); });
    for (auto& x : th) x.join();
}
}  // namespace emu
#else
#include <ucontext.h>
namespace emu {
namespace {
constexpr size_t kStack = 512 * 1024;
struct WarpRun {
    ucontext_t sched;
    ucontext_t lane[32];
    bool done[32];
    int cur = 0, warp = 0;
    const std::function<void(int)>* body = nullptr;
    std::vector<char> stacks;
};
thread_local WarpRun* t_run = nullptr;
void lane_entry() {
    WarpRun* r = t_run;
    (*r->body)(r->warp * 32 + r->cur);
    r->done[r->cur] = true;            // returning resumes uc_link = the scheduler
}
}  // namespace
void yield_lane() {
    WarpRun* r = t_run;
    swapcontext(&r->lane[r->cur], &r->sched);
}
void run_cta(const std::function<void(int)>& body) {
    std::vector<std::thread> th;
    th.reserve(kWarps);
    for (int w = 0; w < kWarps; ++w)
        th.emplace_back([&body, w] {
            WarpRun r;
            r.warp = w; r.body = &body;
            r.stacks.resize(32 * kStack);
            t_run = &r;
            t_warp = w;
            for (int l = 0; l < 32; ++l) {
                r.done[l] = false;
                getcontext(&r.lane[l]);
                r.lane[l].uc_stack.ss_sp = r.stacks.data() + (size_t)l * kStack;
                r.lane[l].uc_stack.ss_size = kStack;
                r.lane[l].uc_link = &r.sched;
                makecontext(&r.lane[l], lane_entry, 0);
            }
            for (int left = 32; left > 0;) {
                left = 0;
                for (int l = 0; l < 32; ++l) {
                    if (r.done[l]) continue;
                    r.cur = l; t_lane = l;
                    threadIdx = {(unsigned)(w * 32 + l), 0, 0};
                    swapcontext(&r.sched, &r.lane[l]);
                    if (!r.done[l]) ++left;
                }
            }
            t_run = nullptr;
        });
    for (auto& x : th) x.join();
}
}  // namespace emu
#endif

namespace { int g_pair_grid = 0; }

extern "C" {

void emu_set_pair_grid(int g) { g_pair_grid = g; }
int emu_table_floats(void) { size_t off[kPackedTableCount]; return (int)packed_table_values(off).size(); }
int emu_smem_bytes(void) { return (int)packed_smem_bytes(3) + 16; }
int emu_query_desc_bytes(void) { return (int)sizeof(sb::QueryDesc); }
int emu_quad_row_floats(void) { return QROW * 4; }

// kernel: 0 = k_match_packed (one CTA per lag block), 1 = k_match_pair; epi: 1 | 2; is_u8: sample type of img.
// Runs CTAs [0, n_ctas) one after the other.  Returns 0, or the number of emulation errors (messages on stderr).
int emu_run(int kernel, int epi, int is_u8, const float* That, int64_t part_first, const float* Xhat, int64_t nblk,
            const void* img, int64_t img_n, const double* ipfx, const double* tpfx, const void* desc,
            const int* cta_query, int64_t first, int n_ctas, unsigned long long* keys, float* curve_out,
            void* run_recs, int* run_count) {
    static size_t off[kPackedTableCount];
    static const std::vector<float> tables = packed_table_values(off);
    const PackedTables tab = packed_tables_at(tables.data(), off);
    const float4* T4 = reinterpret_cast<const float4*>(That);
    const float4* X4 = reinterpret_cast<const float4*>(Xhat);
    const double2* ip = reinterpret_cast<const double2*>(ipfx);
    const double2* tp = reinterpret_cast<const double2*>(tpfx);
    const sb::QueryDesc* d = static_cast<const sb::QueryDesc*>(desc);
    int n_err = 0;
    // k_match_pair<uint8, 3> is persistent (a CTA walks the pairs b, b + grid, ...): g_pair_grid > 0 runs it with that many CTAs
    const int grid = (kernel == 1 && is_u8 && epi == 3 && g_pair_grid > 0 && g_pair_grid < n_ctas) ? g_pair_grid : n_ctas;   // like the launcher: body 3 only
    gridDim = dim3((unsigned)grid, 1, 1);
    for (int b = 0; b < grid; ++b) {
        emu::Cta cta;
        emu::cta() = &cta;
        std::memset(smem_raw, 0xCD, sizeof(smem_raw));                      // uninitialised reads show up as garbage
        for (auto& v : g_park) v = make_float4(std::nanf(""), std::nanf(""), std::nanf(""), std::nanf(""));
        auto body = [&](int t) {
            blockIdx = {(unsigned)b, 0, 0};       // threadIdx and the lane / warp numbers are set by run_cta
#define SB_EMU_ARGS(S) T4, part_first, X4, nblk, static_cast<const S*>(img), img_n, ip, tp, d, cta_query, first
#define SB_EMU_CALL(K, S, E, ...) K<S, E>(SB_EMU_ARGS(S), ##__VA_ARGS__, tab, keys, curve_out, static_cast<RunRecord*>(run_recs), run_count)
#define SB_EMU_KERNEL(K, ...) do { if (!is_u8) SB_EMU_CALL(K, float, 1, ##__VA_ARGS__); else if (epi == 3) SB_EMU_CALL(K, uint8_t, 3, ##__VA_ARGS__); \
                                   else SB_EMU_CALL(K, uint8_t, 1, ##__VA_ARGS__); } while (0)
            if (kernel == 0) SB_EMU_KERNEL(k_match_packed);
            else SB_EMU_KERNEL(k_match_pair, (int64_t)n_ctas, g_park.data(), &g_park_busy, 1);
        };
        emu::run_cta(body);
        if (g_park_busy) { cta.fail("the park slot was not released"); g_park_busy = 0; }
        for (const auto& e : cta.errors) { std::fprintf(stderr, "[emu] CTA %d: %s\n", b, e.c_str()); ++n_err; }
        emu::cta() = nullptr;
        // nothing may be written behind the dynamic shared memory the launchers ask for (the array here is larger)
        const size_t limit = packed_smem_bytes(is_u8 ? epi : 1) + (kernel == 1 ? 16 : 0);
        for (size_t k = limit; k < sizeof(smem_raw); ++k)
            if (smem_raw[k] != 0xCD) {
                std::fprintf(stderr, "[emu] CTA %d wrote shared memory at byte %zu, behind the %zu bytes its launcher allocates\n", b, k, limit);
                ++n_err;
                break;
            }
    }
    return n_err;
}

// The second step of the third kernel body (k_finish_runs, uint8 streams): every record slot of CTAs [0, n_ctas).
int emu_finish_runs(const void* run_recs, const int* run_count, int n_ctas, const void* desc, const double* ipfx, int64_t img_n,
                    const double* tpfx, unsigned long long* keys) {
    const int64_t threads = (int64_t)n_ctas * kRunSlots;
    blockDim = dim3(128, 1, 1);
    for (int64_t t = 0; t < threads; ++t) {
        blockIdx = {(unsigned)(t / 128), 0, 0};
        threadIdx = {(unsigned)(t % 128), 0, 0};
        k_finish_runs<uint8_t>(static_cast<const RunRecord*>(run_recs), run_count, n_ctas, static_cast<const sb::QueryDesc*>(desc),
                               reinterpret_cast<const double2*>(ipfx), img_n, reinterpret_cast<const double2*>(tpfx), keys);
    }
    blockDim = dim3(emu::kThreads, 1, 1);
    return 0;
}
int emu_run_slots(void) { return kRunSlots; }
int emu_run_record_bytes(void) { return (int)sizeof(RunRecord); }

// Block spectra of a stream (k_forward_quad, MODE 0): rows [row_first, row_first + rows) into
// `out` (rows * emu_quad_row_floats() floats).  The twiddle tables are the ones sb_fused.cu's ensure_tables
// builds.
int emu_forward_blocks(int is_u8, const void* src, int64_t src_n, const double* pfx, int64_t row_first, int rows, float* out) {
    typedef Cfg<14> C;
    static std::vector<float2> h;
    static FusedTables tab;
    if (h.empty()) {
        const int N = C::N;
        const size_t nw = N / 2 + 1, n2 = (size_t)C::R2 * 32, n3 = (size_t)C::R3 * 32;
        h.resize(nw + n2 + 2 * n3);
        const double pi = 3.14159265358979323846;
        for (size_t m = 0; m < nw; ++m) h[m] = make_float2((float)cos(pi * m / N), (float)sin(pi * m / N));
        for (int r = 0; r < C::R2; ++r)
            for (int k = 0; k < 32; ++k) {
                const double ang = 2.0 * pi * r * k / (32.0 * C::R2);
                h[nw + r * 32 + k] = make_float2((float)cos(ang), (float)sin(ang));
            }
        for (int r = 0; r < C::R3; ++r)
            for (int k = 0; k < 32; ++k) {
                const double al = 2.0 * pi * r * k / N, ah = 2.0 * pi * r * (k * 32.0) / N;
                h[nw + n2 + r * 32 + k] = make_float2((float)cos(al), (float)sin(al));
                h[nw + n2 + n3 + r * 32 + k] = make_float2((float)cos(ah), (float)sin(ah));
            }
        tab.w = h.data(); tab.t2 = h.data() + nw; tab.a3 = h.data() + nw + n2; tab.b3 = h.data() + nw + n2 + n3;
    }
    const double2* pf = reinterpret_cast<const double2*>(pfx);
    float4* o4 = reinterpret_cast<float4*>(out);
    int n_err = 0;
    for (int b = 0; b < rows; ++b) {
        emu::Cta cta;
        emu::cta() = &cta;
        std::memset(smem_raw, 0xCD, sizeof(smem_raw));
        auto body = [&](int t) {
            blockIdx = {(unsigned)b, 0, 0};       // threadIdx and the lane / warp numbers are set by run_cta
            if (is_u8) k_forward_quad<uint8_t, 0>(static_cast<const uint8_t*>(src), src_n, pf, nullptr, 0, 0, row_first, tab, o4);
            else       k_forward_quad<float, 0>(static_cast<const float*>(src), src_n, pf, nullptr, 0, 0, row_first, tab, o4);
        };
        emu::run_cta(body);
        for (const auto& e : cta.errors) { std::fprintf(stderr, "[emu] forward CTA %d: %s\n", b, e.c_str()); ++n_err; }
        emu::cta() = nullptr;
    }
    return n_err;
}

}  // extern "C"

#ifdef SB_EMU_DEBUG      // g++ ... -DSB_EMU_DEBUG -g -rdynamic: backtrace of the faulting thread on SIGSEGV
#include <execinfo.h>
#include <signal.h>
#include <unistd.h>
namespace {
void on_segv(int) { void* bt[48]; const int n = backtrace(bt, 48); backtrace_symbols_fd(bt, n, 2); _exit(139); }
struct InstallSegv { InstallSegv() { signal(SIGSEGV, on_segv); } } install_segv;
}
#endif
