// TEST INFRASTRUCTURE ONLY (see emu_cuda.h).  The multi-stream instantiations of the packed kernels (MULTI = true:
// every query reads its image and template stream from a per-call stream table) on the host, next to everything
// emu_driver.cpp offers:
//     g++ -std=c++20 -O1 -pthread -DSB_EMULATE -I tests/emu -I sushi_b200/csrc -I include -I /usr/local/cuda/include
//         -shared -fPIC tests/emu/emu_multi_driver.cpp -o tests/emu/_build/libsb_emu_multi.so
#include "emu_driver.cpp"

extern "C" {

int emu_stream_entry_bytes(void) { return (int)sizeof(sb::StreamEntry); }

// As emu_run, but the image / template arguments come from `streams` (StreamEntry[]) through `slots` (int2 per query:
// image slot, template slot).
int emu_run_multi(int kernel, int epi, int is_u8, const float* That, const void* streams, const int* slots, const void* desc,
                  const int* cta_query, int n_ctas, unsigned long long* keys, float* curve_out, void* run_recs, int* run_count) {
    static size_t off[kPackedTableCount];
    static const std::vector<float> tables = packed_table_values(off);
    const PackedTables tab = packed_tables_at(tables.data(), off);
    const float4* T4 = reinterpret_cast<const float4*>(That);
    const sb::StreamEntry* st = static_cast<const sb::StreamEntry*>(streams);
    const int2* sl = reinterpret_cast<const int2*>(slots);
    const sb::QueryDesc* d = static_cast<const sb::QueryDesc*>(desc);
    int n_err = 0;
    const int grid = (kernel == 1 && is_u8 && epi == 3 && g_pair_grid > 0 && g_pair_grid < n_ctas) ? g_pair_grid : n_ctas;
    gridDim = dim3((unsigned)grid, 1, 1);
    for (int b = 0; b < grid; ++b) {
        emu::Cta cta;
        emu::cta() = &cta;
        std::memset(smem_raw, 0xCD, sizeof(smem_raw));
        for (auto& v : g_park) v = make_float4(std::nanf(""), std::nanf(""), std::nanf(""), std::nanf(""));
        auto body = [&](int t) {
            blockIdx = {(unsigned)b, 0, 0};
#define SB_EMU_MARGS(S) T4, (int64_t)0, nullptr, (int64_t)0, static_cast<const S*>(nullptr), (int64_t)0, nullptr, nullptr, d, cta_query, (int64_t)0
#define SB_EMU_MCALL(K, S, E, ...) K<S, E, true>(SB_EMU_MARGS(S), ##__VA_ARGS__, tab, keys, curve_out, static_cast<RunRecord*>(run_recs), run_count, st, sl)
#define SB_EMU_MKERNEL(K, ...) do { if (!is_u8) SB_EMU_MCALL(K, float, 1, ##__VA_ARGS__); else if (epi == 3) SB_EMU_MCALL(K, uint8_t, 3, ##__VA_ARGS__); \
                                    else SB_EMU_MCALL(K, uint8_t, 1, ##__VA_ARGS__); } while (0)
            if (kernel == 0) SB_EMU_MKERNEL(k_match_packed);
            else SB_EMU_MKERNEL(k_match_pair, (int64_t)n_ctas, g_park.data(), &g_park_busy, 1);
        };
        emu::run_cta(body);
        if (g_park_busy) { cta.fail("the park slot was not released"); g_park_busy = 0; }
        for (const auto& e : cta.errors) { std::fprintf(stderr, "[emu] CTA %d: %s\n", b, e.c_str()); ++n_err; }
        emu::cta() = nullptr;
    }
    return n_err;
}

int emu_finish_runs_multi(const void* run_recs, const int* run_count, int n_ctas, const void* desc, const void* streams,
                          const int* slots, unsigned long long* keys) {
    const int64_t threads = (int64_t)n_ctas * kRunSlots;
    blockDim = dim3(128, 1, 1);
    for (int64_t t = 0; t < threads; ++t) {
        blockIdx = {(unsigned)(t / 128), 0, 0};
        threadIdx = {(unsigned)(t % 128), 0, 0};
        k_finish_runs<uint8_t, true>(static_cast<const RunRecord*>(run_recs), run_count, n_ctas, static_cast<const sb::QueryDesc*>(desc),
                                     nullptr, 0, nullptr, keys, static_cast<const sb::StreamEntry*>(streams),
                                     reinterpret_cast<const int2*>(slots));
    }
    blockDim = dim3(emu::kThreads, 1, 1);
    return 0;
}

// Block spectra of several uint8 streams in one launch (k_forward_quad, MODE 0, MULTI): row_list[i] = (slot, row), each
// row written into its own stream's specq.  The twiddle tables are the ones emu_forward_blocks builds.
int emu_forward_blocks_multi(const void* streams, const int* row_list, int n_rows) {
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
    int n_err = 0;
    for (int b = 0; b < n_rows; ++b) {
        emu::Cta cta;
        emu::cta() = &cta;
        std::memset(smem_raw, 0xCD, sizeof(smem_raw));
        auto body = [&](int t) {
            blockIdx = {(unsigned)b, 0, 0};
            k_forward_quad<uint8_t, 0, true>(nullptr, 0, nullptr, nullptr, 0, 0, 0, tab, nullptr,
                                             static_cast<const sb::StreamEntry*>(streams), nullptr,
                                             reinterpret_cast<const int2*>(row_list));
        };
        emu::run_cta(body);
        for (const auto& e : cta.errors) { std::fprintf(stderr, "[emu] forward CTA %d: %s\n", b, e.c_str()); ++n_err; }
        emu::cta() = nullptr;
    }
    return n_err;
}

}  // extern "C"
