// TEST INFRASTRUCTURE ONLY (see emu_cuda.h).  The persistent walk of k_forward_quad on the host: a launch of `grid` CTAs,
// each walking the rows b, b + grid, ..., next to everything emu_driver.cpp and emu_multi_driver.cpp offer (whose
// forward entry points launch one CTA per row):
//     g++ -std=c++20 -O1 -pthread -DSB_EMULATE -I tests/emu -I sushi_b200/csrc -I include -I /usr/local/cuda/include
//         -shared -fPIC tests/emu/emu_forward_driver.cpp -o tests/emu/_build/libsb_emu_forward.so
#include "emu_multi_driver.cpp"

namespace {
// The twiddle tables sb_fused.cu's ensure_tables builds (the same values as emu_forward_blocks)
const FusedTables& walk_tables() {
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
    return tab;
}

// A launch of k_forward_quad over `rows` rows with `grid` CTAs (grid <= 0: one CTA per row, rows argument -1 as the
// kernel's default); call(tab, rows_arg) is one thread's kernel call
template <typename Call>
int run_walk(int grid, int64_t rows, const Call& call) {
    const FusedTables& tab = walk_tables();
    const int64_t rows_arg = grid > 0 ? rows : -1;
    if (grid <= 0 || grid > rows) grid = (int)rows;
    gridDim = dim3((unsigned)grid, 1, 1);
    int n_err = 0;
    for (int b = 0; b < grid; ++b) {
        emu::Cta cta;
        emu::cta() = &cta;
        std::memset(smem_raw, 0xCD, sizeof(smem_raw));
        auto body = [&](int t) {
            blockIdx = {(unsigned)b, 0, 0};       // threadIdx and the lane / warp numbers are set by run_cta
            call(tab, rows_arg);
        };
        emu::run_cta(body);
        for (const auto& e : cta.errors) { std::fprintf(stderr, "[emu] forward CTA %d: %s\n", b, e.c_str()); ++n_err; }
        emu::cta() = nullptr;
        // nothing may be written behind the dynamic shared memory the launcher asks for (the array here is larger)
        const size_t limit = forward_smem_bytes14();
        for (size_t k = limit; k < sizeof(smem_raw); ++k)
            if (smem_raw[k] != 0xCD) {
                std::fprintf(stderr, "[emu] forward CTA %d wrote shared memory at byte %zu, behind the %zu bytes its launcher allocates\n", b, k, limit);
                ++n_err;
                break;
            }
    }
    return n_err;
}
}  // namespace

extern "C" {

// Block spectra of a stream (MODE 0): rows [row_first, row_first + rows) into `out`
int emu_walk_blocks(int grid, int is_u8, const void* src, int64_t src_n, const double* pfx, int64_t row_first, int rows, float* out) {
    const double2* pf = reinterpret_cast<const double2*>(pfx);
    float4* o4 = reinterpret_cast<float4*>(out);
    return run_walk(grid, rows, [&](const FusedTables& tab, int64_t n) {
        if (is_u8) k_forward_quad<uint8_t, 0>(static_cast<const uint8_t*>(src), src_n, pf, nullptr, 0, 0, row_first, tab, o4, nullptr, nullptr, nullptr, n);
        else       k_forward_quad<float, 0>(static_cast<const float*>(src), src_n, pf, nullptr, 0, 0, row_first, tab, o4, nullptr, nullptr, nullptr, n);
    });
}

// Partition spectra of the templates of queries [q_begin, q_end) (MODE 1): rows [part_first, part_first + rows) of the
// partitions the descriptors number (partBase), into `out`
int emu_walk_parts(int grid, int is_u8, const void* src, int64_t src_n, const double* pfx, const void* desc, int q_begin, int q_end,
                   int64_t part_first, int rows, float* out) {
    const double2* pf = reinterpret_cast<const double2*>(pfx);
    const sb::QueryDesc* d = static_cast<const sb::QueryDesc*>(desc);
    float4* o4 = reinterpret_cast<float4*>(out);
    return run_walk(grid, rows, [&](const FusedTables& tab, int64_t n) {
        if (is_u8) k_forward_quad<uint8_t, 1>(static_cast<const uint8_t*>(src), src_n, pf, d, q_begin, q_end, part_first, tab, o4, nullptr, nullptr, nullptr, n);
        else       k_forward_quad<float, 1>(static_cast<const float*>(src), src_n, pf, d, q_begin, q_end, part_first, tab, o4, nullptr, nullptr, nullptr, n);
    });
}

// Block spectra of several uint8 streams in one launch (MODE 0, MULTI): row_list[i] = (slot, row)
int emu_walk_blocks_multi(int grid, const void* streams, const int* row_list, int n_rows) {
    return run_walk(grid, n_rows, [&](const FusedTables& tab, int64_t n) {
        k_forward_quad<uint8_t, 0, true>(nullptr, 0, nullptr, nullptr, 0, 0, 0, tab, nullptr, static_cast<const sb::StreamEntry*>(streams),
                                         nullptr, reinterpret_cast<const int2*>(row_list), n);
    });
}

// Partition spectra of uint8 templates that live in several streams (MODE 1, MULTI): query q reads stream slots[q].y
int emu_walk_parts_multi(int grid, const void* streams, const int* slots, const void* desc, int q_begin, int q_end,
                         int64_t part_first, int rows, float* out) {
    const sb::QueryDesc* d = static_cast<const sb::QueryDesc*>(desc);
    float4* o4 = reinterpret_cast<float4*>(out);
    return run_walk(grid, rows, [&](const FusedTables& tab, int64_t n) {
        k_forward_quad<uint8_t, 1, true>(nullptr, 0, nullptr, d, q_begin, q_end, part_first, tab, o4, static_cast<const sb::StreamEntry*>(streams),
                                         reinterpret_cast<const int2*>(slots), nullptr, n);
    });
}

}  // extern "C"
