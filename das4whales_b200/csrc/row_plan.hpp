// row_plan.hpp -- the Hilbert row plan (d4w_row_plan_create, d4w_rows.cu), shared with the translation units that run
// their own kernels on it (d4w_noise.cu), and the dispatch over the split radices its kernels are built for.
#pragma once
#include <type_traits>
#include "../../include/d4w.h"
#include "fk_kernels.cuh"

struct d4w_row_plan {
    int ns = 0, device = 0, t1 = 1, t2 = 0;
    d4w::RowParams row{};
    float2 *d_tw = nullptr, *d_twT = nullptr;
    float* d_hilbert = nullptr;
    float* d_sgn = nullptr;      // sgn(f)/ns in the middle pass's table order (split rows: two real rows per transform)
    size_t row_smem = 0;
    int fused = 0;               // split rows: middle pass by k_row_mid_fused (weights stored in its table order)
    int pair = 0;                // t1 > 1: two real rows per complex transform
    // chirp-z rows (no mixed-radix split of ns): t1 x t2 = czt_m is the convolution length, hilbert_czt.cuh
    int czt_m = 0;
    float2 *d_chirp = nullptr, *d_bhat = nullptr, *d_bhatc = nullptr;
};

namespace d4w {

// f(std::integral_constant<int, T1>{}) for the split radices T1 the row kernels are instantiated for; D4W_ERR_UNSUPPORTED
// for any other t1
template <class F>
int with_t1(int t1, F&& f) {
    switch (t1) {
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 5: return f(std::integral_constant<int, 5>{});
        case 6: return f(std::integral_constant<int, 6>{});
        case 8: return f(std::integral_constant<int, 8>{});
        case 10: return f(std::integral_constant<int, 10>{});
        case 12: return f(std::integral_constant<int, 12>{});
        case 15: return f(std::integral_constant<int, 15>{});
        case 16: return f(std::integral_constant<int, 16>{});
        case 20: return f(std::integral_constant<int, 20>{});
        case 25: return f(std::integral_constant<int, 25>{});
        default: return D4W_ERR_UNSUPPORTED;
    }
}

}  // namespace d4w
