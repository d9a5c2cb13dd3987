// row_plan.hpp -- the Hilbert row plan (d4w_row_plan_create, d4w_rows.cu), shared with the translation units that run
// their own kernels on it (d4w_noise.cu).
#pragma once
#include "fk_kernels.cuh"

struct d4w_row_plan {
    int ns = 0, device = 0, t1 = 1, t2 = 0;
    d4w::RowParams row{};
    float2 *d_tw = nullptr, *d_twT = nullptr;
    float* d_hilbert = nullptr;
    float* d_sgn = nullptr;      // sgn(f)/ns in k_row_mid_fused's table order (two-rows-per-transform route)
    size_t row_smem = 0;
    int fused = 0;               // split rows: middle pass by k_row_mid_fused (weights stored in its table order)
    // chirp-z rows (no mixed-radix split of ns): t1 x t2 = czt_m is the convolution length, hilbert_czt.cuh
    int czt_m = 0, pair = 0;
    float2 *d_chirp = nullptr, *d_bhat = nullptr, *d_bhatc = nullptr;
};
