// d4w_mask_design.cu -- host side of the hybrid, hybrid_gs and hybrid_ninf_gs f-k masks designed on the device (C ABI in
// include/d4w.h; bodies in tools_kernels.cuh).  A translation unit of its own, so that d4w_tools.cu's kernels compile as
// before.  The plane goes to d4w_fk_mask_create_dense like any dense mask.
#include <cmath>
#include <string>
#include "d4w_common.hpp"
#include "tools_kernels.cuh"

using namespace d4w;

namespace {

constexpr int kHybThreads = 256;

// the weights and running sums (one thread, deterministic), and the interval list of every row
__global__ void k_design_rows(DesignParams p, double* w, double* cw) {
    if (blockIdx.x == 0 && threadIdx.x == 0) fan_weights(kDesignSigma, p.r, w, cw);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.nx) body_design_row(p, i);
}

// the fan's tile: exact axis-1 blur of the interval lists, then the 2r + 1 axis-0 taps; no normalisation
__global__ void __launch_bounds__(kFanThreads, 2)
k_design_blur(DesignParams p, float* out) {
    extern __shared__ double sm[];
    double* wz = sm;
    double* cw = wz + fan_steps(p.r);
    double* H = cw + 2 * p.r + 2;
    const int i0 = blockIdx.y * kFanRT, j0 = blockIdx.x * kFanTJ;
    body_fan_weights(p, wz, cw, threadIdx.x, kFanThreads);
    __syncthreads();
    body_fan_fill_tile(p, i0, j0, cw, H, threadIdx.x, kFanThreads);
    __syncthreads();
    const int lane = threadIdx.x % kFanTJ, g = threadIdx.x / kFanTJ, j = j0 + lane;
    double acc[kFanU];
    body_fan_taps(p, wz, H, g, lane, acc);
    if (j >= p.ns) return;
    const int ib = i0 + g * kFanU;
#pragma unroll
    for (int u = 0; u < kFanU; ++u)
        if (ib + u < p.nx) out[(size_t)(ib + u) * p.ns + j] = (float)acc[u];
}

// grid (column blocks, rows): one element per thread
__global__ void __launch_bounds__(kHybThreads)
k_design_hybrid(DesignParams p, float* out) {
    const int i = blockIdx.y, j = blockIdx.x * kHybThreads + threadIdx.x;
    if (j < p.ns) out[(size_t)i * p.ns + j] = (float)body_hybrid(p, i, j);
}

bool positive_finite(double c) { return c > 0.0 && std::isfinite(c); }

}  // namespace

extern "C" size_t d4w_mask_design_workspace_bytes(int nx, int ns) {
    if (nx < 1 || ns < 1) return 0;
    return design_ws_bytes(nx, ns, fan_radius(kDesignSigma));
}

extern "C" int d4w_mask_design(int kind, float* out, int nx, int ns, double kval, double fval, double cs_min, double cp_min,
                               double cp_max, double fmin, double fmax, int col_lo, int col_hi, const double* host_H, void* ws,
                               void* stream_v) {
    if (!out || !ws || !host_H) return fail(D4W_ERR_ARG, "d4w_mask_design: null pointer");
    if (kind != kDesignHybrid && kind != kDesignHybridGs && kind != kDesignHybridNinfGs)
        return fail(D4W_ERR_ARG, "d4w_mask_design: kind must be 0 (hybrid), 1 (hybrid_gs) or 2 (hybrid_ninf_gs)");
    if (nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_mask_design: nx and ns must be >= 1");
    if (!positive_finite(fval) || !std::isfinite(kval))
        return fail(D4W_ERR_ARG, "d4w_mask_design: fval must be finite and > 0, kval finite");
    if (!positive_finite(cs_min) || !positive_finite(cp_min) || !positive_finite(cp_max))
        return fail(D4W_ERR_ARG, "d4w_mask_design: the speeds must be finite and > 0");
    if (!std::isfinite(fmin) || !std::isfinite(fmax) || !(fmin < fmax))
        return fail(D4W_ERR_ARG, "d4w_mask_design: need finite fmin < fmax");
    if (col_lo < 0 || col_lo > ns || col_hi < 0 || col_hi > ns)
        return fail(D4W_ERR_ARG, "d4w_mask_design: col_lo and col_hi must lie in [0, ns]");
    if (kind == kDesignHybrid && col_hi < col_lo) return fail(D4W_ERR_ARG, "d4w_mask_design: hybrid needs col_lo <= col_hi");
    int h_lo = ns, h_hi = ns;
    if (kind != kDesignHybrid && !design_h_band(host_H, ns, &h_lo, &h_hi))
        return fail(D4W_ERR_ARG, "d4w_mask_design: H of a gs mask must be 1 on one band of columns and 0 elsewhere");
    const int r = fan_radius(kDesignSigma);
    if ((nx + kFanRT - 1) / kFanRT > 65535 || nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_mask_design: more than 65 535 rows");
    cudaStream_t st = (cudaStream_t)stream_v;
    double* w = static_cast<double*>(ws);
    double* cw = w + 2 * r + 1;
    double* H = cw + 2 * r + 2;
    int* iv = reinterpret_cast<int*>(H + ns);
    DesignParams p{kind, nx, ns, r, kval, fval, cs_min, cp_min, cp_max, col_lo, col_hi, h_lo, h_hi, H, w, cw, iv};
    if (kind == kDesignHybrid) {
        D4W_CUDA_TRY(cudaMemcpyAsync(H, host_H, sizeof(double) * (size_t)ns, cudaMemcpyHostToDevice, st));
        k_design_hybrid<<<dim3((unsigned)((ns + kHybThreads - 1) / kHybThreads), (unsigned)nx), kHybThreads, 0, st>>>(p, out);
        D4W_CHECK_LAUNCH("k_design_hybrid");
        return D4W_OK;
    }
    k_design_rows<<<(unsigned)((nx + 255) / 256), 256, 0, st>>>(p, w, cw);
    D4W_CHECK_LAUNCH("k_design_rows");
    const size_t smem = fan_smem_bytes(r);
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_design_blur, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((unsigned)((ns + kFanTJ - 1) / kFanTJ), (unsigned)((nx + kFanRT - 1) / kFanRT));
    k_design_blur<<<grid, kFanThreads, smem, st>>>(p, out);
    D4W_CHECK_LAUNCH("k_design_blur");
    return D4W_OK;
}
