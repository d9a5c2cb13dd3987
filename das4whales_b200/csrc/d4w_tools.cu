// d4w_tools.cu -- host side of the reference's tools module kernels (C ABI in include/d4w.h; bodies in tools_kernels.cuh):
// the Gaussian-blurred f-k fan designed on the device, and the per-row moments / linear detrend of a time block.
#include <string>
#include "d4w_common.hpp"
#include "tools_kernels.cuh"

using namespace d4w;

namespace {

constexpr int kMomThreads = 256;

// one CTA: the weights and running sums (sequential, deterministic), and the row prefixes of every CTA
__global__ void k_fan_rows(FanParams p, double sigma, double* w, double* cw, int* J) {
    if (blockIdx.x == 0 && threadIdx.x == 0) fan_weights(sigma, p.r, w, cw);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.nx) body_fan_row(p.nx, p.ns, p.kval, p.fval, p.c_min, p.c_max, J, i);
}

// pass 0: global min / max of the blurred fan into keys[0..1]; pass 1: (g - min) / (max - min) as float32 into out
__global__ void __launch_bounds__(kFanThreads, 2)
k_fan_blur(FanParams p, int pass, unsigned long long* keys, float* out) {
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
    const int ib = i0 + g * kFanU;
    if (pass == 0) {
        double mn = INFINITY, mx = -INFINITY;
#pragma unroll
        for (int u = 0; u < kFanU; ++u)
            if (j < p.ns && ib + u < p.nx) { mn = fmin(mn, acc[u]); mx = fmax(mx, acc[u]); }
        for (int o = 16; o > 0; o >>= 1) {
            mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if (lane == 0 && mn <= mx) {
            atomicMin(keys, fan_key(mn));
            atomicMax(keys + 1, fan_key(mx));
        }
        return;
    }
    if (j >= p.ns) return;
    const double mn = fan_unkey(keys[0]), span = fan_unkey(keys[1]) - mn;
#pragma unroll
    for (int u = 0; u < kFanU; ++u)
        if (ib + u < p.nx) out[(size_t)(ib + u) * p.ns + j] = (float)((acc[u] - mn) / span);
}

__device__ inline double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x / 32, nw = blockDim.x / 32;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    for (int k = 0; k < nw; ++k) s += red[k];    // fixed order: runs are bit-identical
    return s;
}

// CTA b: row b / nchunks, chunk b % nchunks
__global__ void __launch_bounds__(kMomThreads)
k_row_moments(const float* x, size_t ld, int n, int chunk, int nchunks, double* out) {
    __shared__ double red[kMomThreads / 32];
    const long long b = blockIdx.x;
    const long long row = b / nchunks, c = b % nchunks;
    const int c0 = (int)c * chunk, len = min(chunk, n - c0);
    double s[3];
    body_moments(x + row * ld + c0, len, threadIdx.x, kMomThreads, s);
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const double t = block_sum(s[q], red);
        if (threadIdx.x == 0) out[b * 3 + q] = t;
    }
}

__global__ void k_detrend(const float* x, size_t ld, int nrows, int n, const double* mom, float* y) {
    const int row = blockIdx.y;
    const double* m = mom + (size_t)row * 3;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x)
        y[(size_t)row * n + t] = detrend_sample(x[row * ld + t], t, n, m);
}

}  // namespace

extern "C" size_t d4w_fan_blur_workspace_bytes(int nx, double sigma) {
    if (nx < 1 || !(sigma > 0.0) || !(sigma < 1e6)) return 0;
    return fan_ws_bytes(nx, fan_radius(sigma));
}

extern "C" int d4w_fan_blur(float* out, int nx, int ns, double kval, double fval, double c_min, double c_max, double sigma,
                            void* ws, void* stream_v) {
    if (!out || !ws) return fail(D4W_ERR_ARG, "d4w_fan_blur: null pointer");
    if (nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_fan_blur: nx and ns must be >= 1");
    if (!(fval > 0.0) || !std::isfinite(fval) || !std::isfinite(kval))
        return fail(D4W_ERR_ARG, "d4w_fan_blur: fval must be finite and > 0, kval finite");
    if (!(sigma > 0.0) || !(sigma < 1e6)) return fail(D4W_ERR_ARG, "d4w_fan_blur: sigma must be > 0");
    const int r = fan_radius(sigma);
    const size_t smem = fan_smem_bytes(r);
    if (smem > 227 * 1024)
        return fail(D4W_ERR_UNSUPPORTED, "d4w_fan_blur: sigma = " + std::to_string(sigma) + " needs a " + std::to_string(smem) +
                    "-byte tile, more than an SM's 227 KB of shared memory");
    if ((nx + kFanRT - 1) / kFanRT > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_fan_blur: too many rows");
    cudaStream_t st = (cudaStream_t)stream_v;
    unsigned long long* keys = static_cast<unsigned long long*>(ws);
    double* w = reinterpret_cast<double*>(static_cast<char*>(ws) + 16);
    double* cw = w + 2 * r + 1;
    int* J = reinterpret_cast<int*>(cw + 2 * r + 2);
    FanParams p{nx, ns, r, kval, fval, c_min, c_max, w, cw, J};
    D4W_CUDA_TRY(cudaMemsetAsync(keys, 0xff, 8, st));
    D4W_CUDA_TRY(cudaMemsetAsync(keys + 1, 0, 8, st));
    k_fan_rows<<<(unsigned)((nx + 255) / 256), 256, 0, st>>>(p, sigma, w, cw, J);
    D4W_CHECK_LAUNCH("k_fan_rows");
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_fan_blur, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((unsigned)((ns + kFanTJ - 1) / kFanTJ), (unsigned)((nx + kFanRT - 1) / kFanRT));
    for (int pass = 0; pass < 2; ++pass) {
        k_fan_blur<<<grid, kFanThreads, smem, st>>>(p, pass, keys, out);
        D4W_CHECK_LAUNCH("k_fan_blur");
    }
    return D4W_OK;
}

extern "C" int d4w_row_moments(const float* x, size_t ld, int nrows, int n, int chunk, double* out, void* stream_v) {
    if (!x || !out) return fail(D4W_ERR_ARG, "d4w_row_moments: null pointer");
    if (nrows < 1 || n < 1 || chunk < 1 || ld < (size_t)n) return fail(D4W_ERR_ARG, "d4w_row_moments: need nrows, n, chunk >= 1 and ld >= n");
    const long long nchunks = (n + (long long)chunk - 1) / chunk, blocks = nrows * nchunks;
    if (blocks > 0x7fffffffLL) return fail(D4W_ERR_UNSUPPORTED, "d4w_row_moments: too many row chunks for one launch");
    k_row_moments<<<(unsigned)blocks, kMomThreads, 0, (cudaStream_t)stream_v>>>(x, ld, n, chunk, (int)nchunks, out);
    D4W_CHECK_LAUNCH("k_row_moments");
    return D4W_OK;
}

extern "C" int d4w_detrend_linear(const float* x, size_t ld, int nrows, int n, const double* mom, float* y, void* stream_v) {
    if (!x || !mom || !y) return fail(D4W_ERR_ARG, "d4w_detrend_linear: null pointer");
    if (nrows < 1 || n < 1 || ld < (size_t)n) return fail(D4W_ERR_ARG, "d4w_detrend_linear: need nrows, n >= 1 and ld >= n");
    return for_row_blocks(nrows, kMaxGridRows, [&](size_t r0, int rows) -> int {
        const dim3 grid((unsigned)std::min((n + 255) / 256, 64), (unsigned)rows);
        k_detrend<<<grid, 256, 0, (cudaStream_t)stream_v>>>(x + r0 * ld, ld, rows, n, mom + r0 * 3, y + r0 * n);
        D4W_CHECK_LAUNCH("k_detrend");
        return D4W_OK;
    });
}
