// d4w_noise.cu -- envelope and moment statistics of row windows (C ABI d4w_env_stats in include/d4w.h), the per-channel
// quantities of scripts/main_bathynoise.py:183-189 and :257-259.
//
// The record is composed from existing entry points on a workspace: d4w_row_stats of the window, d4w_hilbert's envelope,
// d4w_row_stats of the envelope (its mean) and d4w_row_median_ld of the envelope, then k_env_pack.  A one-CTA-per-row
// kernel that kept the window in shared memory and did all four there was slower on an H100 at 11 020 x 12 000 (5.04 ms
// against 4.61 ms for these calls, whole rows plus a 1 400-sample window): at 144 KB of shared memory per row it runs one
// CTA per SM.
#include <algorithm>
#include "d4w_common.hpp"
#include "row_plan.hpp"

using namespace d4w;

namespace {

// A row with zero variance is constant and its envelope is |mean| exactly; d4w_hilbert's split route transforms two rows
// per complex FFT, which would leave a zero channel an fp32-rounding residue of its neighbour's envelope instead of 0.
__global__ void __launch_bounds__(256)
k_env_pack(const double* __restrict__ stx, const double* __restrict__ ste, const float* __restrict__ med, int nrows,
           double* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    const double mean = stx[4 * (size_t)r], var = stx[4 * (size_t)r + 2];
    const bool flat = var == 0.0;
    double* o = out + 5 * (size_t)r;
    o[0] = flat ? fabs(mean) : (double)med[r];
    o[1] = flat ? fabs(mean) : ste[4 * (size_t)r];
    o[2] = mean;
    o[3] = var + mean * mean;
    o[4] = var;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// workspace for `rows` rows: [window copy if strided][envelope][Hilbert workspace][stats of x][stats of env][median]
struct EnvWs { size_t env, hil, stx, ste, med, total; };
EnvWs env_ws_layout(const d4w_row_plan* p, int rows, bool strided) {
    EnvWs w{};
    const size_t mat = align256((size_t)rows * p->ns * sizeof(float));
    w.env = strided ? mat : 0;                           // the window copy, when there is one, is at offset 0
    w.hil = w.env + mat;
    w.stx = w.hil + align256(d4w_row_workspace_bytes(p, rows));
    w.ste = w.stx + align256((size_t)rows * 4 * sizeof(double));
    w.med = w.ste + align256((size_t)rows * 4 * sizeof(double));
    w.total = w.med + align256((size_t)rows * sizeof(float));
    return w;
}

}  // namespace

extern "C" size_t d4w_env_stats_workspace_bytes(const d4w_row_plan* p, int nrows, size_t ld) {
    if (!p || nrows < 1) return 0;
    return env_ws_layout(p, std::min(nrows, kMaxGridRows), ld != (size_t)p->ns).total;
}

extern "C" int d4w_env_stats(d4w_row_plan* p, const float* x, int nrows, size_t ld, double* out, void* ws, void* stream_v) {
    if (!p || !x || !out || !ws || nrows < 1) return fail(D4W_ERR_ARG, "d4w_env_stats: bad argument");
    const int n = p->ns;
    if (ld < (size_t)n) return fail(D4W_ERR_ARG, "d4w_env_stats: ld must be >= the plan's row length");
    DeviceGuard guard(p->device);
    cudaStream_t stream = (cudaStream_t)stream_v;
    const bool strided = ld != (size_t)n;
    // passes of kMaxGridRows rows bound the workspace
    const EnvWs w = env_ws_layout(p, std::min(nrows, kMaxGridRows), strided);
    char* base = static_cast<char*>(ws);
    float* env = reinterpret_cast<float*>(base + w.env);
    double* stx = reinterpret_cast<double*>(base + w.stx);
    double* ste = reinterpret_cast<double*>(base + w.ste);
    float* med = reinterpret_cast<float*>(base + w.med);
    return for_row_blocks(nrows, kMaxGridRows, [&](size_t r0, int rows) -> int {
        const float* xr = x + r0 * ld;
        if (strided) {
            float* xc = reinterpret_cast<float*>(base);
            D4W_CUDA_TRY(cudaMemcpy2DAsync(xc, (size_t)n * sizeof(float), xr, ld * sizeof(float), (size_t)n * sizeof(float), rows,
                                           cudaMemcpyDeviceToDevice, stream));
            xr = xc;
        }
        int rc = d4w_row_stats(xr, rows, n, 0, stx, nullptr, stream);
        if (rc == D4W_OK) rc = d4w_hilbert(p, xr, env, rows, base + w.hil, /*mode: envelope*/ 0, nullptr, stream);
        if (rc == D4W_OK) rc = d4w_row_stats(env, rows, n, 0, ste, nullptr, stream);
        if (rc == D4W_OK) rc = d4w_row_median_ld(env, rows, (size_t)n, (size_t)n, med, stream);
        if (rc != D4W_OK) return rc;
        k_env_pack<<<(rows + 255) / 256, 256, 0, stream>>>(stx, ste, med, rows, out + 5 * r0);
        D4W_CHECK_LAUNCH("k_env_pack");
        return D4W_OK;
    });
}
