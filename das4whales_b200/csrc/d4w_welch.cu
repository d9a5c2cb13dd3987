// d4w_welch.cu -- per-channel Welch power spectral density (C ABI d4w_welch in include/d4w.h): scipy.signal.welch over
// whole chunks of every row, the long-term spectral average of tools.spec (das4whales/tools.py:212-236).  The CTA body is
// welch_kernels.cuh; a median over more segments than fit shared memory goes through the workspace and d4w_row_median.
// Its own translation unit, so the kernels of d4w_rows.cu keep their code.
#include <climits>
#include <string>
#include "d4w_common.hpp"
#include "welch_kernels.cuh"
#include "plan_k2pos.cuh"

using namespace d4w;

namespace {

__global__ void __launch_bounds__(kWelchThreads, 2)
k_welch(WelchParams wp, const float* __restrict__ x, const float* __restrict__ win, float* __restrict__ out, float* __restrict__ ws) {
    extern __shared__ __align__(16) double welch_smem[];
    welch_body(wp, x, win, out, ws, (long long)blockIdx.x, threadIdx.x, blockDim.x, welch_smem);
}

// argument check shared by the entry and its workspace query; "" when the sizes are consistent
std::string welch_args(const d4w_fft_plan* p, int nrows, int ns, int chunk, int nperseg, int step, int average) {
    if (!p) return "null plan";
    if (nrows < 1 || ns < 1) return "nrows and ns must be >= 1";
    if (chunk < 1 || chunk > ns) return "chunk must be in [1, ns]";
    if (nperseg < 1 || nperseg > chunk) return "nperseg must be in [1, chunk]";
    if (step < 1) return "step (nperseg - noverlap) must be >= 1";
    if (p->n < nperseg) return "nfft (the plan's length) must be >= nperseg";
    if (average != 0 && average != 1) return "average must be 0 (mean) or 1 (median)";
    return "";
}

// largest nfft whose one frame pair fits `cap` bytes of shared memory (the mean route; the median never needs more)
int welch_max_nfft(size_t cap) {
    int n = 2;
    while (welch_smem_bytes(n + 1, (n + 1) / 2 + 1, 1, 1, kWelchMean) <= cap) ++n;
    return n;
}

}  // namespace

extern "C" size_t d4w_welch_workspace_bytes(const d4w_fft_plan* p, int nrows, int ns, int chunk, int nperseg, int step, int average) {
    if (!welch_args(p, nrows, ns, chunk, nperseg, step, average).empty()) return 0;
    WelchParams wp;
    size_t smem = 0;
    welch_config(p->pl, ns, chunk, nperseg, step, 0, 1.0, average, p->smem_cap, wp, smem);
    if (wp.mode != kWelchMedianWs) return 0;
    return (size_t)nrows * wp.nchunks * wp.nbins * wp.nseg * sizeof(float);
}

extern "C" int d4w_welch(d4w_fft_plan* p, const float* x, int nrows, int ns, int chunk, int nperseg, int step, const float* win,
                         int detrend, double scale, int average, float* out, void* ws, void* stream_v) {
    const std::string bad = welch_args(p, nrows, ns, chunk, nperseg, step, average);
    if (!bad.empty()) return fail(D4W_ERR_ARG, "d4w_welch: " + bad);
    if (!x || !win || !out) return fail(D4W_ERR_ARG, "d4w_welch: null pointer");
    DeviceGuard guard(p->device);
    WelchParams wp;
    size_t smem = 0;
    if (welch_config(p->pl, ns, chunk, nperseg, step, detrend, scale, average, p->smem_cap, wp, smem))
        return fail(D4W_ERR_UNSUPPORTED, "d4w_welch: nfft = " + std::to_string(p->n) + " needs " + std::to_string(smem) +
                                             " bytes of shared memory per block, more than the " + std::to_string(p->smem_cap) +
                                             " available: nfft <= " + std::to_string(welch_max_nfft(p->smem_cap)));
    const long long blocks = (long long)nrows * wp.nchunks;
    if (blocks > INT_MAX) return fail(D4W_ERR_UNSUPPORTED, "d4w_welch: more than 2^31 - 1 (row, chunk) pairs per call");
    if (wp.mode == kWelchMedianWs && !ws) return fail(D4W_ERR_ARG, "d4w_welch: the median over this many segments needs a workspace");
    if (blocks * wp.nbins > INT_MAX && wp.mode == kWelchMedianWs)
        return fail(D4W_ERR_UNSUPPORTED, "d4w_welch: more than 2^31 - 1 median rows per call");
    wp.tw = p->d_tw;
    D4W_CUDA_TRY(welch_k2pos(p, &wp.k2pos));
    cudaStream_t st = (cudaStream_t)stream_v;
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_welch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_welch<<<(unsigned)blocks, kWelchThreads, smem, st>>>(wp, x, win, out, static_cast<float*>(ws));
    D4W_CHECK_LAUNCH("k_welch");
    if (wp.mode == kWelchMedianWs)
        return d4w_row_median(static_cast<const float*>(ws), (int)(blocks * wp.nbins), (size_t)wp.nseg, out, stream_v);
    return D4W_OK;
}
