// d4w_csd.cu -- cross-spectral density and coherence of row pairs (C ABI d4w_csd in include/d4w.h): scipy.signal.csd and
// scipy.signal.coherence for every output row in one launch.  The CTA bodies are csd_kernels.cuh; a median over more
// segments than fit shared memory goes through the workspace and k_csd_median, an exact selection of signed values.
// Its own translation unit, so the kernels of d4w_welch.cu and d4w_rows.cu keep their code.
#include <climits>
#include <string>
#include "d4w_common.hpp"
#include "csd_kernels.cuh"
#include "plan_k2pos.cuh"

using namespace d4w;

namespace {

__global__ void __launch_bounds__(kWelchThreads, 2)
k_csd(CsdParams cp, const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ win,
      void* __restrict__ out, float* __restrict__ ws) {
    extern __shared__ __align__(16) double csd_smem[];
    csd_body(cp, x, y, win, out, ws, (long long)blockIdx.x, threadIdx.x, blockDim.x, csd_smem);
}

__global__ void __launch_bounds__(kCsdSelThreads)
k_csd_median(const float* __restrict__ v, long long nrows, int n, float* __restrict__ out) {
    __shared__ int sel_smem[kCsdSelThreads / kCsdSelGroup * kCsdSelInts];
    csd_median_body(v, nrows, n, out, (long long)blockIdx.x, threadIdx.x, blockDim.x, sel_smem);
}

// argument check shared by the entry and its workspace query; "" when the sizes are consistent
std::string csd_args(const d4w_fft_plan* p, int nrows, int ns, int nperseg, int step, int what, int average) {
    if (!p) return "null plan";
    if (nrows < 1 || ns < 1) return "nrows and ns must be >= 1";
    if (nperseg < 1 || nperseg > ns) return "nperseg must be in [1, ns]";
    if (step < 1) return "step (nperseg - noverlap) must be >= 1";
    if (p->n < nperseg) return "nfft (the plan's length) must be >= nperseg";
    if (average != 0 && average != 1) return "average must be 0 (mean) or 1 (median)";
    if (what != 0 && what != 1) return "what must be 0 (Pxy) or 1 (Cxy)";
    if (what == 1 && average != 0) return "the coherence is computed from mean spectra only (average = 0)";
    return "";
}

// largest nfft whose one frame fits `cap` bytes of shared memory on the route `cp` takes: the mean route keeps 2 or 4
// doubles of bin sums per bin, the workspace median none (the median in shared memory always fits: its budget is lower)
int csd_max_nfft(size_t cap, const CsdParams& cp) {
    int n = 2;
    while (csd_smem_bytes(n + 1, (n + 1) / 2 + 1, cp.nseg, 1, cp.mode, cp.coherence) <= cap) ++n;
    return n;
}

}  // namespace

extern "C" size_t d4w_csd_workspace_bytes(const d4w_fft_plan* p, int nrows, int ns, int nperseg, int step, int what, int average) {
    if (!csd_args(p, nrows, ns, nperseg, step, what, average).empty()) return 0;
    CsdParams cp;
    size_t smem = 0;
    csd_config(p->pl, ns, nperseg, step, 0, 1.0, what, average, p->smem_cap, cp, smem);
    if (cp.mode != kCsdMedianWs) return 0;
    return (size_t)nrows * cp.nbins * 2 * cp.nseg * sizeof(float);
}

extern "C" int d4w_csd(d4w_fft_plan* p, const float* x, long long x_row_stride, const float* y, long long y_row_stride,
                       int nrows, int ns, int nperseg, int step, const float* win, int detrend, double scale, int what,
                       int average, void* out, void* ws, void* stream_v) {
    const std::string bad = csd_args(p, nrows, ns, nperseg, step, what, average);
    if (!bad.empty()) return fail(D4W_ERR_ARG, "d4w_csd: " + bad);
    if (!x || !y || !win || !out) return fail(D4W_ERR_ARG, "d4w_csd: null pointer");
    if ((x_row_stride != 0 && x_row_stride < ns) || (y_row_stride != 0 && y_row_stride < ns))
        return fail(D4W_ERR_ARG, "d4w_csd: a row stride must be 0 (one broadcast row) or >= ns");
    DeviceGuard guard(p->device);
    CsdParams cp;
    size_t smem = 0;
    if (csd_config(p->pl, ns, nperseg, step, detrend, scale, what, average, p->smem_cap, cp, smem))
        return fail(D4W_ERR_UNSUPPORTED, std::string("d4w_csd: nfft = ") + std::to_string(p->n) + " needs " + std::to_string(smem) +
                                             " bytes of shared memory per block, more than the " + std::to_string(p->smem_cap) +
                                             " available: nfft <= " + std::to_string(csd_max_nfft(p->smem_cap, cp)) +
                                             (what ? " for the coherence"
                                              : cp.mode == kCsdMean ? " for the mean cross spectrum" : " for the median cross spectrum"));
    if (cp.mode == kCsdMedianWs && !ws) return fail(D4W_ERR_ARG, "d4w_csd: the median over this many segments needs a workspace");
    const long long nsel = (long long)nrows * cp.nbins * 2;                        // rows of the workspace median
    if (cp.mode == kCsdMedianWs && (nsel + kCsdSelThreads / kCsdSelGroup - 1) / (kCsdSelThreads / kCsdSelGroup) > INT_MAX)
        return fail(D4W_ERR_UNSUPPORTED, "d4w_csd: more than 2^31 - 1 median blocks per call");
    cp.tw = p->d_tw;
    cp.xstride = x_row_stride;
    cp.ystride = y_row_stride;
    D4W_CUDA_TRY(welch_k2pos(p, &cp.k2pos));
    cudaStream_t st = (cudaStream_t)stream_v;
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_csd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_csd<<<(unsigned)nrows, kWelchThreads, smem, st>>>(cp, x, y, win, out, static_cast<float*>(ws));
    D4W_CHECK_LAUNCH("k_csd");
    if (cp.mode == kCsdMedianWs) {
        const long long rows_per_cta = kCsdSelThreads / kCsdSelGroup;
        k_csd_median<<<(unsigned)((nsel + rows_per_cta - 1) / rows_per_cta), kCsdSelThreads, 0, st>>>(
            static_cast<const float*>(ws), nsel, cp.nseg, static_cast<float*>(out));
        D4W_CHECK_LAUNCH("k_csd_median");
    }
    return D4W_OK;
}
