// xcorr_launch.cuh -- the generic shared-memory FFT plan and the launch of the overlap-save matched-filter kernels, shared by
// d4w_xcorr (d4w_rows.cu) and d4w_xcorr_same (d4w_xcorr_same.cu).  The two modes are compiled in separate translation units
// so that adding the "same" instantiations leaves the code generated for the rest of d4w_rows.cu untouched.
#pragma once
#include <string>
#include <vector>
#include "d4w_common.hpp"
#include "fk_hostplan.hpp"
#include "rows_kernels.cuh"

struct d4w_fft_plan {
    int n = 0, device = 0;
    size_t smem_cap = 0;
    d4w::FftPlan pl{};
    std::vector<int> pos2k;
    std::vector<int> tab2k;      // frequency of each entry of a multiplier table in d4w_xcorr's order
    int fused = 0;               // k_xcorr_fused usable: >= 2 stages, first and last stage in-register radices
    float2* d_tw = nullptr;
    int* d_k2pos = nullptr;
    int pfa = 0;                 // n == 2520: prime-factor blocks of the matched filter (fft_pfa.cuh)
    int* d_tpos = nullptr;       // pfa: position of time index i
    float2* d_wn = nullptr;      // exp(-2 pi i j / n), j < n (sliding-DFT STFT)
};

namespace d4w {

// One dispatch for both modes (rows_kernels.cuh, k_xcorr*): SAME = false is d4w_xcorr, SAME = true d4w_xcorr_same.
// nx rows of one launch; out_tpl_stride is the distance between the templates' output matrices.
template <bool SAME>
static int xcorr_launch_block(d4w_fft_plan* p, const float* x, int nx, int ns, int valid, int ntpl, const void* dev_tabs,
                              const double* dev_mu_over_m, const double* dev_stats, const double* dev_segpre,
                              const float* dev_rowmax, int lag0, float* out, size_t out_tpl_stride, void* stream) {
    const char* fn = SAME ? "d4w_xcorr_same" : "d4w_xcorr";
    XcorrParams xp{};
    xp.pl = p->pl; xp.tw = p->d_tw; xp.nb = p->n; xp.valid = valid; xp.ntpl = ntpl; xp.ns = ns;
    xp.normalize = dev_stats != nullptr ? 1 : 0;
    xp.nseg = (ns + valid - 1) / valid;
    // dual-lane kernel (four segments per CTA, packed f32x2 butterflies): needs the fused plan shape; 2 CTAs per SM.
    // Shared memory: S and B (16 B per sample each) and the mu-term prefix per group of 8 samples.
    const size_t smem_dual = (size_t)2 * p->n * 16 + (size_t)((valid + 7) / 8) * 16 + 16;
    if (p->pfa) {
        const size_t smem_pfa = smem_dual + (size_t)valid * 8;                   // + the fp16 in-group prefixes
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_xcorr_pfa<SAME>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
        if (smem_pfa > 112 * 1024) return fail(D4W_ERR_UNSUPPORTED, std::string(fn) + ": shared memory");
        dim3 gridp((xp.nseg + 3) / 4, nx);
        k_xcorr_pfa<SAME><<<gridp, kPfaThreads, smem_pfa, (cudaStream_t)stream>>>(xp, p->d_tpos, x, (const float2*)dev_tabs, dev_stats,
                                                                          dev_segpre, dev_mu_over_m, out, out_tpl_stride,
                                                                          dev_rowmax, lag0);
        D4W_CHECK_LAUNCH("k_xcorr_pfa");
        return D4W_OK;
    }
    bool small_radices = true;
    for (int st = 0; st < p->pl.nstages; ++st) small_radices = small_radices && xcorr_dual_radix_ok(p->pl.radix[st]);
    if (p->fused && p->pl.nstages >= 2 && small_radices && smem_dual <= 110 * 1024) {
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_xcorr_dual<SAME>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
        dim3 gridd((xp.nseg + 3) / 4, nx);
        k_xcorr_dual<SAME><<<gridd, 256, smem_dual, (cudaStream_t)stream>>>(xp, x, (const float2*)dev_tabs, dev_stats, dev_segpre,
                                                                           dev_mu_over_m, out, out_tpl_stride, dev_rowmax, lag0);
        D4W_CHECK_LAUNCH("k_xcorr_dual");
        return D4W_OK;
    }
    const size_t smem = (size_t)3 * p->n * sizeof(float2);
    if (smem + 1024 > p->smem_cap) return fail(D4W_ERR_UNSUPPORTED, std::string(fn) + ": block length too large for shared memory");
    dim3 grid((xp.nseg + 1) / 2, nx);
    if (p->fused) {
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_xcorr_fused<SAME>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_cap - 1024));
        k_xcorr_fused<SAME><<<grid, 128, smem, (cudaStream_t)stream>>>(xp, x, (const float2*)dev_tabs, dev_stats, dev_segpre, dev_mu_over_m,
                                                                      out, out_tpl_stride, dev_rowmax, lag0);
    } else {
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_xcorr<SAME>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_cap - 1024));  // minus its static smem
        k_xcorr<SAME><<<grid, 128, smem, (cudaStream_t)stream>>>(xp, x, (const float2*)dev_tabs, dev_stats, dev_segpre, dev_mu_over_m, out,
                                                                out_tpl_stride, dev_rowmax, lag0);
    }
    D4W_CHECK_LAUNCH("k_xcorr");
    return D4W_OK;
}

// Any number of rows, in blocks of kMaxGridRows; out is [ntpl][nx][ns] for the whole call.
template <bool SAME>
static int xcorr_launch(d4w_fft_plan* p, const float* x, int nx, int ns, int valid, int ntpl, const void* dev_tabs,
                        const double* dev_mu_over_m, const double* dev_stats, const double* dev_segpre, const float* dev_rowmax,
                        int lag0, float* out, void* stream) {
    DeviceGuard guard(p->device);
    const int nseg = (ns + valid - 1) / valid;
    return for_row_blocks(nx, kMaxGridRows, [&](size_t r0, int rows) -> int {
        return xcorr_launch_block<SAME>(p, x + r0 * ns, rows, ns, valid, ntpl, dev_tabs, dev_mu_over_m,
                                        dev_stats ? dev_stats + 4 * r0 : nullptr, dev_segpre ? dev_segpre + r0 * nseg : nullptr,
                                        dev_rowmax ? dev_rowmax + r0 : nullptr, lag0, out + r0 * ns, (size_t)nx * ns, stream);
    });
}

}  // namespace d4w
