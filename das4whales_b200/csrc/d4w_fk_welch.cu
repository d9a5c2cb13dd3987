// d4w_fk_welch.cu -- segment staging of the f-k Welch spectrum (C ABI d4w_fk_segment_stage in include/d4w.h): each
// segment of a batch is detrended, windowed in time and channel, and written as its own contiguous matrix, which
// d4w_fk_spectrum_apply then transforms unchanged.  The body is fk_welch.cuh's, shared with the host emulator.  Its own
// translation unit, so every kernel of the other objects keeps its code.
#include <cstdint>
#include <string>
#include "d4w_common.hpp"
#include "fk_welch.cuh"

using namespace d4w;

namespace {

constexpr int kStageThreads = 256;
// Rows up to this many samples go through shared memory (read once from HBM); longer ones are read twice, the second time
// from L2.  Up to here four 256-thread CTAs share an SM; at 24 000 samples only two do, and re-reading was faster on an
// H100 (DESIGN.md §4 has the measurement).
constexpr int kStageSmemRowMax = 12 * 1024;

__global__ void __launch_bounds__(kStageThreads)
k_fk_segment_stage(StageParams sp, const float* __restrict__ x, const float* __restrict__ wx, const float* __restrict__ wt,
                   float* __restrict__ out) {
    extern __shared__ __align__(16) double stage_smem[];
    body_fk_segment_stage(sp, x, wx, wt, out, (long long)blockIdx.x, (int)blockIdx.y, threadIdx.x, blockDim.x, stage_smem);
}

// block size: 256 threads, fewer for short rows (about 8 samples per thread, whole warps)
int stage_threads(int l) {
    const int t = ((l + 7) / 8 + 31) / 32 * 32;
    return t < kStageThreads ? t : kStageThreads;
}

}  // namespace

extern "C" int d4w_fk_segment_stage(const float* x, int nx, int ns, int c0, int lx, int t0, int l, int step, int nseg,
                                    const float* wx, const float* wt, int detrend, float* out, size_t seg_stride, void* stream_v) {
    if (!x || !wx || !wt || !out) return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: null pointer");
    if (nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: nx and ns must be >= 1");
    if (lx < 1 || c0 < 0 || (long long)c0 + lx > nx)
        return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: channels [" + std::to_string(c0) + ", " + std::to_string((long long)c0 + lx) +
                                     ") empty or outside [0, " + std::to_string(nx) + ")");
    if (lx > 65535) return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: more than 65 535 channels per segment");
    if (l < 1 || t0 < 0 || step < 1 || nseg < 1 || (long long)t0 + (long long)(nseg - 1) * step + l > ns)
        return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: segments t0 = " + std::to_string(t0) + " + s * " + std::to_string(step) +
                                     ", s < " + std::to_string(nseg) + ", of " + std::to_string(l) + " samples, empty or outside [0, " +
                                     std::to_string(ns) + ")");
    if (detrend != 0 && detrend != 1) return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: detrend must be 0 or 1");
    if (seg_stride < (size_t)lx * l) return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: seg_stride is shorter than one segment");
    // every staged segment must start where d4w_fk_spectrum_apply's column kernels need it (check_matrix_alignment)
    const uintptr_t align = l % 4 == 0 ? 16 : l % 2 == 0 ? 8 : sizeof(float);
    if ((uintptr_t)out % align || (seg_stride * sizeof(float)) % align)
        return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: out and seg_stride must keep every segment " + std::to_string(align) +
                                     "-byte aligned for " + std::to_string(l) + " samples per row");
    if (l % 4 == 0 && (uintptr_t)wt % 16) return fail(D4W_ERR_ARG, "d4w_fk_segment_stage: wt must be 16-byte aligned when l % 4 == 0");
    int device = 0;
    D4W_CUDA_TRY(cudaGetDevice(&device));
    StageParams sp{};
    sp.ns = ns; sp.c0 = c0; sp.t0 = t0; sp.step = step; sp.lx = lx; sp.l = l; sp.seg_stride = seg_stride; sp.detrend = detrend;
    sp.smem_row = detrend && l <= kStageSmemRowMax;
    const int threads = stage_threads(l);
    const size_t smem = fk_stage_smem_bytes(l, threads, sp.smem_row);
    static bool attr_done_dev[64] = {};      // opt in to the device's shared memory once per device
    if (!attr_done_dev[device & 63]) {
        int cap = 0;
        D4W_CUDA_TRY(cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_fk_segment_stage, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
        attr_done_dev[device & 63] = true;
    }
    k_fk_segment_stage<<<dim3((unsigned)nseg, (unsigned)lx), threads, smem, (cudaStream_t)stream_v>>>(sp, x, wx, wt, out);
    D4W_CHECK_LAUNCH("k_fk_segment_stage");
    return D4W_OK;
}
