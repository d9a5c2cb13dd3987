// d4w_fk_spectrum.cu -- device side of the f-k power spectrum (d4w_fk.cu: d4w_fk_spectrum_*): the forward-only power
// pass that follows the filter's P1 and P2.  The kernel lives in a translation unit of its own so that every kernel of
// d4w_fk.o and d4w_rows.o compiles to the same code as without it (ptxas allocates kernels differently when the
// non-inlined FFT stage helpers gain callers in the same module).  The body is fk_spectrum.cuh's, shared with the host
// emulator.
#include "d4w_common.hpp"
#include "fk_spectrum.cuh"

namespace d4w {

static __global__ void __launch_bounds__(256, 2)
k_fk_power(RowParams rp, SpecParams sp, const float2* __restrict__ w, size_t ldw, float* __restrict__ out) {
    body_fk_power(rp, sp, w, ldw, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, d4w_dyn_smem, out);
}

// grid (T1, kept rows), the middle row pass's block size and shared memory
int launch_fk_power(dim3 grid, int threads, size_t smem, const RowParams& rp, const SpecParams& sp, const float2* w, size_t ldw,
                    float* out, int device, cudaStream_t stream) {
    static bool attr_done_dev[64] = {};      // opt in to the device's shared memory once per device, as plan creation does
    if (!attr_done_dev[device & 63]) {
        int cap = 0;
        D4W_CUDA_TRY(cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_fk_power, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
        attr_done_dev[device & 63] = true;
    }
    k_fk_power<<<grid, threads, smem, stream>>>(rp, sp, w, ldw, out);
    D4W_CHECK_LAUNCH("k_fk_power");
    return D4W_OK;
}

}  // namespace d4w
