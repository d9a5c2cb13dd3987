// d4w_fk_bank.cu -- device side of the f-k mask bank (d4w_fk.cu: d4w_fk_bank_*): the out-of-place middle pass
// (W -> W', one mask table per launch) and the gather of each mask's table onto the bank's union support.
// The kernels live in a translation unit of their own so that every kernel of d4w_fk.o and d4w_rows.o compiles to the
// same code as without them (ptxas allocates kernels differently when the non-inlined FFT stage helpers gain callers
// in the same module).  The bodies are fk_kernels.cuh's, shared with the host emulator.
#include "d4w_common.hpp"
#include "fk_kernels.cuh"

namespace d4w {

static __global__ void __launch_bounds__(256, 2)
k_row_mid_oop(RowParams rp, float2* __restrict__ w, size_t ldw, const float* __restrict__ tab, size_t tab_slot_stride,
              float2* __restrict__ dst) {
    body_row_mid<float, true>(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, d4w_dyn_smem, dst);
}

static __global__ void __launch_bounds__(128, 2)     // as k_row_mid_dual: radix-25 dual butterflies need ~190 registers
k_row_mid_dual_oop(RowParams rp, float2* __restrict__ w, size_t ldw, const float* __restrict__ tab, size_t tab_slot_stride,
                   int nslots, float2* __restrict__ dst) {
    body_row_mid_dual<true>(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, nslots, threadIdx.x, blockDim.x,
                            reinterpret_cast<cpd*>(d4w_dyn_smem), dst);
}

static __global__ void k_bank_gather(const float* src, float* dst, const int* src_row, int ns, size_t total) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < total) body_bank_gather(src, dst, src_row, ns, idx);
}

// P3 of a bank: same grid, block and shared memory as the in-place launch of d4w_fk.cu; dual: k_row_mid_dual_oop with
// `nslots` rows, fused: k_row_mid_fused writing to dst, otherwise k_row_mid_oop
int launch_row_mid_oop(bool dual, bool fused, dim3 grid, int threads, size_t smem, const RowParams& rp, float2* w, size_t ldw,
                       const float* tab, size_t tab_slot_stride, int nslots, float2* dst, int device, cudaStream_t stream) {
    static bool attr_done_dev[64] = {};      // opt in to the device's shared memory once per device, as plan creation does
    if (!attr_done_dev[device & 63]) {
        int cap = 0;
        D4W_CUDA_TRY(cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_row_mid_oop, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_row_mid_dual_oop, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
        attr_done_dev[device & 63] = true;
    }
    if (fused) return launch_row_mid_fused(grid, threads, smem, rp, w, ldw, tab, tab_slot_stride, dst, device, stream);
    if (dual) k_row_mid_dual_oop<<<grid, threads, smem, stream>>>(rp, w, ldw, tab, tab_slot_stride, nslots, dst);
    else k_row_mid_oop<<<grid, threads, smem, stream>>>(rp, w, ldw, tab, tab_slot_stride, dst);
    D4W_CHECK_LAUNCH("k_row_mid_oop");
    return D4W_OK;
}

int launch_bank_gather(const float* src, float* dst, const int* src_row, int ns, size_t total, cudaStream_t stream) {
    const size_t blocks = (total + 255) / 256;
    if (blocks > 0x7fffffffull) return fail(D4W_ERR_UNSUPPORTED, "bank table too large for one launch");
    k_bank_gather<<<(unsigned)blocks, 256, 0, stream>>>(src, dst, src_row, ns, total);
    D4W_CHECK_LAUNCH("k_bank_gather");
    return D4W_OK;
}

}  // namespace d4w
