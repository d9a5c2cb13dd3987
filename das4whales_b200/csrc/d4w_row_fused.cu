// d4w_row_fused.cu -- k_row_mid_fused, the middle row pass with its first stage straight from global memory and its last
// stage, table multiply and inverse in registers, instantiated once per (first, last) radix pair of D4W_ROW_FUSED_PAIRS:
// the f-k filter's P3 (mask table, in place or into a bank's W'), the Hilbert rows (sgn table) and the chirp-z rows
// (complex kernel spectrum).  With only its own pair of butterflies each kernel fits 128 registers without spilling.
// The kernels live in a translation unit of their own so that every kernel of d4w_fk.o and d4w_rows.o compiles to the
// same code as without them (ptxas allocates kernels differently when the non-inlined FFT stage helpers gain callers
// in the same module).
#include "d4w_common.hpp"
#include "fk_kernels.cuh"

namespace d4w {

template <int R0, int RL, typename TabT, bool OOP>
static __global__ void __launch_bounds__(256, 2)
k_row_mid_fused(RowParams rp, float2* __restrict__ w, size_t ldw, const TabT* __restrict__ tab, size_t tab_slot_stride,
                float2* __restrict__ dst) {
    body_row_mid_fused<R0, RL, TabT, OOP>(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x,
                                          d4w_dyn_smem, dst);
}

template <int R0, int RL, typename TabT, bool OOP>
bool attr_done_dev[64] = {};      // opt in to the device's shared memory once per device and kernel

template <int R0, int RL, typename TabT, bool OOP>
static int launch_one(dim3 grid, int threads, size_t smem, const RowParams& rp, float2* w, size_t ldw, const TabT* tab,
                      size_t tab_slot_stride, float2* dst, int device, cudaStream_t stream) {
    if (!attr_done_dev<R0, RL, TabT, OOP>[device & 63]) {
        int cap = 0;
        D4W_CUDA_TRY(cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_row_mid_fused<R0, RL, TabT, OOP>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
        attr_done_dev<R0, RL, TabT, OOP>[device & 63] = true;
    }
    k_row_mid_fused<R0, RL, TabT, OOP><<<grid, threads, smem, stream>>>(rp, w, ldw, tab, tab_slot_stride, dst);
    D4W_CHECK_LAUNCH("k_row_mid_fused");
    return D4W_OK;
}

template <typename TabT>
int launch_row_mid_fused(dim3 grid, int threads, size_t smem, const RowParams& rp, float2* w, size_t ldw, const TabT* tab,
                         size_t tab_slot_stride, float2* dst, int device, cudaStream_t stream) {
    int rc = D4W_ERR_UNSUPPORTED;
    with_row_fused_pair(rp.pl.radix[0], rp.pl.radix[rp.pl.nstages - 1], [&](auto r0, auto rl) {
        constexpr int R0 = decltype(r0)::value, RL = decltype(rl)::value;
        if constexpr (std::is_same<TabT, float>::value)
            if (dst) { rc = launch_one<R0, RL, TabT, true>(grid, threads, smem, rp, w, ldw, tab, tab_slot_stride, dst, device, stream); return; }
        rc = launch_one<R0, RL, TabT, false>(grid, threads, smem, rp, w, ldw, tab, tab_slot_stride, nullptr, device, stream);
    });
    return rc == D4W_ERR_UNSUPPORTED ? fail(rc, "k_row_mid_fused: not built for this row plan's first / last radix") : rc;
}

template int launch_row_mid_fused<float>(dim3, int, size_t, const RowParams&, float2*, size_t, const float*, size_t, float2*, int,
                                         cudaStream_t);
template int launch_row_mid_fused<float2>(dim3, int, size_t, const RowParams&, float2*, size_t, const float2*, size_t, float2*,
                                          int, cudaStream_t);

}  // namespace d4w
