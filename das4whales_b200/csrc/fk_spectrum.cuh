// fk_spectrum.cuh -- the forward-only power pass of the f-k spectrum (d4w_fk_spectrum_apply).
//
// After the filter's P1 (channel transform of the kept half-plane rows k' in [0, nx/2]) and P2 (radix-T1 time split),
// sub-row kt1 of slot k' holds the length-T2 sequence whose DFT is X[k', kt1 + T1*kt2].  The power pass finishes that
// transform in shared memory exactly as the forward half of body_row_mid does, then writes p = |X|^2 of every frequency
// inside the band to two places of the shifted plane P (fftshift's placement, row(k) = (k + nx/2) mod nx and
// col(f) = (f + ns/2) mod ns):
//   P[row(+k'), col(f)]  and, since X[-k, f] = conj X[k, -f] for real input,  P[row(-k'), col((ns - f) mod ns)].
// The self-conjugate rows (k' = 0, and k' = nx/2 for even nx) are written once.  Every element of P is written by one
// thread, so `accumulate` (P += scale*p, for averaging time blocks) needs no atomics.
//
// The epilogue reads shared memory in natural frequency order (k2pos_row), so a warp stores consecutive columns when
// T1 = 1; with T1 > 1 the columns of one CTA are T1 apart, and the T1 CTAs of a slot (adjacent in blockIdx.x) fill the
// same L2 sectors at about the same time.
#pragma once
#include "fk_kernels.cuh"

namespace d4w {

struct SpecParams {
    const int* act_k;              // half-plane wavenumber k' of each slot
    const int* k2pos_row;          // natural T2-point frequency -> position after the forward stages
    int nx, ns;
    int k_lo, k_hi, f_lo, f_hi;    // the band: half-open row and column ranges of the shifted plane
    float scale;
    int accumulate;                // 0: out = scale*p, 1: out += scale*p
};

__host__ __device__ inline void body_fk_power(const RowParams& rp, const SpecParams& sp, const float2* __restrict__ w, size_t ldw,
                                              int kt1, int slot, int tid, int nthr, float2* smem, float* __restrict__ out) {
    const int n = rp.t2;
    const float2* g = w + (size_t)slot * ldw + (size_t)kt1 * n;
    bool staged = false;
#ifdef __CUDA_ARCH__
    if ((n & 1) == 0 && ((((size_t)slot * ldw + (size_t)kt1 * n) & 1) == 0)) {
        for (int i = tid; i < n / 2; i += nthr) cp_async16(smem + 2 * i, g + 2 * i);     // whole tile in flight
        cp_async_wait_all();
        __syncthreads();
        staged = true;
    }
#endif
    if (!staged) {
        for (int i = tid; i < n; i += nthr) smem[i] = g[i];
        D4W_SYNC();
    }
    fft_forward_stages(smem, rp.pl, rp.tw, 1, n, tid, nthr, 0, rp.pl.nstages);
    const int nx = sp.nx, ns = sp.ns, nf = sp.f_hi - sp.f_lo;
    const int k = sp.act_k[slot];
    const int row_p = (k + nx / 2) % nx, row_n = (nx - k + nx / 2) % nx;
    const bool self = k == 0 || 2 * k == nx;
    const bool use_p = row_p >= sp.k_lo && row_p < sp.k_hi;
    const bool use_n = !self && row_n >= sp.k_lo && row_n < sp.k_hi;
    float* op = out + (size_t)(use_p ? row_p - sp.k_lo : 0) * nf;
    float* on = out + (size_t)(use_n ? row_n - sp.k_lo : 0) * nf;
    for (int i = tid; i < n; i += nthr) {
        const float2 v = smem[sp.k2pos_row[i]];
        const float p = (v.x * v.x + v.y * v.y) * sp.scale;
        const int f = kt1 + rp.t1 * i;                               // natural frequency index, < ns
        if (use_p) {
            int c = f + ns / 2;
            if (c >= ns) c -= ns;
            c -= sp.f_lo;
            if (c >= 0 && c < nf) op[c] = sp.accumulate ? op[c] + p : p;
        }
        if (use_n) {
            int c = (f == 0 ? 0 : ns - f) + ns / 2;
            if (c >= ns) c -= ns;
            c -= sp.f_lo;
            if (c >= 0 && c < nf) on[c] = sp.accumulate ? on[c] + p : p;
        }
    }
}

}  // namespace d4w
