// fk_kernels.cuh -- the five passes of the support-pruned f-k filter and the mask builders.
//
//   x[c][t] real  --P1-->  W[slot][t]   (R2C along channels, 2*NC time samples per tile, only
//                                        wavenumber rows whose folded mask is non-zero are kept)
//   W  --P2-->  W      radix-T1 split of the length-ns time transform (streaming, registers only)
//   W  --P3-->  W      length-T2 FFT -> x folded mask -> length-T2 inverse FFT (one smem visit)
//   W  --P4-->  W      inverse radix-T1 split
//   W  --P5-->  y[c][t] real  (C2R along channels)
//
// Reference arithmetic replaced: dsp.fk_filter_filt / fk_filter_sparsefilt
// (/root/reference/src/das4whales/dsp.py:725-786) and the mask definitions of
// dsp.fk_filter_design (:85-171) and dsp.hybrid_ninf_filter_design (:308-454).
//
// Each kernel body is a __host__ __device__ function of (block index, tid, nthr, smem) whose
// per-thread loops are `for (i = tid; i < n; i += nthr)`, so tests/host_emul runs the very
// same code on the CPU with nthr = 1.
#pragma once
#include "fft_smem.cuh"
#include "fft_dual.cuh"

namespace d4w {

struct ColParams {
    FftPlan pl;
    const float2* tw;      // W_nx^j
    const int* k2pos;      // frequency index -> smem position after the forward stages
    const int* pos2k;      // inverse map
    int nx, ns;
    int nc;                // complex columns per tile (tile = 2*nc time samples)
    int nc_shift;          // log2(nc)
    int fstride;           // smem stride between columns (float2 units)
    int aligned;           // rows 8-byte aligned (ns even) -> float2 global accesses
    int dual;              // 1: dual-lane (f32x2) kernels, tile = 4*npair samples stored as cpd elements
    int npair, npair_shift;
    int aligned16;         // rows 16-byte aligned (ns % 4 == 0)
    int tma;               // 1: TMA-fed persistent kernels (npair == 1, ns % 4 == 0)
};

struct RowParams {
    FftPlan pl;            // length T2
    const float2* tw;      // W_T2^j
    const float2* twT;     // W_ns^j for j < T2 (split twiddles)
    int t1, t2;
    int dual;              // 1: k_row_mid_dual (two kept rows per CTA as f32x2 lanes)
};

enum { MASK_FAN = 0, MASK_HYBRID_NINF = 1, MASK_DENSE = 2 };

struct MaskParams {
    int kind;
    int nx, ns;
    double kval, fval;               // numpy fftfreq steps
    double c0, c1, c2, c3;           // cs_min, cp_min, cp_max, cs_max
    const double* h;                 // hybrid: H(f) profile over the shifted axis (ns entries)
    int col_lo, col_hi;              // hybrid: speed-filtered column range
    const float* dense;              // dense: [nx][ns] shifted layout
};

// ------------------------------------------------------------------ mask definitions
// Value of the reference's mask at shifted-layout index (i, j), in double.
__host__ __device__ inline double mask_fan(const MaskParams& mp, int i, int j) {
    const double k = (double)(i - mp.nx / 2) * mp.kval;       // dsp.py:130
    if (fabs(k) < 0.005) return 0.0;                          // dsp.py:142
    const double f = (double)(j - mp.ns / 2) * mp.fval;       // dsp.py:129
    const double v = fabs(f / k);                             // dsp.py:146
    const double half_pi = 1.57079632679489661923;
    double m = 1.0;
    if (v >= mp.c0 && v <= mp.c1) m = sin(half_pi * (v - mp.c0) / (mp.c1 - mp.c0));          // :149-151
    if (v >= mp.c2 && v <= mp.c3) m = 1.0 - sin(half_pi * (v - mp.c2) / (mp.c3 - mp.c2));    // :153-155
    if (v >= mp.c3) m = 0.0;                                  // :157
    if (v < mp.c0) m = 0.0;                                   // :158
    return m;
}

__host__ __device__ inline double hybrid_a(const MaskParams& mp, int i, int j) {
    double a = mp.h[j];                                       // dsp.py:372 (tiled H)
    if (j >= mp.col_lo && j < mp.col_hi) {                    // dsp.py:376
        const double half_pi = 1.57079632679489661923;
        const double f = (double)(j - mp.ns / 2) * mp.fval;
        const double k = (double)(i - mp.nx / 2) * mp.kval;
        const double ks_lo = f / mp.c3, kp_lo = f / mp.c2;    // :381-382
        const double ks_hi = f / mp.c0, kp_hi = f / mp.c1;    // :384-385
        double col = 0.0;
        if (ks_lo != kp_lo && k >= ks_lo && k <= kp_lo) col = sin(half_pi * (k - ks_lo) / (kp_lo - ks_lo));   // :388-391
        if (ks_hi != kp_hi && k >= kp_hi && k <= ks_hi) col = -sin(half_pi * (k - ks_hi) / (ks_hi - kp_hi));  // :392-395
        if (k > kp_lo && k < kp_hi) col = 1.0;                // :399
        a *= col;                                             // :402
    }
    return a;
}

__host__ __device__ inline double mask_shifted(const MaskParams& mp, int i, int j) {
    switch (mp.kind) {
        case MASK_FAN: return mask_fan(mp, i, j);
        case MASK_HYBRID_NINF: {                              // += fliplr ; += flipud  (dsp.py:405-406)
            const int i2 = mp.nx - 1 - i, j2 = mp.ns - 1 - j;
            return hybrid_a(mp, i, j) + hybrid_a(mp, i, j2) + hybrid_a(mp, i2, j) + hybrid_a(mp, i2, j2);
        }
        default: return (double)mp.dense[(size_t)i * mp.ns + j];
    }
}

// Folded mask at un-shifted DFT indices (k, f):  (M[k,f] + M[-k,-f]) / 2   (SURVEY App. A.1)
__host__ __device__ inline double mask_folded(const MaskParams& mp, int k, int f) {
    const int nx = mp.nx, ns = mp.ns;
    const int i1 = (k + nx / 2) % nx, j1 = (f + ns / 2) % ns;
    const int i2 = ((nx - k) % nx + nx / 2) % nx, j2 = ((ns - f) % ns + ns / 2) % ns;
    return 0.5 * (mask_shifted(mp, i1, j1) + mask_shifted(mp, i2, j2));
}

// row-support scan: rowmax[k] = max_f |M_sym[k][f]| for k in [0, nx/2]  (float bits, atomicMax)
__host__ __device__ inline void body_mask_rowmax(const MaskParams& mp, unsigned int* rowmax, int k, int fchunk0,
                                                 int fchunk1, int tid, int nthr) {
    float m = 0.f;
    for (int f = fchunk0 + tid; f < fchunk1; f += nthr) m = fmaxf(m, (float)fabs(mask_folded(mp, k, f)));
#ifdef __CUDA_ARCH__
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0 && m > 0.f) atomicMax(rowmax + k, __float_as_uint(m));
#else
    unsigned int u; memcpy(&u, &m, 4);
    if (u > rowmax[k]) rowmax[k] = u;
#endif
}

// transform-order table: tab[slot][kt1][p] = M_sym[act_k[slot]][kt1 + T1*pos2k_row[p]] * scale
__host__ __device__ inline void body_mask_build(const MaskParams& mp, float* tab, const int* act_k, const int* pos2k_row,
                                                int t1, int t2, double scale, size_t idx) {
    const int p = (int)(idx % t2);
    const size_t r = idx / t2;
    const int kt1 = (int)(r % t1);
    const int slot = (int)(r / t1);
    const int f = kt1 + t1 * pos2k_row[p];
    tab[idx] = (float)(mask_folded(mp, act_k[slot], f) * scale);
}

// ------------------------------------------------------------------ async copy helpers
#ifdef __CUDACC__
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }
#endif

// ------------------------------------------------------------------ P1: column forward (R2C over channels)
// slot_pos[slot] = (smem position of wavenumber k, position of nx-k) after the forward stages.
__host__ __device__ inline void body_col_fwd(const ColParams& cp, const float* __restrict__ x, float2* __restrict__ w,
                                             size_t ldw, const int2* __restrict__ slot_pos, int nact,
                                             const float* __restrict__ taper, int bx, int tid, int nthr, float2* smem) {
    const int nc = cp.nc, sh = cp.nc_shift, ns = cp.ns, nx = cp.nx;
    const int t0 = bx * 2 * nc;
    bool staged = false;
#ifdef __CUDA_ARCH__
    if (cp.aligned && t0 + 2 * nc <= ns) {
        // whole tile in flight at once: one 8-byte async copy per (channel, column), no register staging
        for (int i = tid; i < (nx << sh); i += nthr) {
            const int c = i >> sh, col = i & (nc - 1);
            cp_async8(smem + col * cp.fstride + c, x + (size_t)c * ns + t0 + 2 * col);
        }
        cp_async_wait_all();
        __syncthreads();
        if (taper) {
            for (int i = tid; i < (nx << sh); i += nthr) {
                const int c = i >> sh, col = i & (nc - 1);
                const int t = t0 + 2 * col;
                float2 v = smem[col * cp.fstride + c];
                v.x *= taper[t]; v.y *= taper[t + 1];
                smem[col * cp.fstride + c] = v;
            }
            __syncthreads();
        }
        staged = true;
    }
#endif
    if (!staged) {
        for (int i = tid; i < (nx << sh); i += nthr) {
            const int c = i >> sh, col = i & (nc - 1);
            const int t = t0 + 2 * col;
            const float* row = x + (size_t)c * ns;
            float a = 0.f, b = 0.f;
            if (t + 1 < ns) {
                if (cp.aligned) { const float2 v = *reinterpret_cast<const float2*>(row + t); a = v.x; b = v.y; }
                else { a = row[t]; b = row[t + 1]; }
                if (taper) { a *= taper[t]; b *= taper[t + 1]; }
            } else if (t < ns) {
                a = row[t];
                if (taper) a *= taper[t];
            }
            smem[col * cp.fstride + c] = make_float2(a, b);
        }
        D4W_SYNC();
    }
    fft_forward_stages(smem, cp.pl, cp.tw, nc, cp.fstride, tid, nthr, 0, cp.pl.nstages);
    // two-for-one untangle: column z = x_t + i*x_{t+1}  ->  X_t[k], X_{t+1}[k] for the kept rows
    for (int i = tid; i < (nact << sh); i += nthr) {
        const int slot = i >> sh, col = i & (nc - 1);
        const int2 pp = slot_pos[slot];
        const float2 z = smem[col * cp.fstride + pp.x], z2 = smem[col * cp.fstride + pp.y];
        const float2 xa = make_float2(0.5f * (z.x + z2.x), 0.5f * (z.y - z2.y));   // (z + conj z2)/2
        const float2 xb = make_float2(0.5f * (z.y + z2.y), 0.5f * (z2.x - z.x));   // (z - conj z2)/(2i)
        const int t = t0 + 2 * col;
        float2* o = w + (size_t)slot * ldw + t;
        if (cp.aligned && t + 1 < ns) {
            *reinterpret_cast<float4*>(o) = make_float4(xa.x, xa.y, xb.x, xb.y);
        } else {
            if (t < ns) o[0] = xa;
            if (t + 1 < ns) o[1] = xb;
        }
    }
}

// ------------------------------------------------------------------ P5: column inverse (C2R over channels)
__host__ __device__ inline void body_col_inv(const ColParams& cp, const float2* __restrict__ w, size_t ldw,
                                             const int2* __restrict__ slot_pos, int nact, float* __restrict__ y, int bx,
                                             int tid, int nthr, float2* smem) {
    const int nc = cp.nc, sh = cp.nc_shift, ns = cp.ns, nx = cp.nx;
    const int t0 = bx * 2 * nc;
    // pruned rows are zero: clear the tile, then scatter only the kept rows and their conjugate partners
    for (int i = tid; i < nc * cp.fstride; i += nthr) smem[i] = make_float2(0.f, 0.f);
    D4W_SYNC();
    for (int i = tid; i < (nact << sh); i += nthr) {
        const int slot = i >> sh, col = i & (nc - 1);
        const int2 pp = slot_pos[slot];
        const int t = t0 + 2 * col;
        const float2* src = w + (size_t)slot * ldw + t;
        float2 y0 = make_float2(0.f, 0.f), y1 = make_float2(0.f, 0.f);
        if (cp.aligned && t + 1 < ns) {
            const float4 v = *reinterpret_cast<const float4*>(src);
            y0 = make_float2(v.x, v.y); y1 = make_float2(v.z, v.w);
        } else {
            if (t < ns) y0 = src[0];
            if (t + 1 < ns) y1 = src[1];
        }
        if (pp.x == pp.y) {                                   // self-conjugate rows (k = 0, nx/2) are real
            smem[col * cp.fstride + pp.x] = make_float2(y0.x, y1.x);
        } else {
            smem[col * cp.fstride + pp.x] = make_float2(y0.x - y1.y, y0.y + y1.x);   // Y_t + i Y_{t+1}
            smem[col * cp.fstride + pp.y] = make_float2(y0.x + y1.y, y1.x - y0.y);   // conj(Y_t) + i conj(Y_{t+1})
        }
    }
    D4W_SYNC();
    fft_inverse_stages(smem, cp.pl, cp.tw, nc, cp.fstride, tid, nthr, 0, cp.pl.nstages);
    for (int i = tid; i < (nx << sh); i += nthr) {
        const int c = i >> sh, col = i & (nc - 1);
        const float2 z = smem[col * cp.fstride + c];
        const int t = t0 + 2 * col;
        float* row = y + (size_t)c * ns;
        if (t + 1 < ns) {
            if (cp.aligned) *reinterpret_cast<float2*>(row + t) = z;
            else { row[t] = z.x; row[t + 1] = z.y; }
        } else if (t < ns) {
            row[t] = z.x;
        }
    }
}


// ================================================================== dual-lane column passes (f32x2)
// Tile = 4*npair time samples.  Pair pr of channel c holds samples t = t0 + 4*pr + {0,1,2,3} as the
// 16-byte element {a0, a1, a2, a3} = cpd{x = (a0, a1), y = (a2, a3)}: lane A is the complex column
// a0 + i*a2 (samples t, t+2), lane B is a1 + i*a3 (samples t+1, t+3) -- exactly the memory image of
// the row, so the load is one 16-byte cp.async and the store one 16-byte st per channel.
__host__ __device__ inline void body_col_fwd_dual(const ColParams& cp, const float* __restrict__ x, float2* __restrict__ w,
                                                  size_t ldw, const int2* __restrict__ slot_pos, int nact,
                                                  const float* __restrict__ taper, int bx, int tid, int nthr, cpd* smem) {
    const int np = cp.npair, sh = cp.npair_shift, ns = cp.ns, nx = cp.nx;
    const int t0 = bx * 4 * np;
    bool staged = false;
#ifdef __CUDA_ARCH__
    if (cp.aligned16 && t0 + 4 * np <= ns) {
        for (int i = tid; i < (nx << sh); i += nthr) {
            const int c = i >> sh, pr = i & (np - 1);
            cp_async16(smem + pr * cp.fstride + c, x + (size_t)c * ns + t0 + 4 * pr);
        }
        cp_async_wait_all();
        __syncthreads();
        if (taper) {
            for (int i = tid; i < (nx << sh); i += nthr) {
                const int c = i >> sh, pr = i & (np - 1);
                const int t = t0 + 4 * pr;
                cpd v = smem[pr * cp.fstride + c];
                v.x = vmul(v.x, f2x_set(taper[t], taper[t + 1]));
                v.y = vmul(v.y, f2x_set(taper[t + 2], taper[t + 3]));
                smem[pr * cp.fstride + c] = v;
            }
            __syncthreads();
        }
        staged = true;
    }
#endif
    if (!staged) {
        for (int i = tid; i < (nx << sh); i += nthr) {
            const int c = i >> sh, pr = i & (np - 1);
            const int t = t0 + 4 * pr;
            const float* row = x + (size_t)c * ns;
            float a[4];
            for (int q = 0; q < 4; ++q) {
                a[q] = (t + q < ns) ? row[t + q] : 0.f;
                if (taper && t + q < ns) a[q] *= taper[t + q];
            }
            smem[pr * cp.fstride + c] = dmake(f2x_set(a[0], a[1]), f2x_set(a[2], a[3]));
        }
        D4W_SYNC();
    }
    fft_forward_stages_dual(smem, cp.pl, cp.tw, np, cp.fstride, tid, nthr);
    const f2x half = vbc(0.5f);
    for (int i = tid; i < (nact << sh); i += nthr) {
        const int slot = i >> sh, pr = i & (np - 1);
        const int2 pp = slot_pos[slot];
        const cpd z = smem[pr * cp.fstride + pp.x], z2 = smem[pr * cp.fstride + pp.y];
        // lane-wise two-for-one untangle: Xa = (z + conj z2)/2, Xb = (z - conj z2)/(2i)
        const cpd xa = dmake(vmul(vadd(z.x, z2.x), half), vmul(vsub(z.y, z2.y), half));
        const cpd xb = dmake(vmul(vadd(z.y, z2.y), half), vmul(vsub(z2.x, z.x), half));
        const int t = t0 + 4 * pr;
        float2* o = w + (size_t)slot * ldw + t;
        // lane A of xa -> sample t, lane B of xa -> t+1, lane A of xb -> t+2, lane B of xb -> t+3
        const float2 o0 = make_float2(f2x_lo(xa.x), f2x_lo(xa.y)), o1 = make_float2(f2x_hi(xa.x), f2x_hi(xa.y));
        const float2 o2 = make_float2(f2x_lo(xb.x), f2x_lo(xb.y)), o3 = make_float2(f2x_hi(xb.x), f2x_hi(xb.y));
        if (cp.aligned16 && t + 3 < ns) {
            reinterpret_cast<float4*>(o)[0] = make_float4(o0.x, o0.y, o1.x, o1.y);
            reinterpret_cast<float4*>(o)[1] = make_float4(o2.x, o2.y, o3.x, o3.y);
        } else {
            if (t < ns) o[0] = o0;
            if (t + 1 < ns) o[1] = o1;
            if (t + 2 < ns) o[2] = o2;
            if (t + 3 < ns) o[3] = o3;
        }
    }
}

__host__ __device__ inline void body_col_inv_dual(const ColParams& cp, const float2* __restrict__ w, size_t ldw,
                                                  const int2* __restrict__ slot_pos, int nact, float* __restrict__ y, int bx,
                                                  int tid, int nthr, cpd* smem) {
    const int np = cp.npair, sh = cp.npair_shift, ns = cp.ns, nx = cp.nx;
    const int t0 = bx * 4 * np;
    const cpd zero = dmake(vbc(0.f), vbc(0.f));
    for (int i = tid; i < np * cp.fstride; i += nthr) smem[i] = zero;
    D4W_SYNC();
    for (int i = tid; i < (nact << sh); i += nthr) {
        const int slot = i >> sh, pr = i & (np - 1);
        const int2 pp = slot_pos[slot];
        const int t = t0 + 4 * pr;
        const float2* src = w + (size_t)slot * ldw + t;
        float2 y0 = make_float2(0.f, 0.f), y1 = y0, y2 = y0, y3 = y0;
        if (cp.aligned16 && t + 3 < ns) {
            const float4 u = reinterpret_cast<const float4*>(src)[0], v = reinterpret_cast<const float4*>(src)[1];
            y0 = make_float2(u.x, u.y); y1 = make_float2(u.z, u.w); y2 = make_float2(v.x, v.y); y3 = make_float2(v.z, v.w);
        } else {
            if (t < ns) y0 = src[0];
            if (t + 1 < ns) y1 = src[1];
            if (t + 2 < ns) y2 = src[2];
            if (t + 3 < ns) y3 = src[3];
        }
        // lane A: Y_t + i Y_{t+2};  lane B: Y_{t+1} + i Y_{t+3}
        if (pp.x == pp.y) {                                   // self-conjugate rows are real
            smem[pr * cp.fstride + pp.x] = dmake(f2x_set(y0.x, y1.x), f2x_set(y2.x, y3.x));
        } else {
            smem[pr * cp.fstride + pp.x] = dmake(f2x_set(y0.x - y2.y, y1.x - y3.y), f2x_set(y0.y + y2.x, y1.y + y3.x));
            smem[pr * cp.fstride + pp.y] = dmake(f2x_set(y0.x + y2.y, y1.x + y3.y), f2x_set(y2.x - y0.y, y3.x - y1.y));
        }
    }
    D4W_SYNC();
    fft_inverse_stages_dual(smem, cp.pl, cp.tw, np, cp.fstride, tid, nthr);
    for (int i = tid; i < (nx << sh); i += nthr) {
        const int c = i >> sh, pr = i & (np - 1);
        const cpd z = smem[pr * cp.fstride + c];
        const int t = t0 + 4 * pr;
        float* row = y + (size_t)c * ns + t;
        if (cp.aligned16 && t + 3 < ns) {
            *reinterpret_cast<float4*>(row) = make_float4(f2x_lo(z.x), f2x_hi(z.x), f2x_lo(z.y), f2x_hi(z.y));
        } else {
            if (t < ns) row[0] = f2x_lo(z.x);
            if (t + 1 < ns) row[1] = f2x_hi(z.x);
            if (t + 2 < ns) row[2] = f2x_lo(z.y);
            if (t + 3 < ns) row[3] = f2x_hi(z.y);
        }
    }
}

// ================================================================== chirp-z column passes (nx with a prime factor > 61)
// X[k] = c[k] * sum_n (x[n] c[n]) b[k - n] with c[n] = exp(-i pi n^2 / nx) and b = conj(c): the sum is a circular
// convolution of length M >= 2 nx - 1, done as FFT_M -> x bhat -> IFFT_M with the shared-memory engine (bhat = FFT_M(b) / M
// in transform order, so no reordering).  The inverse DFT is the same with every chirp conjugated (bhat -> conj bhat, as
// b is even).  Same tile (2*nc time samples, nc complex columns) and kept-row slot layout as body_col_fwd / body_col_inv;
// slot_pos holds natural wavenumbers (k, nx - k).
struct CztParams {
    FftPlan pl;            // length M
    const float2* tw;      // W_M^j
    const float2* chirp;   // c[n], n < nx
    const float2* bhat;    // FFT_M(b) / M, transform order
    int nx, ns, m;
    int nc, nc_shift, fstride, aligned;
};

__host__ __device__ inline void czt_convolve(const CztParams& cp, float2* smem, bool conj_kernel, int tid, int nthr) {
    const int nc = cp.nc, sh = cp.nc_shift;
    fft_forward_stages(smem, cp.pl, cp.tw, nc, cp.fstride, tid, nthr, 0, cp.pl.nstages);
    for (int i = tid; i < (cp.m << sh); i += nthr) {
        const int p = i >> sh, col = i & (nc - 1);
        float2& v = smem[col * cp.fstride + p];
        v = conj_kernel ? cmulc(v, cp.bhat[p]) : cmul(v, cp.bhat[p]);
    }
    D4W_SYNC();
    fft_inverse_stages(smem, cp.pl, cp.tw, nc, cp.fstride, tid, nthr, 0, cp.pl.nstages);
}

__host__ __device__ inline void body_col_fwd_czt(const CztParams& cp, const float* __restrict__ x, float2* __restrict__ w,
                                                 size_t ldw, const int2* __restrict__ slot_pos, int nact,
                                                 const float* __restrict__ taper, int bx, int tid, int nthr, float2* smem) {
    const int nc = cp.nc, sh = cp.nc_shift, ns = cp.ns, nx = cp.nx;
    const int t0 = bx * 2 * nc;
    // two real time columns as one complex column z = x_t + i x_{t+1}, tapered, times c[n], zero-padded to M
    for (int i = tid; i < (cp.m << sh); i += nthr) {
        const int c = i >> sh, col = i & (nc - 1);
        const int t = t0 + 2 * col;
        float a = 0.f, b = 0.f;
        if (c < nx) {
            const float* row = x + (size_t)c * ns;
            if (t + 1 < ns) {
                if (cp.aligned) { const float2 v = *reinterpret_cast<const float2*>(row + t); a = v.x; b = v.y; }
                else { a = row[t]; b = row[t + 1]; }
                if (taper) { a *= taper[t]; b *= taper[t + 1]; }
            } else if (t < ns) {
                a = row[t];
                if (taper) a *= taper[t];
            }
        }
        smem[col * cp.fstride + c] = c < nx ? cmul(make_float2(a, b), cp.chirp[c]) : make_float2(0.f, 0.f);
    }
    D4W_SYNC();
    czt_convolve(cp, smem, false, tid, nthr);
    // Z[k] = c[k] * conv[k]; two-for-one untangle as in body_col_fwd
    for (int i = tid; i < (nact << sh); i += nthr) {
        const int slot = i >> sh, col = i & (nc - 1);
        const int2 pp = slot_pos[slot];
        const float2 z = cmul(smem[col * cp.fstride + pp.x], cp.chirp[pp.x]);
        const float2 z2 = cmul(smem[col * cp.fstride + pp.y], cp.chirp[pp.y]);
        const float2 xa = make_float2(0.5f * (z.x + z2.x), 0.5f * (z.y - z2.y));   // (z + conj z2)/2
        const float2 xb = make_float2(0.5f * (z.y + z2.y), 0.5f * (z2.x - z.x));   // (z - conj z2)/(2i)
        const int t = t0 + 2 * col;
        float2* o = w + (size_t)slot * ldw + t;
        if (cp.aligned && t + 1 < ns) {
            *reinterpret_cast<float4*>(o) = make_float4(xa.x, xa.y, xb.x, xb.y);
        } else {
            if (t < ns) o[0] = xa;
            if (t + 1 < ns) o[1] = xb;
        }
    }
}

__host__ __device__ inline void body_col_inv_czt(const CztParams& cp, const float2* __restrict__ w, size_t ldw,
                                                 const int2* __restrict__ slot_pos, int nact, float* __restrict__ y, int bx,
                                                 int tid, int nthr, float2* smem) {
    const int nc = cp.nc, sh = cp.nc_shift, ns = cp.ns, nx = cp.nx;
    const int t0 = bx * 2 * nc;
    // pruned rows (and the padding up to M) are zero
    for (int i = tid; i < nc * cp.fstride; i += nthr) smem[i] = make_float2(0.f, 0.f);
    D4W_SYNC();
    // Z[k] = Y_t[k] + i Y_{t+1}[k] over the full k range (Hermitian partners k -> nx - k), times conj(c[k])
    for (int i = tid; i < (nact << sh); i += nthr) {
        const int slot = i >> sh, col = i & (nc - 1);
        const int2 pp = slot_pos[slot];
        const int t = t0 + 2 * col;
        const float2* src = w + (size_t)slot * ldw + t;
        float2 y0 = make_float2(0.f, 0.f), y1 = make_float2(0.f, 0.f);
        if (cp.aligned && t + 1 < ns) {
            const float4 v = *reinterpret_cast<const float4*>(src);
            y0 = make_float2(v.x, v.y); y1 = make_float2(v.z, v.w);
        } else {
            if (t < ns) y0 = src[0];
            if (t + 1 < ns) y1 = src[1];
        }
        if (pp.x == pp.y) {                                   // self-conjugate rows (k = 0, nx/2) are real
            smem[col * cp.fstride + pp.x] = cmulc(make_float2(y0.x, y1.x), cp.chirp[pp.x]);
        } else {
            smem[col * cp.fstride + pp.x] = cmulc(make_float2(y0.x - y1.y, y0.y + y1.x), cp.chirp[pp.x]);
            smem[col * cp.fstride + pp.y] = cmulc(make_float2(y0.x + y1.y, y1.x - y0.y), cp.chirp[pp.y]);
        }
    }
    D4W_SYNC();
    czt_convolve(cp, smem, true, tid, nthr);
    // z[n] = conj(c[n]) * conv[n]: real part -> sample t, imaginary part -> t + 1
    for (int i = tid; i < (nx << sh); i += nthr) {
        const int c = i >> sh, col = i & (nc - 1);
        const float2 z = cmulc(smem[col * cp.fstride + c], cp.chirp[c]);
        const int t = t0 + 2 * col;
        float* row = y + (size_t)c * ns;
        if (t + 1 < ns) {
            if (cp.aligned) *reinterpret_cast<float2*>(row + t) = z;
            else { row[t] = z.x; row[t + 1] = z.y; }
        } else if (t < ns) {
            row[t] = z.x;
        }
    }
}

// ------------------------------------------------------------------ P2 / P4: radix-T1 time split (registers only)
template <int T1, bool INV>
__host__ __device__ inline void body_row_split(float2* __restrict__ w, size_t ldw, int t2len, const float2* __restrict__ twT,
                                               int slot, int t2) {
    float2* base = w + (size_t)slot * ldw + t2;
    float2 v[T1];
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; v[j] = base[(size_t)j * t2len]; });
    float2 p[T1];
    twiddle_powers<T1>(twT[t2], p);
    if constexpr (!INV) {
        DFT<T1, false>::run(v);
        static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; if constexpr (j > 0) v[j] = cmul(v[j], p[j]); });
    } else {
        static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; if constexpr (j > 0) v[j] = cmulc(v[j], p[j]); });
        DFT<T1, true>::run(v);
    }
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; base[(size_t)j * t2len] = v[j]; });
}

// ------------------------------------------------------------------ P3: FFT(T2) -> x table -> IFFT(T2)
// `tab` is indexed [slot*tab_slot_stride + kt1*T2 + p] in transform (digit-reversed) order;
// tab_slot_stride = 0 shares one table between all rows (Hilbert weights, template spectra).
// TabT = float2 (the chirp-z Hilbert rows' kernel spectrum): the table multiplies instead of scaling.
template <typename TabT>
__host__ __device__ inline void body_row_mid(const RowParams& rp, float2* __restrict__ w, size_t ldw,
                                             const TabT* __restrict__ tab, size_t tab_slot_stride, int kt1, int slot,
                                             int tid, int nthr, float2* smem) {
    const int n = rp.t2;
    float2* g = w + (size_t)slot * ldw + (size_t)kt1 * n;
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
    const TabT* m = tab + (size_t)slot * tab_slot_stride + (size_t)kt1 * n;
    if constexpr (std::is_same<TabT, float>::value) {
        for (int i = tid; i < n; i += nthr) { const float s = m[i]; float2 v = smem[i]; v.x *= s; v.y *= s; smem[i] = v; }
    } else {
        for (int i = tid; i < n; i += nthr) smem[i] = cmul(smem[i], m[i]);
    }
    D4W_SYNC();
    fft_inverse_stages(smem, rp.pl, rp.tw, 1, n, tid, nthr, 0, rp.pl.nstages);
    for (int i = tid; i < n; i += nthr) g[i] = smem[i];
}


// ------------------------------------------------------------------ P3 dual: two kept rows per CTA as f32x2 lanes
// Rows slotA = 2*pair, slotB = slotA + 1 (same kt1 tile) are interleaved on the way into shared memory
// ({reA, reB, imA, imB} per sample), share every butterfly / twiddle, and each lane is multiplied by its
// own row of the mask table.  An odd trailing row runs with lane B = 0.
__host__ __device__ inline void body_row_mid_dual(const RowParams& rp, float2* __restrict__ w, size_t ldw,
                                                  const float* __restrict__ tab, size_t tab_slot_stride, int kt1, int pair,
                                                  int nslots, int tid, int nthr, cpd* smem) {
    const int n = rp.t2;
    const int sa = 2 * pair, sb = sa + 1;
    const bool has_b = sb < nslots;
    float2* ga = w + (size_t)sa * ldw + (size_t)kt1 * n;
    float2* gb = w + (size_t)(has_b ? sb : sa) * ldw + (size_t)kt1 * n;
#pragma unroll 8
    for (int i = tid; i < n; i += nthr) {
        const float2 a = ga[i];
        const float2 b = has_b ? gb[i] : make_float2(0.f, 0.f);
        smem[i] = dmake(f2x_set(a.x, b.x), f2x_set(a.y, b.y));
    }
    D4W_SYNC();
    fft_forward_stages_dual(smem, rp.pl, rp.tw, 1, n, tid, nthr);
    const float* ma = tab + (size_t)sa * tab_slot_stride + (size_t)kt1 * n;
    const float* mb = tab + (size_t)(has_b ? sb : sa) * tab_slot_stride + (size_t)kt1 * n;
#pragma unroll 4
    for (int i = tid; i < n; i += nthr) {
        const f2x m = f2x_set(ma[i], mb[i]);
        cpd v = smem[i];
        v.x = vmul(v.x, m); v.y = vmul(v.y, m);
        smem[i] = v;
    }
    D4W_SYNC();
    fft_inverse_stages_dual(smem, rp.pl, rp.tw, 1, n, tid, nthr);
    for (int i = tid; i < n; i += nthr) {
        const cpd v = smem[i];
        ga[i] = make_float2(f2x_lo(v.x), f2x_lo(v.y));
        if (has_b) gb[i] = make_float2(f2x_hi(v.x), f2x_hi(v.y));
    }
}


// ================================================================== two-level column transform (nx = X1 * X2)
// Channel c = X2*c1 + c2, wavenumber k = k1 + X1*k2:
//   level A: radix-X1 DFT over c1 (rows X2 apart) entirely in registers, times W_nx^{c2 k1}      (streaming)
//   level B: X2-point FFT over c2 in shared memory, wide coalesced tiles, several CTAs per SM
// Real input => only planes k1 = 0..X1/2 of the intermediate V are stored (Hermitian in k1), and the
// outputs of plane X1-k1 are conj(P_{k1}[X2-1-k2]) of the same level-B transform, so each kept
// wavenumber row is produced exactly once.  V[plane][c2][sample pair] holds 16-byte elements
// {re_t, re_t+1, im_t, im_t+1}.  Forward: A then B (pruned rows out); inverse: B then A.
struct Col2Params {
    FftPlan plb;             // X2-point plan (dual lanes)
    const float2* twb;       // W_X2^j
    const float2* twn;       // W_nx^j
    int nx, ns, x1, x2, planes, np, fstride;
    int np_shift;            // np is a power of two
    // time chunk handled by one level-A/level-B launch pair: sample pairs [tpb, tpb + tpn) of the record; the
    // intermediate V holds just this chunk (row stride vhp pairs) so that it stays resident in L2 between the two
    int vhp, tpb, tpn;
};

// ---- global-memory access with an L2 eviction policy (pipelined level A/B kernel) -------------------------------
// `keep` (evict_last) is used for the chunk ring of the intermediate V, which must survive in L2 from its producer
// CTA to its consumer CTA; `stream` (evict_first) for data touched once (x, y, the kept rows W).  V is read with
// .cg so that a re-used ring slot can never be served from a stale L1 line.
struct L2Pol { unsigned long long keep, stream; };
#ifdef __CUDACC__
__device__ __forceinline__ L2Pol make_l2pol(bool hints) {
    L2Pol p;
    if (hints) {
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p.keep));
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p.stream));
    } else {
        asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p.keep));
        p.stream = p.keep;
    }
    return p;
}
__device__ __forceinline__ float4 ldg16_pol(const void* p, unsigned long long pol) {
    float4 r;
    asm volatile("ld.global.cg.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol) : "memory");
    return r;
}
__device__ __forceinline__ void stg16_pol(void* p, float4 v, unsigned long long pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
#endif
template <bool PIPE> D4W_HD float4 ld16(const void* p, unsigned long long pol) {
#ifdef __CUDA_ARCH__
    if constexpr (PIPE) return ldg16_pol(p, pol);
#endif
    (void)pol;
    return *reinterpret_cast<const float4*>(p);
}
template <bool PIPE> D4W_HD void st16(void* p, float4 v, unsigned long long pol) {
#ifdef __CUDA_ARCH__
    if constexpr (PIPE) { stg16_pol(p, v, pol); return; }
#endif
    (void)pol;
    *reinterpret_cast<float4*>(p) = v;
}
template <bool PIPE> D4W_HD cpd ldc(const cpd* p, unsigned long long pol) {
    const float4 u = ld16<PIPE>(p, pol);
    return dmake(f2x_set(u.x, u.y), f2x_set(u.z, u.w));
}
template <bool PIPE> D4W_HD void stc(cpd* p, cpd z, unsigned long long pol) {
    st16<PIPE>(p, make_float4(f2x_lo(z.x), f2x_hi(z.x), f2x_lo(z.y), f2x_hi(z.y)), pol);
}

struct Col2Entry { int pos, slot, flags, pad; };     // flags bit0: conjugate, bit1: stored by the forward pass

template <int X1, bool PIPE = false>
__host__ __device__ inline void body_colA_fwd(const Col2Params& cp, const float* __restrict__ x, cpd* __restrict__ v2,
                                              const float* __restrict__ taper, int c2, int t4, int tpb, L2Pol pol = L2Pol{0, 0}) {
    const int ns = cp.ns, x2 = cp.x2;
    const size_t hp = (size_t)cp.vhp;
    const size_t tg = 4 * (size_t)(tpb / 2 + t4);      // first of this thread's four samples in the record
    cpd v[X1];
    float2 twp[X1 / 2 + 1];                                          // W_nx^{c2 k1}, k1 = 0 .. X1/2, from one table read
    twiddle_powers<X1 / 2 + 1>(cp.twn[c2], twp);
    // window (Tukey taper) of the four samples; 1.0 when not tapering: an unconditional multiply is exact and cheaper than
    // selecting between tapered and untapered registers
    f2x wa = vbc(1.f), wb = vbc(1.f);
    if (taper) { wa = f2x_set(taper[tg], taper[tg + 1]); wb = f2x_set(taper[tg + 2], taper[tg + 3]); }
    static_for<X1>([&](auto c1c) {
        constexpr int c1 = decltype(c1c)::value;
        const float4 a = ld16<PIPE>(x + (size_t)(x2 * c1 + c2) * ns + tg, pol.stream);
        v[c1] = dmake(vmul(f2x_set(a.x, a.y), wa), vmul(f2x_set(a.z, a.w), wb));
    });
    DFTD<X1, false>::run(v);
    const f2x half = vbc(0.5f);
    static_for<X1 / 2 + 1>([&](auto kc) {
        constexpr int k1 = decltype(kc)::value;
        const cpd z = v[outpos<X1>(k1)], z2 = v[outpos<X1>((X1 - k1) % X1)];
        // F_t, F_t+1 (fa) and F_t+2, F_t+3 (fb) = halves of the sum / difference; the 1/2 rides on the twiddle for k1 > 0
        cpd fa = dmake(vadd(z.x, z2.x), vsub(z.y, z2.y));
        cpd fb = dmake(vadd(z.y, z2.y), vsub(z2.x, z.x));
        if constexpr (k1 > 0) {
            const float2 w = make_float2(0.5f * twp[k1].x, 0.5f * twp[k1].y);
            fa = dmul_s(fa, w); fb = dmul_s(fb, w);
        } else {
            fa = dmake(vmul(fa.x, half), vmul(fa.y, half)); fb = dmake(vmul(fb.x, half), vmul(fb.y, half));
        }
        cpd* o = v2 + ((size_t)k1 * x2 + c2) * hp + 2 * t4;
        stc<PIPE>(o, fa, pol.keep); stc<PIPE>(o + 1, fb, pol.keep);
    });
}
template <int X1, bool PIPE = false>
__host__ __device__ inline void body_colA_inv(const Col2Params& cp, const cpd* __restrict__ v2, float* __restrict__ y, int c2, int t4,
                                              int tpb, L2Pol pol = L2Pol{0, 0}) {
    const int ns = cp.ns, x2 = cp.x2;
    const size_t hp = (size_t)cp.vhp;
    const size_t tg = 4 * (size_t)(tpb / 2 + t4);
    cpd v[X1];
    float2 twp[X1 / 2 + 1];
    twiddle_powers<X1 / 2 + 1>(cp.twn[c2], twp);
    static_for<X1 / 2 + 1>([&](auto kc) {
        constexpr int k1 = decltype(kc)::value;
        const cpd* in = v2 + ((size_t)k1 * x2 + c2) * hp + 2 * t4;
        cpd fa = ldc<PIPE>(in, pol.keep), fb = ldc<PIPE>(in + 1, pol.keep);
        if (k1 > 0) { const float2 w = twp[k1]; fa = dmulc_s(fa, w); fb = dmulc_s(fb, w); }
        if (k1 == 0 || 2 * k1 == X1) {                       // self-conjugate in k1: real
            v[k1] = dmake(fa.x, fb.x);
        } else {
            v[k1] = dmake(vsub(fa.x, fb.y), vadd(fa.y, fb.x));            // F_a + i F_b
            v[X1 - k1] = dmake(vadd(fa.x, fb.y), vsub(fb.x, fa.y));       // conj(F_a) + i conj(F_b)
        }
    });
    DFTD<X1, true>::run(v);
    static_for<X1>([&](auto c1c) {
        constexpr int c1 = decltype(c1c)::value;
        const cpd z = v[outpos<X1>(c1)];
        st16<PIPE>(y + (size_t)(x2 * c1 + c2) * ns + tg, make_float4(f2x_lo(z.x), f2x_hi(z.x), f2x_lo(z.y), f2x_hi(z.y)), pol.stream);
    });
}

// level B forward: one plane, np consecutive sample pairs; writes the kept wavenumber rows
__host__ __device__ inline void body_colB_fwd(const Col2Params& cp, const cpd* __restrict__ v2, float2* __restrict__ w, size_t ldw,
                                              const int* __restrict__ plane_ptr, const Col2Entry* __restrict__ ents, int plane,
                                              int tile, int tid, int nthr, cpd* smem) {
    const int x2 = cp.x2, np = cp.np, hp = cp.vhp, tpn = cp.tpn;
    const int tp0 = tile * np;
    const cpd zero = dmake(vbc(0.f), vbc(0.f));
    const int sh = cp.np_shift;
    for (int i = tid; i < (x2 << sh); i += nthr) {
        const int c2 = i >> sh, j = i & (np - 1);
        const cpd* src = v2 + ((size_t)plane * x2 + c2) * hp + tp0 + j;
#ifdef __CUDA_ARCH__
        if (tp0 + j < tpn) cp_async16(smem + j * cp.fstride + c2, src); else smem[j * cp.fstride + c2] = zero;
#else
        smem[j * cp.fstride + c2] = (tp0 + j < tpn) ? *src : zero;
#endif
    }
#ifdef __CUDA_ARCH__
    cp_async_wait_all();
#endif
    D4W_SYNC();
    fft_forward_stages_dual(smem, cp.plb, cp.twb, np, cp.fstride, tid, nthr);
    const int e0 = plane_ptr[plane], ne = plane_ptr[plane + 1] - e0;
    for (int i = tid; i < (ne << sh); i += nthr) {
        const int ei = i >> sh, j = i & (np - 1);
        const Col2Entry e = ents[e0 + ei];
        if (!(e.flags & 2) || tp0 + j >= tpn) continue;
        cpd v = smem[j * cp.fstride + e.pos];
        if (e.flags & 1) v.y = vneg(v.y);
        *reinterpret_cast<float4*>(w + (size_t)e.slot * ldw + 2 * (size_t)(cp.tpb + tp0 + j)) = make_float4(f2x_lo(v.x), f2x_lo(v.y), f2x_hi(v.x), f2x_hi(v.y));
    }
}

// level B inverse: kept rows -> plane of V
__host__ __device__ inline void body_colB_inv(const Col2Params& cp, cpd* __restrict__ v2, const float2* __restrict__ w, size_t ldw,
                                              const int* __restrict__ plane_ptr, const Col2Entry* __restrict__ ents, int plane,
                                              int tile, int tid, int nthr, cpd* smem) {
    const int x2 = cp.x2, np = cp.np, hp = cp.vhp, tpn = cp.tpn;
    const int tp0 = tile * np;
    const cpd zero = dmake(vbc(0.f), vbc(0.f));
    for (int i = tid; i < np * cp.fstride; i += nthr) smem[i] = zero;
    D4W_SYNC();
    const int e0 = plane_ptr[plane], ne = plane_ptr[plane + 1] - e0;
    const int sh = cp.np_shift;
    for (int i = tid; i < (ne << sh); i += nthr) {
        const int ei = i >> sh, j = i & (np - 1);
        if (tp0 + j >= tpn) continue;
        const Col2Entry e = ents[e0 + ei];
        const float4 u = *reinterpret_cast<const float4*>(w + (size_t)e.slot * ldw + 2 * (size_t)(cp.tpb + tp0 + j));
        cpd v = dmake(f2x_set(u.x, u.z), f2x_set(u.y, u.w));
        if (e.flags & 1) v.y = vneg(v.y);
        smem[j * cp.fstride + e.pos] = v;
    }
    D4W_SYNC();
    fft_inverse_stages_dual(smem, cp.plb, cp.twb, np, cp.fstride, tid, nthr);
    for (int i = tid; i < (x2 << sh); i += nthr) {
        const int c2 = i >> sh, j = i & (np - 1);
        if (tp0 + j < tpn) v2[((size_t)plane * x2 + c2) * hp + tp0 + j] = smem[j * cp.fstride + c2];
    }
}


// ------------------------------------------------------------------ fused two-stage level B (X2 = RA * RB)
// Stage 0 (radix RA over c2 = n + RB*q) runs straight from global memory in registers, stage 1 (radix RB
// on contiguous groups) writes only the kept wavenumber rows straight to global memory; shared memory is
// used once, for the transposition between the two stages.  need[plane][k2] = (slot of X[k1' + X1*k2] or -1,
// slot whose value is conj(P[k2]): >= 0 both directions, <= -2 encodes -2-slot for the inverse only, -1 none).
template <int RA, int RB, bool PIPE = false>
__host__ __device__ inline void body_colB_fwd_fused(const Col2Params& cp, const cpd* __restrict__ v2, float2* __restrict__ w,
                                                    size_t ldw, const int2* __restrict__ need, int plane, int tile, int tid,
                                                    int nthr, cpd* smem, int tpb, int tpn, L2Pol pol = L2Pol{0, 0}) {
    const int x2 = cp.x2, np = cp.np, sh = cp.np_shift, hp = cp.vhp, fs = cp.fstride;
    const int tp0 = tile * np;
    const cpd zero = dmake(vbc(0.f), vbc(0.f));
    for (int it = tid; it < (RB << sh); it += nthr) {              // item = (n, j)
        const int n = it >> sh, j = it & (np - 1);
        const bool ok = tp0 + j < tpn;
        cpd v[RA];
        const cpd* src = v2 + ((size_t)plane * x2 + n) * hp + tp0 + j;
        static_for<RA>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = ok ? ldc<PIPE>(src + (size_t)(RB * q) * hp, pol.keep) : zero; });
        DFTD<RA, false>::run(v);
        apply_stage_twiddles<RA, false, true>(v, cp.twb[n]);
        cpd* dst = smem + j * fs + n;
        static_for<RA>([&](auto mc) { constexpr int m = decltype(mc)::value; dst[RB * m] = v[outpos<RA>(m)]; });
    }
    D4W_SYNC();
    const int2* nd = need + (size_t)plane * x2;
    for (int it = tid; it < (RA << sh); it += nthr) {              // item = (group m, j)
        const int m = it >> sh, j = it & (np - 1);
        if (tp0 + j >= tpn) continue;
        cpd v[RB];
        const cpd* src = smem + j * fs + RB * m;
        static_for<RB>([&](auto ic) { constexpr int i = decltype(ic)::value; v[i] = src[i]; });
        DFTD<RB, false>::run(v);
        float2* wo = w + 2 * (size_t)(tpb + tp0 + j);
        static_for<RB>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            const int2 e = nd[m + RA * i];
            const cpd z = v[outpos<RB>(i)];
            if (e.x >= 0) st16<PIPE>(wo + (size_t)e.x * ldw, make_float4(f2x_lo(z.x), f2x_lo(z.y), f2x_hi(z.x), f2x_hi(z.y)), pol.stream);
            if (e.y >= 0) st16<PIPE>(wo + (size_t)e.y * ldw, make_float4(f2x_lo(z.x), -f2x_lo(z.y), f2x_hi(z.x), -f2x_hi(z.y)), pol.stream);
        });
    }
}

template <int RA, int RB, bool PIPE = false>
__host__ __device__ inline void body_colB_inv_fused(const Col2Params& cp, cpd* __restrict__ v2, const float2* __restrict__ w,
                                                    size_t ldw, const int2* __restrict__ need, int plane, int tile, int tid,
                                                    int nthr, cpd* smem, int tpb, int tpn, L2Pol pol = L2Pol{0, 0}) {
    const int x2 = cp.x2, np = cp.np, sh = cp.np_shift, hp = cp.vhp, fs = cp.fstride;
    const int tp0 = tile * np;
    const int2* nd = need + (size_t)plane * x2;
    for (int it = tid; it < (RA << sh); it += nthr) {              // item = (group m, j): undo the radix-RB stage
        const int m = it >> sh, j = it & (np - 1);
        const bool ok = tp0 + j < tpn;
        cpd v[RB];
        const float2* wi = w + 2 * (size_t)(tpb + tp0 + j);
        static_for<RB>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            const int2 e = nd[m + RA * i];
            const int sd = e.x, sm = (e.y >= 0) ? e.y : ((e.y <= -2) ? -2 - e.y : -1);
            const int sl = sd >= 0 ? sd : sm;                           // one predicated load, sign applied afterwards
            const float sg = sd >= 0 ? 1.f : -1.f;
            float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok && sl >= 0) u = ld16<PIPE>(wi + (size_t)sl * ldw, pol.stream);
            v[i] = dmake(f2x_set(u.x, u.z), f2x_set(sg * u.y, sg * u.w));
        });
        DFTD<RB, true>::run(v);
        cpd* dst = smem + j * fs + RB * m;
        static_for<RB>([&](auto ic) { constexpr int i = decltype(ic)::value; dst[i] = v[outpos<RB>(i)]; });
    }
    D4W_SYNC();
    for (int it = tid; it < (RB << sh); it += nthr) {              // item = (n, j): undo the radix-RA stage
        const int n = it >> sh, j = it & (np - 1);
        if (tp0 + j >= tpn) continue;
        cpd v[RA];
        const cpd* src = smem + j * fs + n;
        static_for<RA>([&](auto mc) { constexpr int m = decltype(mc)::value; v[m] = src[RB * m]; });
        apply_stage_twiddles<RA, true, false>(v, cp.twb[n]);
        DFTD<RA, true>::run(v);
        cpd* dst = v2 + ((size_t)plane * x2 + n) * hp + tp0 + j;
        static_for<RA>([&](auto qc) { constexpr int q = decltype(qc)::value; stc<PIPE>(dst + (size_t)(RB * q) * hp, v[outpos<RA>(q)], pol.keep); });
    }
}


// ------------------------------------------------------------------ three-stage level B (X2 = R0 * R1 * R2, small radices)
// Same contract as the fused two-stage version (stage 0 from global memory, last stage to the kept rows), with one more
// in-place shared-memory stage in between.  Radices <= 10 keep every butterfly under ~45 data registers, so the pipelined
// kernel built on it (k_col3_pipe, X1 = 10) needs ~70 registers instead of 128 and 21 - 28 warps share an SM instead of 15:
// the round-1 / round-2 profiles show the column kernels bound by latency at low occupancy, not by any one unit.
// Positions follow the engine's decimation in frequency: after the forward stages position m0*L0 + m1*L1 + m2 holds
// k2 = m0 + R0*m1 + R0*R1*m2 (L0 = X2/R0, L1 = R2).
template <int R0, int R1, int R2, bool PIPE = false>
__host__ __device__ inline void body_colB3_fwd(const Col2Params& cp, const cpd* __restrict__ v2, float2* __restrict__ w, size_t ldw,
                                               const int2* __restrict__ need, int plane, int tile, int tid, int nthr, cpd* smem,
                                               int tpb, int tpn, L2Pol pol = L2Pol{0, 0}) {
    constexpr int X2 = R0 * R1 * R2, L0 = X2 / R0, L1 = L0 / R1;
    const int np = cp.np, sh = cp.np_shift, hp = cp.vhp, fs = cp.fstride;
    const int tp0 = tile * np;
    const cpd zero = dmake(vbc(0.f), vbc(0.f));
    for (int it = tid; it < (L0 << sh); it += nthr) {              // stage 0: item (n, j), inputs c2 = n + L0*q
        const int n = it >> sh, j = it & (np - 1);
        const bool ok = tp0 + j < tpn;
        cpd v[R0];
        const cpd* src = v2 + ((size_t)plane * X2 + n) * hp + tp0 + j;
        static_for<R0>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = ok ? ldc<PIPE>(src + (size_t)(L0 * q) * hp, pol.keep) : zero; });
        DFTD<R0, false>::run(v);
        apply_stage_twiddles<R0, false, true>(v, cp.twb[n]);                       // W_X2^{n m}
        cpd* dst = smem + j * fs + n;
        static_for<R0>([&](auto mc) { constexpr int m = decltype(mc)::value; dst[L0 * m] = v[outpos<R0>(m)]; });
    }
    D4W_SYNC();
    for (int it = tid; it < ((R0 * L1) << sh); it += nthr) {        // stage 1: item (b0, n1, j) inside block b0
        const int idx = it >> sh, j = it & (np - 1);
        const int b0 = idx / L1, n1 = idx - b0 * L1;
        cpd* base = smem + j * fs + b0 * L0 + n1;
        cpd v[R1];
        static_for<R1>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = base[L1 * q]; });
        DFTD<R1, false>::run(v);
        apply_stage_twiddles<R1, false, true>(v, cp.twb[R0 * n1]);                  // W_L0^{n1 m} = W_X2^{R0 n1 m}
        static_for<R1>([&](auto mc) { constexpr int m = decltype(mc)::value; base[L1 * m] = v[outpos<R1>(m)]; });
    }
    D4W_SYNC();
    const int2* nd = need + (size_t)plane * X2;
    for (int it = tid; it < ((R0 * R1) << sh); it += nthr) {        // stage 2: contiguous group g = b0*R1 + b1 -> kept rows
        const int g = it >> sh, j = it & (np - 1);
        if (tp0 + j >= tpn) continue;
        const int b0 = g / R1, b1 = g - b0 * R1;
        cpd v[R2];
        const cpd* src = smem + j * fs + g * R2;
        static_for<R2>([&](auto ic) { constexpr int i = decltype(ic)::value; v[i] = src[i]; });
        DFTD<R2, false>::run(v);
        float2* wo = w + 2 * (size_t)(tpb + tp0 + j);
        const int k0 = b0 + R0 * b1;
        static_for<R2>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            const int2 e = nd[k0 + R0 * R1 * i];
            const cpd z = v[outpos<R2>(i)];
            if (e.x >= 0) st16<PIPE>(wo + (size_t)e.x * ldw, make_float4(f2x_lo(z.x), f2x_lo(z.y), f2x_hi(z.x), f2x_hi(z.y)), pol.stream);
            if (e.y >= 0) st16<PIPE>(wo + (size_t)e.y * ldw, make_float4(f2x_lo(z.x), -f2x_lo(z.y), f2x_hi(z.x), -f2x_hi(z.y)), pol.stream);
        });
    }
}

template <int R0, int R1, int R2, bool PIPE = false>
__host__ __device__ inline void body_colB3_inv(const Col2Params& cp, cpd* __restrict__ v2, const float2* __restrict__ w, size_t ldw,
                                               const int2* __restrict__ need, int plane, int tile, int tid, int nthr, cpd* smem,
                                               int tpb, int tpn, L2Pol pol = L2Pol{0, 0}) {
    constexpr int X2 = R0 * R1 * R2, L0 = X2 / R0, L1 = L0 / R1;
    const int np = cp.np, sh = cp.np_shift, hp = cp.vhp, fs = cp.fstride;
    const int tp0 = tile * np;
    const int2* nd = need + (size_t)plane * X2;
    for (int it = tid; it < ((R0 * R1) << sh); it += nthr) {        // undo stage 2: gather the kept rows
        const int g = it >> sh, j = it & (np - 1);
        const bool ok = tp0 + j < tpn;
        const int b0 = g / R1, b1 = g - b0 * R1;
        const int k0 = b0 + R0 * b1;
        cpd v[R2];
        const float2* wi = w + 2 * (size_t)(tpb + tp0 + j);
        static_for<R2>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            const int2 e = nd[k0 + R0 * R1 * i];
            const int sd = e.x, sm = (e.y >= 0) ? e.y : ((e.y <= -2) ? -2 - e.y : -1);
            const int sl = sd >= 0 ? sd : sm;
            const float sg = sd >= 0 ? 1.f : -1.f;
            float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok && sl >= 0) u = ld16<PIPE>(wi + (size_t)sl * ldw, pol.stream);
            v[i] = dmake(f2x_set(u.x, u.z), f2x_set(sg * u.y, sg * u.w));
        });
        DFTD<R2, true>::run(v);
        cpd* dst = smem + j * fs + g * R2;
        static_for<R2>([&](auto ic) { constexpr int i = decltype(ic)::value; dst[i] = v[outpos<R2>(i)]; });
    }
    D4W_SYNC();
    for (int it = tid; it < ((R0 * L1) << sh); it += nthr) {        // undo stage 1
        const int idx = it >> sh, j = it & (np - 1);
        const int b0 = idx / L1, n1 = idx - b0 * L1;
        cpd* base = smem + j * fs + b0 * L0 + n1;
        cpd v[R1];
        static_for<R1>([&](auto mc) { constexpr int m = decltype(mc)::value; v[m] = base[L1 * m]; });
        apply_stage_twiddles<R1, true, false>(v, cp.twb[R0 * n1]);
        DFTD<R1, true>::run(v);
        static_for<R1>([&](auto qc) { constexpr int q = decltype(qc)::value; base[L1 * q] = v[outpos<R1>(q)]; });
    }
    D4W_SYNC();
    for (int it = tid; it < (L0 << sh); it += nthr) {              // undo stage 0 -> plane of V
        const int n = it >> sh, j = it & (np - 1);
        if (tp0 + j >= tpn) continue;
        cpd v[R0];
        const cpd* src = smem + j * fs + n;
        static_for<R0>([&](auto mc) { constexpr int m = decltype(mc)::value; v[m] = src[L0 * m]; });
        apply_stage_twiddles<R0, true, false>(v, cp.twb[n]);
        DFTD<R0, true>::run(v);
        cpd* dst = v2 + ((size_t)plane * X2 + n) * hp + tp0 + j;
        static_for<R0>([&](auto qc) { constexpr int q = decltype(qc)::value; stc<PIPE>(dst + (size_t)(L0 * q) * hp, v[outpos<R0>(q)], pol.keep); });
    }
}

// ---- fused row kernel: first stage straight from global memory, last stage . mask . its inverse in registers ----
// The T2-point piece makes one trip through shared memory per middle stage instead of one per stage plus a mask
// pass.  Table order for this kernel: tab[m * (n / RL) + j] belongs to position j * RL + m of the engine's order.
template <int R>
__host__ __device__ inline void row_first_fwd(const float2* __restrict__ g, float2* __restrict__ s, const float2* __restrict__ tw,
                                              int n_total, int tid, int nthr) {
    const int L = n_total / R;
    for (int n = tid; n < L; n += nthr) {
        float2 v[R];
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = g[n + q * L]; });
        DFT<R, false>::run(v);
        float2 p[R];
        twiddle_powers<R>(tw[n], p);
        static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; s[n + m * L] = (m > 0) ? cmul(v[m], p[m]) : v[m]; });
    }
}
template <int R>
__host__ __device__ inline void row_first_inv(float2* __restrict__ g, const float2* __restrict__ s, const float2* __restrict__ tw,
                                              int n_total, int tid, int nthr) {
    const int L = n_total / R;
    for (int n = tid; n < L; n += nthr) {
        float2 v[R], p[R];
        twiddle_powers<R>(tw[n], p);
        static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; const float2 u = s[n + m * L]; v[m] = (m > 0) ? cmulc(u, p[m]) : u; });
        DFT<R, true>::run(v);
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; g[n + q * L] = v[q]; });
    }
}
template <int R, typename TabT>
__host__ __device__ inline void row_last_masked(float2* __restrict__ s, const TabT* __restrict__ tab, int n_total, int tid, int nthr) {
    const int G = n_total / R;
    for (int j = tid; j < G; j += nthr) {
        float2* base = s + j * R;
        float2 v[R];
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = base[q]; });
        DFT<R, false>::run(v);
        if constexpr (std::is_same<TabT, float>::value)
            static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; const float c = tab[m * G + j]; v[m].x *= c; v[m].y *= c; });
        else
            static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; v[m] = cmul(v[m], tab[m * G + j]); });
        DFT<R, true>::run(v);
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; base[q] = v[q]; });
    }
}
#define D4W_ROW_RADIX_SWITCH(r, CALL)                                                                         \
    switch (r) {                                                                                              \
        case 2: { CALL(2) } break; case 3: { CALL(3) } break; case 4: { CALL(4) } break; case 5: { CALL(5) } break;         \
        case 6: { CALL(6) } break; case 8: { CALL(8) } break; case 10: { CALL(10) } break; case 12: { CALL(12) } break;     \
        case 15: { CALL(15) } break; case 16: { CALL(16) } break; case 20: { CALL(20) } break; default: { CALL(25) } break; \
    }
__host__ __device__ inline bool row_radix_inreg(int r) {
    return r == 2 || r == 3 || r == 4 || r == 5 || r == 6 || r == 8 || r == 10 || r == 12 || r == 15 || r == 16 || r == 20 || r == 25;
}
template <typename TabT>
__host__ __device__ inline void body_row_mid_fused(const RowParams& rp, float2* __restrict__ w, size_t ldw,
                                                   const TabT* __restrict__ tab, size_t tab_slot_stride, int kt1, int slot,
                                                   int tid, int nthr, float2* smem) {
    const int n = rp.t2, nst = rp.pl.nstages;
    float2* g = w + (size_t)slot * ldw + (size_t)kt1 * n;
    const TabT* m = tab + (size_t)slot * tab_slot_stride + (size_t)kt1 * n;
    const int r0 = rp.pl.radix[0], rl = rp.pl.radix[nst - 1];
#define D4W_CALL(R) row_first_fwd<R>(g, smem, rp.tw, n, tid, nthr);
    D4W_ROW_RADIX_SWITCH(r0, D4W_CALL)
#undef D4W_CALL
    D4W_SYNC();
    fft_forward_stages(smem, rp.pl, rp.tw, 1, n, tid, nthr, 1, nst - 1);
#define D4W_CALL(R) row_last_masked<R>(smem, m, n, tid, nthr);
    D4W_ROW_RADIX_SWITCH(rl, D4W_CALL)
#undef D4W_CALL
    D4W_SYNC();
    fft_inverse_stages(smem, rp.pl, rp.tw, 1, n, tid, nthr, 1, nst - 1);
#define D4W_CALL(R) row_first_inv<R>(g, smem, rp.tw, n, tid, nthr);
    D4W_ROW_RADIX_SWITCH(r0, D4W_CALL)
#undef D4W_CALL
}

// ================================================================== __global__ wrappers
#ifdef __CUDACC__
extern __shared__ __align__(1024) float2 d4w_dyn_smem[];

template <int MAXT>
static __global__ void __launch_bounds__(MAXT, 1)
k_col_fwd(ColParams cp, const float* __restrict__ x, float2* __restrict__ w, size_t ldw, const int2* __restrict__ slot_pos,
          int nact, const float* __restrict__ taper) {
    body_col_fwd(cp, x, w, ldw, slot_pos, nact, taper, blockIdx.x, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

template <int MAXT>
static __global__ void __launch_bounds__(MAXT, 1)
k_col_inv(ColParams cp, const float2* __restrict__ w, size_t ldw, const int2* __restrict__ slot_pos, int nact,
          float* __restrict__ y) {
    body_col_inv(cp, w, ldw, slot_pos, nact, y, blockIdx.x, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

static __global__ void __launch_bounds__(512, 1)
k_col_fwd_czt(CztParams cp, const float* __restrict__ x, float2* __restrict__ w, size_t ldw, const int2* __restrict__ slot_pos,
              int nact, const float* __restrict__ taper) {
    body_col_fwd_czt(cp, x, w, ldw, slot_pos, nact, taper, blockIdx.x, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

static __global__ void __launch_bounds__(512, 1)
k_col_inv_czt(CztParams cp, const float2* __restrict__ w, size_t ldw, const int2* __restrict__ slot_pos, int nact,
              float* __restrict__ y) {
    body_col_inv_czt(cp, w, ldw, slot_pos, nact, y, blockIdx.x, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

template <int MAXT>
static __global__ void __launch_bounds__(MAXT, 1)
k_col_fwd_dual(ColParams cp, const float* __restrict__ x, float2* __restrict__ w, size_t ldw, const int2* __restrict__ slot_pos,
               int nact, const float* __restrict__ taper) {
    body_col_fwd_dual(cp, x, w, ldw, slot_pos, nact, taper, blockIdx.x, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem));
}

template <int MAXT>
static __global__ void __launch_bounds__(MAXT, 1)
k_col_inv_dual(ColParams cp, const float2* __restrict__ w, size_t ldw, const int2* __restrict__ slot_pos, int nact,
               float* __restrict__ y) {
    body_col_inv_dual(cp, w, ldw, slot_pos, nact, y, blockIdx.x, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem));
}


// ================================================================== TMA-fed persistent column kernels
// TMA path for the dominant case (one dual column per tile, ns % 4 == 0): the whole
// [nx x 4 samples] tile moves with 2-D tensor copies (cp.async.bulk.tensor, boxes of 256 rows x 16 B)
// issued by one thread -- no per-row LSU instruction, completion through an mbarrier (load) or a
// bulk group (store, fully asynchronous w.r.t. the next tile).  CTAs are persistent (one per SM).
#ifdef __CUDACC__
#include <cuda.h>

constexpr int kTmaBoxRows = 256;

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, unsigned long long* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* smem_src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(map), "r"(c0), "r"(c1),
                 "r"(smem_u32(smem_src))
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// forward: x --TMA + cp.async--> smem, forward stages, untangle + pruned store.
// The tile's rows are split between the two copy engines (TMA boxes for the first tma_rows rows,
// 16-byte cp.async for the rest) so their per-row request rates add up; the kept elements of the
// finished tile are pulled into registers first, so the next tile's copy runs under the untangle.
constexpr int kMaxOutPerThread = 6;
template <int MAXT>
static __global__ void __maxnreg__(MAXT <= 256 ? 255 : MAXT <= 416 ? 152 : 128)
k_col_fwd_tma(const __grid_constant__ CUtensorMap tmx, ColParams cp, const float* __restrict__ x, float2* __restrict__ w, size_t ldw,
              const int2* __restrict__ slot_pos, int nact, const float* __restrict__ taper, int ntiles, int tma_boxes,
              unsigned long long* __restrict__ dbg) {
    cpd* smem = reinterpret_cast<cpd*>(d4w_dyn_smem);
    __shared__ __align__(8) unsigned long long bar;
    long long c_load = 0, c_fft = 0, c_out = 0, tc = 0;
    const int tid = threadIdx.x, nthr = blockDim.x, nx = cp.nx, ns = cp.ns;
    const int tma_rows = min(nx, tma_boxes * kTmaBoxRows);
    const bool regs_ok = nact <= kMaxOutPerThread * nthr;
    if (tid == 0) { mbar_init(&bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    unsigned parity = 0;
    const f2x half = vbc(0.5f);
    auto issue_load = [&](int tile) {
        const int t0 = tile * 4;
        if (tid == 0 && tma_boxes > 0) {
            mbar_expect_tx(&bar, (unsigned)(tma_boxes * kTmaBoxRows * 16));
            for (int b = 0; b < tma_boxes; ++b) tma_load_2d(smem + b * kTmaBoxRows, &tmx, t0, b * kTmaBoxRows, &bar);
        }
        for (int c = tma_rows + tid; c < nx; c += nthr) cp_async16(smem + c, x + (size_t)c * ns + t0);
    };
    int tile = blockIdx.x;
    if (tile < ntiles) issue_load(tile);
    for (; tile < ntiles; tile += gridDim.x) {
        const int t0 = tile * 4;
        if (dbg && tid == 0) tc = clock64();
        cp_async_wait_all();
        if (tma_boxes > 0) { mbar_wait(&bar, parity); parity ^= 1u; }
        __syncthreads();
        if (dbg && tid == 0) { const long long t = clock64(); c_load += t - tc; tc = t; }
        if (taper) {
            const f2x wa = f2x_set(taper[t0], taper[t0 + 1]), wb = f2x_set(taper[t0 + 2], taper[t0 + 3]);
            for (int c = tid; c < nx; c += nthr) { cpd v = smem[c]; v.x = vmul(v.x, wa); v.y = vmul(v.y, wb); smem[c] = v; }
            __syncthreads();
        }
        fft_forward_stages_dual(smem, cp.pl, cp.tw, 1, cp.fstride, tid, nthr);
        if (dbg && tid == 0) { const long long t = clock64(); c_fft += t - tc; tc = t; }
        const int next = tile + gridDim.x;
        if (regs_ok) {
            cpd z[kMaxOutPerThread], z2[kMaxOutPerThread];
#pragma unroll
            for (int j = 0; j < kMaxOutPerThread; ++j) {
                const int slot = tid + j * nthr;
                if (slot < nact) { const int2 pp = slot_pos[slot]; z[j] = smem[pp.x]; z2[j] = smem[pp.y]; }
            }
            // the in-place FFT wrote this buffer through the generic proxy; order those writes (and our reads)
            // before the async-proxy (TMA) writes of the next tile
            fence_async_smem();
            __syncthreads();                       // tile fully consumed -> its buffer is free
            if (next < ntiles) issue_load(next);   // next tile streams in while we untangle from registers
#pragma unroll
            for (int j = 0; j < kMaxOutPerThread; ++j) {
                const int slot = tid + j * nthr;
                if (slot < nact) {
                    const cpd xa = dmake(vmul(vadd(z[j].x, z2[j].x), half), vmul(vsub(z[j].y, z2[j].y), half));
                    const cpd xb = dmake(vmul(vadd(z[j].y, z2[j].y), half), vmul(vsub(z2[j].x, z[j].x), half));
                    float4* o = reinterpret_cast<float4*>(w + (size_t)slot * ldw + t0);
                    o[0] = make_float4(f2x_lo(xa.x), f2x_lo(xa.y), f2x_hi(xa.x), f2x_hi(xa.y));
                    o[1] = make_float4(f2x_lo(xb.x), f2x_lo(xb.y), f2x_hi(xb.x), f2x_hi(xb.y));
                }
            }
        } else {
            for (int slot = tid; slot < nact; slot += nthr) {
                const int2 pp = slot_pos[slot];
                const cpd z = smem[pp.x], z2 = smem[pp.y];
                const cpd xa = dmake(vmul(vadd(z.x, z2.x), half), vmul(vsub(z.y, z2.y), half));
                const cpd xb = dmake(vmul(vadd(z.y, z2.y), half), vmul(vsub(z2.x, z.x), half));
                float4* o = reinterpret_cast<float4*>(w + (size_t)slot * ldw + t0);
                o[0] = make_float4(f2x_lo(xa.x), f2x_lo(xa.y), f2x_hi(xa.x), f2x_hi(xa.y));
                o[1] = make_float4(f2x_lo(xb.x), f2x_lo(xb.y), f2x_hi(xb.x), f2x_hi(xb.y));
            }
            fence_async_smem();
            __syncthreads();
            if (next < ntiles) issue_load(next);
        }
        if (dbg && tid == 0) { const long long t = clock64(); c_out += t - tc; tc = t; }
    }
    if (dbg && tid == 0) {
        atomicAdd(dbg + 0, (unsigned long long)c_load); atomicAdd(dbg + 1, (unsigned long long)c_fft);
        atomicAdd(dbg + 2, (unsigned long long)c_out);
    }
}

// inverse: kept rows -> smem, inverse stages, smem --TMA--> y (asynchronous store)
template <int MAXT>
static __global__ void __maxnreg__(MAXT <= 256 ? 255 : MAXT <= 416 ? 152 : 128)
k_col_inv_tma(const __grid_constant__ CUtensorMap tmy, ColParams cp, const float2* __restrict__ w, size_t ldw,
              const int2* __restrict__ slot_pos, int nact, int ntiles, float* __restrict__ y, int tma_boxes,
              unsigned long long* __restrict__ dbg) {
    cpd* smem = reinterpret_cast<cpd*>(d4w_dyn_smem);
    const int tid = threadIdx.x, nthr = blockDim.x, nx = cp.nx, ns = cp.ns;
    const int nbox = tma_boxes;
    const int tma_rows = min(nx, tma_boxes * kTmaBoxRows);
    const cpd zero = dmake(vbc(0.f), vbc(0.f));
    long long c_wait = 0, c_fill = 0, c_fft = 0, c_st = 0, tc = 0;
    // the slots a thread scatters are the same for every tile: keep their positions in registers
    const bool regs_ok = nact <= kMaxOutPerThread * nthr;
    int2 ppr[kMaxOutPerThread];
#pragma unroll
    for (int j = 0; j < kMaxOutPerThread; ++j) {
        const int slot = tid + j * nthr;
        ppr[j] = (regs_ok && slot < nact) ? slot_pos[slot] : make_int2(0, 0);
    }
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int t0 = tile * 4;
        if (dbg && tid == 0) tc = clock64();
        // all kept-row loads of this tile go out first; their DRAM latency hides under the drain + clear
        float4 ru[kMaxOutPerThread], rv[kMaxOutPerThread];
        if (regs_ok) {
#pragma unroll
            for (int j = 0; j < kMaxOutPerThread; ++j) {
                const int slot = tid + j * nthr;
                if (slot < nact) {
                    const float4* src = reinterpret_cast<const float4*>(w + (size_t)slot * ldw + t0);
                    ru[j] = src[0]; rv[j] = src[1];
                }
            }
        }
        if (tid == 0) { tma_store_wait_read(); fence_async_smem(); }   // previous tile's store has finished READING smem
        __syncthreads();
        if (dbg && tid == 0) { const long long t = clock64(); c_wait += t - tc; tc = t; }
        for (int i = tid; i < cp.fstride; i += nthr) smem[i] = zero;
        __syncthreads();
        if (regs_ok) {
#pragma unroll
            for (int j = 0; j < kMaxOutPerThread; ++j) {
                const int slot = tid + j * nthr;
                if (slot < nact) {
                    const int2 pp = ppr[j];
                    const float4 u = ru[j], v = rv[j];
                    if (pp.x == pp.y) {
                        smem[pp.x] = dmake(f2x_set(u.x, u.z), f2x_set(v.x, v.z));
                    } else {
                        smem[pp.x] = dmake(f2x_set(u.x - v.y, u.z - v.w), f2x_set(u.y + v.x, u.w + v.z));
                        smem[pp.y] = dmake(f2x_set(u.x + v.y, u.z + v.w), f2x_set(v.x - u.y, v.z - u.w));
                    }
                }
            }
        } else {
            for (int slot = tid; slot < nact; slot += nthr) {
                const int2 pp = slot_pos[slot];
                const float4* src = reinterpret_cast<const float4*>(w + (size_t)slot * ldw + t0);
                const float4 u = src[0], v = src[1];
                if (pp.x == pp.y) {
                    smem[pp.x] = dmake(f2x_set(u.x, u.z), f2x_set(v.x, v.z));
                } else {
                    smem[pp.x] = dmake(f2x_set(u.x - v.y, u.z - v.w), f2x_set(u.y + v.x, u.w + v.z));
                    smem[pp.y] = dmake(f2x_set(u.x + v.y, u.z + v.w), f2x_set(v.x - u.y, v.z - u.w));
                }
            }
        }
        __syncthreads();
        if (dbg && tid == 0) { const long long t = clock64(); c_fill += t - tc; tc = t; }
        fft_inverse_stages_dual(smem, cp.pl, cp.tw, 1, cp.fstride, tid, nthr);
        fence_async_smem();                            // generic-proxy writes visible to the async proxy
        __syncthreads();
        if (dbg && tid == 0) { const long long t = clock64(); c_fft += t - tc; tc = t; }
        if (tid == 0 && nbox > 0) {
            for (int b = 0; b < nbox; ++b) tma_store_2d(&tmy, t0, b * kTmaBoxRows, smem + b * kTmaBoxRows);
            tma_store_commit();
        }
        // the remaining rows leave through the LSU at the same time (16-byte row stores)
        for (int c = tma_rows + tid; c < nx; c += nthr)
            *reinterpret_cast<float4*>(y + (size_t)c * ns + t0) = *reinterpret_cast<const float4*>(smem + c);
        if (dbg && tid == 0) { const long long t = clock64(); c_st += t - tc; tc = t; }
    }
    if (tid == 0) tma_store_wait_all();
    if (dbg && tid == 0) {
        atomicAdd(dbg + 4, (unsigned long long)c_wait); atomicAdd(dbg + 5, (unsigned long long)c_fill);
        atomicAdd(dbg + 6, (unsigned long long)c_fft); atomicAdd(dbg + 7, (unsigned long long)c_st);
    }
}
#endif  // __CUDACC__

template <int T1, bool INV>
static __global__ void __launch_bounds__(128)
k_row_split(float2* __restrict__ w, size_t ldw, int t2len, const float2* __restrict__ twT) {
    const int t2 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t2 < t2len) body_row_split<T1, INV>(w, ldw, t2len, twT, blockIdx.y, t2);
}

static __global__ void __launch_bounds__(256, 2)
k_row_mid(RowParams rp, float2* __restrict__ w, size_t ldw, const float* __restrict__ tab, size_t tab_slot_stride) {
    body_row_mid(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

static __global__ void __launch_bounds__(256, 2)
k_row_mid_fused(RowParams rp, float2* __restrict__ w, size_t ldw, const float* __restrict__ tab, size_t tab_slot_stride) {
    body_row_mid_fused(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

static __global__ void __launch_bounds__(128, 2)     // radix-25 dual butterflies need ~190 registers: 2 x 128-thread CTAs per SM
k_row_mid_dual(RowParams rp, float2* __restrict__ w, size_t ldw, const float* __restrict__ tab, size_t tab_slot_stride, int nslots) {
    body_row_mid_dual(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, nslots, threadIdx.x, blockDim.x,
                      reinterpret_cast<cpd*>(d4w_dyn_smem));
}

template <int X1>
static __global__ void __launch_bounds__(128)
k_colA_fwd(Col2Params cp, const float* __restrict__ x, cpd* __restrict__ v2, const float* __restrict__ taper) {
    const int t4 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t4 < cp.tpn / 2) body_colA_fwd<X1>(cp, x, v2, taper, blockIdx.y, t4, cp.tpb);
}
template <int X1>
static __global__ void __launch_bounds__(128)
k_colA_inv(Col2Params cp, const cpd* __restrict__ v2, float* __restrict__ y) {
    const int t4 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t4 < cp.tpn / 2) body_colA_inv<X1>(cp, v2, y, blockIdx.y, t4, cp.tpb);
}
static __global__ void __launch_bounds__(160, 3)
k_colB_fwd(Col2Params cp, const cpd* __restrict__ v2, float2* __restrict__ w, size_t ldw, const int* __restrict__ plane_ptr,
           const Col2Entry* __restrict__ ents) {
    body_colB_fwd(cp, v2, w, ldw, plane_ptr, ents, blockIdx.y, blockIdx.x, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem));
}
static __global__ void __launch_bounds__(160, 3)
k_colB_inv(Col2Params cp, cpd* __restrict__ v2, const float2* __restrict__ w, size_t ldw, const int* __restrict__ plane_ptr,
           const Col2Entry* __restrict__ ents) {
    body_colB_inv(cp, v2, w, ldw, plane_ptr, ents, blockIdx.y, blockIdx.x, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem));
}

template <int RA, int RB>
static __global__ void __launch_bounds__(160, 3)
k_colB_fwd_fused(Col2Params cp, const cpd* __restrict__ v2, float2* __restrict__ w, size_t ldw, const int2* __restrict__ need) {
    body_colB_fwd_fused<RA, RB>(cp, v2, w, ldw, need, blockIdx.y, blockIdx.x, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem), cp.tpb, cp.tpn);
}
template <int RA, int RB>
static __global__ void __launch_bounds__(160, 3)
k_colB_inv_fused(Col2Params cp, cpd* __restrict__ v2, const float2* __restrict__ w, size_t ldw, const int2* __restrict__ need) {
    body_colB_inv_fused<RA, RB>(cp, v2, w, ldw, need, blockIdx.y, blockIdx.x, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem), cp.tpb, cp.tpn);
}

// ---- single-launch pipelined level A + level B ------------------------------------------------------------------
// The record is cut into time chunks of cp.vhp sample pairs.  CTAs take tickets in start order; ticket -> (slot, role):
// slot s holds the producer CTAs of chunk s followed by the consumer CTAs of chunk s - lag (forward: level A produces V,
// level B consumes it; inverse: the other way round).  V lives in a ring of nbuf > lag chunk buffers that stays in L2:
// a consumer waits until all producers of its chunk have signalled, a producer re-using a ring slot waits for the
// consumers of the chunk that held it.  Every wait is on CTAs with smaller tickets, which have already started, so
// the scheme cannot deadlock whatever the dispatch order.
struct PipeParams {
    int nchunks, lag, nbuf;
    int nA, nB;                  // level-A / level-B CTAs per chunk
    int cq, rpc;                 // level A: quads per row handled by one CTA, c2 rows per CTA (cq * rpc <= blockDim)
    int tiles;                   // level B: np-pair tiles per chunk
    int hints;                   // L2 eviction-priority hints on/off
    unsigned* cnt;               // [0] ticket, [1 .. nchunks] A done, [1 + nchunks .. 2 nchunks] B done
    size_t vbuf_elems;           // cpd elements per ring slot
};

#ifdef __CUDACC__
__device__ __forceinline__ void pipe_wait(const unsigned* p, unsigned target) {
    if (threadIdx.x == 0) {
        unsigned v;
        for (;;) {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
            if (v >= target) break;
            __nanosleep(64);
        }
    }
    __syncthreads();
}
__device__ __forceinline__ void pipe_signal(unsigned* p) {
    __syncthreads();
    if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" :: "l"(p) : "memory");
}

template <int X1, int RA, int RB, bool INV, int OCC = 3>
static __global__ void __launch_bounds__(160, OCC)
k_col2_pipe(Col2Params cp, PipeParams pp, const float* __restrict__ x, float* __restrict__ y, cpd* v2, float2* w, size_t ldw,
            const int2* __restrict__ need, const float* __restrict__ taper) {
    __shared__ unsigned s_ticket;
    if (threadIdx.x == 0) s_ticket = atomicAdd(pp.cnt, 1u);
    __syncthreads();
    const int per = pp.nA + pp.nB;
    const int slot = (int)(s_ticket / (unsigned)per), r = (int)(s_ticket % (unsigned)per);
    const int nfirst = INV ? pp.nB : pp.nA;                 // producers come first in a slot
    const bool first = r < nfirst;
    const int c = first ? slot : slot - pp.lag;
    if (c < 0 || c >= pp.nchunks) return;
    const int idx = first ? r : r - nfirst;
    const bool roleA = first != INV;
    unsigned* cntA = pp.cnt + 1;
    unsigned* cntB = pp.cnt + 1 + pp.nchunks;
    const int tpb = c * cp.vhp, tpn = min(cp.vhp, cp.ns / 2 - tpb);
    cpd* vb = v2 + (size_t)(c % pp.nbuf) * pp.vbuf_elems;
    const L2Pol pol = make_l2pol(pp.hints != 0);
    if (first) { if (c >= pp.nbuf) pipe_wait((INV ? cntA : cntB) + (c - pp.nbuf), (unsigned)(INV ? pp.nA : pp.nB)); }
    else pipe_wait((INV ? cntB : cntA) + c, (unsigned)(INV ? pp.nB : pp.nA));
    if (roleA) {
        const int row = (int)threadIdx.x / pp.cq, q = (int)threadIdx.x - row * pp.cq;
        const int c2 = idx * pp.rpc + row;
        if (row < pp.rpc && c2 < cp.x2 && q < tpn / 2) {
            if constexpr (!INV) body_colA_fwd<X1, true>(cp, x, vb, taper, c2, q, tpb, pol);
            else body_colA_inv<X1, true>(cp, vb, y, c2, q, tpb, pol);
        }
        pipe_signal(cntA + c);
    } else {
        const int plane = idx / pp.tiles, tile = idx - plane * pp.tiles;
        if (tile * cp.np < tpn) {
            if constexpr (!INV) body_colB_fwd_fused<RA, RB, true>(cp, vb, w, ldw, need, plane, tile, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem), tpb, tpn, pol);
            else body_colB_inv_fused<RA, RB, true>(cp, vb, w, ldw, need, plane, tile, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem), tpb, tpn, pol);
        }
        pipe_signal(cntB + c);
    }
}
#endif

#ifdef __CUDACC__
// pipelined level A (radix X1 in registers) + three-stage level B: same ticket / ring protocol as k_col2_pipe
template <int X1, int R0, int R1, int R2, bool INV, int OCC>
static __global__ void __launch_bounds__(224, OCC)
k_col3_pipe(Col2Params cp, PipeParams pp, const float* __restrict__ x, float* __restrict__ y, cpd* v2, float2* w, size_t ldw,
            const int2* __restrict__ need, const float* __restrict__ taper) {
    __shared__ unsigned s_ticket;
    if (threadIdx.x == 0) s_ticket = atomicAdd(pp.cnt, 1u);
    __syncthreads();
    const int per = pp.nA + pp.nB;
    const int slot = (int)(s_ticket / (unsigned)per), r = (int)(s_ticket % (unsigned)per);
    const int nfirst = INV ? pp.nB : pp.nA;
    const bool first = r < nfirst;
    const int c = first ? slot : slot - pp.lag;
    if (c < 0 || c >= pp.nchunks) return;
    const int idx = first ? r : r - nfirst;
    const bool roleA = first != INV;
    unsigned* cntA = pp.cnt + 1;
    unsigned* cntB = pp.cnt + 1 + pp.nchunks;
    const int tpb = c * cp.vhp, tpn = min(cp.vhp, cp.ns / 2 - tpb);
    cpd* vb = v2 + (size_t)(c % pp.nbuf) * pp.vbuf_elems;
    const L2Pol pol = make_l2pol(pp.hints != 0);
    if (first) { if (c >= pp.nbuf) pipe_wait((INV ? cntA : cntB) + (c - pp.nbuf), (unsigned)(INV ? pp.nA : pp.nB)); }
    else pipe_wait((INV ? cntB : cntA) + c, (unsigned)(INV ? pp.nB : pp.nA));
    if (roleA) {
        const int row = (int)threadIdx.x / pp.cq, q = (int)threadIdx.x - row * pp.cq;
        const int c2 = idx * pp.rpc + row;
        if (row < pp.rpc && c2 < cp.x2 && q < tpn / 2) {
            if constexpr (!INV) body_colA_fwd<X1, true>(cp, x, vb, taper, c2, q, tpb, pol);
            else body_colA_inv<X1, true>(cp, vb, y, c2, q, tpb, pol);
        }
        pipe_signal(cntA + c);
    } else {
        const int plane = idx / pp.tiles, tile = idx - plane * pp.tiles;
        if (tile * cp.np < tpn) {
            if constexpr (!INV) body_colB3_fwd<R0, R1, R2, true>(cp, vb, w, ldw, need, plane, tile, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem), tpb, tpn, pol);
            else body_colB3_inv<R0, R1, R2, true>(cp, vb, w, ldw, need, plane, tile, threadIdx.x, blockDim.x, reinterpret_cast<cpd*>(d4w_dyn_smem), tpb, tpn, pol);
        }
        pipe_signal(cntB + c);
    }
}
#endif

static __global__ void k_mask_rowmax(MaskParams mp, unsigned int* rowmax, int fchunk) {
    const int k = blockIdx.y;
    const int f0 = blockIdx.x * fchunk;
    const int f1 = min(mp.ns, f0 + fchunk);
    body_mask_rowmax(mp, rowmax, k, f0, f1, threadIdx.x, blockDim.x);
}

static __global__ void k_mask_build(MaskParams mp, float* tab, const int* act_k, const int* pos2k_row, int t1, int t2,
                             double scale, size_t total) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < total) body_mask_build(mp, tab, act_k, pos2k_row, t1, t2, scale, idx);
}

static __global__ void k_mask_materialize(MaskParams mp, double* out, size_t total) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < total) out[idx] = mask_shifted(mp, (int)(idx / mp.ns), (int)(idx % mp.ns));
}
#endif  // __CUDACC__

}  // namespace d4w
