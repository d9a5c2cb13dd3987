// fft_dual.cuh -- two-lane ("dual column") variant of the FFT engine.
//
// The column passes of the f-k filter transform a tile of 4 consecutive time samples per
// channel = two complex columns that undergo IDENTICAL butterflies with IDENTICAL twiddles.
// Element c of the tile is stored as 16 bytes {reA, reB, imA, imB}; one thread runs both
// columns through one instruction stream: the twiddles (per-lane equal) are loaded and formed
// once for both lanes, shared memory traffic is LDS.128 / STS.128 and the global side is one
// 16-byte cp.async per channel row.  Hopper has no packed fp32x2 arithmetic, so every lane op
// is one scalar FADD / FMUL / FFMA; the _rn intrinsics stop nvcc from contracting a vmul that
// feeds a vadd into an FFMA, so each lane rounds exactly as the operation written.
// Same __host__ __device__ discipline as fft_smem.cuh.
#pragma once
#include "fft_smem.cuh"

namespace d4w {

// ---------------------------------------------------------------- pair of floats
struct __align__(8) f2x { float a, b; };
D4W_HD f2x f2x_set(float a, float b) { f2x r; r.a = a; r.b = b; return r; }
D4W_HD f2x vbc(float s) { return f2x_set(s, s); }
D4W_HD float f2x_lo(f2x v) { return v.a; }
D4W_HD float f2x_hi(f2x v) { return v.b; }
#ifdef __CUDA_ARCH__
__device__ __forceinline__ f2x vadd(f2x a, f2x b) { return f2x_set(__fadd_rn(a.a, b.a), __fadd_rn(a.b, b.b)); }
__device__ __forceinline__ f2x vsub(f2x a, f2x b) { return f2x_set(__fsub_rn(a.a, b.a), __fsub_rn(a.b, b.b)); }
__device__ __forceinline__ f2x vmul(f2x a, f2x b) { return f2x_set(__fmul_rn(a.a, b.a), __fmul_rn(a.b, b.b)); }
__device__ __forceinline__ f2x vfma(f2x a, f2x b, f2x c) { return f2x_set(__fmaf_rn(a.a, b.a, c.a), __fmaf_rn(a.b, b.b, c.b)); }
#else
inline f2x vadd(f2x a, f2x b) { return f2x_set(a.a + b.a, a.b + b.b); }
inline f2x vsub(f2x a, f2x b) { return f2x_set(a.a - b.a, a.b - b.b); }
inline f2x vmul(f2x a, f2x b) { return f2x_set(a.a * b.a, a.b * b.b); }
inline f2x vfma(f2x a, f2x b, f2x c) { return f2x_set(fmaf(a.a, b.a, c.a), fmaf(a.b, b.b, c.b)); }
#endif
D4W_HD f2x vneg(f2x a) { return vmul(a, vbc(-1.0f)); }

// two complex numbers (lanes A, B): x = real parts, y = imaginary parts; 16 bytes
struct __align__(16) cpd { f2x x, y; };
D4W_HD cpd dmake(f2x x, f2x y) { cpd r; r.x = x; r.y = y; return r; }
D4W_HD cpd dadd(cpd a, cpd b) { return dmake(vadd(a.x, b.x), vadd(a.y, b.y)); }
D4W_HD cpd dsub(cpd a, cpd b) { return dmake(vsub(a.x, b.x), vsub(a.y, b.y)); }
// a * w and a * conj(w) for a scalar complex w shared by both lanes
D4W_HD cpd dmul_s(cpd a, float2 w) {
    return dmake(vfma(a.x, vbc(w.x), vmul(a.y, vbc(-w.y))), vfma(a.x, vbc(w.y), vmul(a.y, vbc(w.x))));
}
D4W_HD cpd dmulc_s(cpd a, float2 w) {
    return dmake(vfma(a.x, vbc(w.x), vmul(a.y, vbc(w.y))), vfma(a.y, vbc(w.x), vmul(a.x, vbc(-w.y))));
}

template <int R, int E, bool INV> D4W_HD cpd dmul_tw(cpd a) {
    constexpr int e = ((E % R) + R) % R;
    if constexpr (e == 0) {
        return a;
    } else if constexpr (2 * e == R) {
        return dmake(vneg(a.x), vneg(a.y));
    } else if constexpr (4 * e == R) {            // -i (fwd), +i (inv)
        return INV ? dmake(vneg(a.y), a.x) : dmake(a.y, vneg(a.x));
    } else if constexpr (4 * e == 3 * R) {        // +i (fwd), -i (inv)
        return INV ? dmake(a.y, vneg(a.x)) : dmake(vneg(a.y), a.x);
    } else {
        constexpr float wr = Tw<R, e>::re;
        constexpr float wi = INV ? -Tw<R, e>::im : Tw<R, e>::im;
        return dmake(vfma(a.x, vbc(wr), vmul(a.y, vbc(-wi))), vfma(a.x, vbc(wi), vmul(a.y, vbc(wr))));
    }
}

// ---------------------------------------------------------------- DFTD<R, INV>: dual-lane butterflies
template <int R, bool INV> struct DFTD;
template <bool INV> struct DFTD<1, INV> { static D4W_HD void run(cpd (&)[1]) {} };

template <bool INV> struct DFTD<2, INV> {
    static D4W_HD void run(cpd (&v)[2]) { cpd a = v[0], b = v[1]; v[0] = dadd(a, b); v[1] = dsub(a, b); }
};

template <bool INV> struct DFTD<3, INV> {
    static D4W_HD void run(cpd (&v)[3]) {
        constexpr float s = INV ? 0.86602540378443864676f : -0.86602540378443864676f;
        const cpd t = dadd(v[1], v[2]), d = dsub(v[1], v[2]);
        const cpd m = dmake(vfma(t.x, vbc(-0.5f), v[0].x), vfma(t.y, vbc(-0.5f), v[0].y));
        v[0] = dadd(v[0], t);
        v[1] = dmake(vfma(d.y, vbc(-s), m.x), vfma(d.x, vbc(s), m.y));
        v[2] = dmake(vfma(d.y, vbc(s), m.x), vfma(d.x, vbc(-s), m.y));
    }
};

template <bool INV> struct DFTD<4, INV> {
    static D4W_HD void run(cpd (&v)[4]) {
        const cpd a = dadd(v[0], v[2]), b = dsub(v[0], v[2]);
        const cpd c = dadd(v[1], v[3]), d = dsub(v[1], v[3]);
        v[0] = dadd(a, c); v[2] = dsub(a, c);
        if constexpr (!INV) {     // b -/+ i d
            v[1] = dmake(vadd(b.x, d.y), vsub(b.y, d.x));
            v[3] = dmake(vsub(b.x, d.y), vadd(b.y, d.x));
        } else {
            v[1] = dmake(vsub(b.x, d.y), vadd(b.y, d.x));
            v[3] = dmake(vadd(b.x, d.y), vsub(b.y, d.x));
        }
    }
};

template <bool INV> struct DFTD<5, INV> {
    static D4W_HD void run(cpd (&v)[5]) {
        constexpr float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
        constexpr float s1 = INV ? 0.95105651629515357212f : -0.95105651629515357212f;
        constexpr float s2 = INV ? 0.58778525229247312917f : -0.58778525229247312917f;
        const cpd t1 = dadd(v[1], v[4]), d1 = dsub(v[1], v[4]);
        const cpd t2 = dadd(v[2], v[3]), d2 = dsub(v[2], v[3]);
        const cpd a0 = v[0];
        v[0] = dadd(a0, dadd(t1, t2));
        const cpd m1 = dmake(vfma(t1.x, vbc(c1), vfma(t2.x, vbc(c2), a0.x)), vfma(t1.y, vbc(c1), vfma(t2.y, vbc(c2), a0.y)));
        const cpd m2 = dmake(vfma(t1.x, vbc(c2), vfma(t2.x, vbc(c1), a0.x)), vfma(t1.y, vbc(c2), vfma(t2.y, vbc(c1), a0.y)));
        const cpd u1 = dmake(vfma(d1.x, vbc(s1), vmul(d2.x, vbc(s2))), vfma(d1.y, vbc(s1), vmul(d2.y, vbc(s2))));
        const cpd u2 = dmake(vfma(d1.x, vbc(s2), vmul(d2.x, vbc(-s1))), vfma(d1.y, vbc(s2), vmul(d2.y, vbc(-s1))));
        // v1 = m1 + i u1, v4 = m1 - i u1, v2 = m2 + i u2, v3 = m2 - i u2
        v[1] = dmake(vsub(m1.x, u1.y), vadd(m1.y, u1.x));
        v[4] = dmake(vadd(m1.x, u1.y), vsub(m1.y, u1.x));
        v[2] = dmake(vsub(m2.x, u2.y), vadd(m2.y, u2.x));
        v[3] = dmake(vadd(m2.x, u2.y), vsub(m2.y, u2.x));
    }
};

// radix 7 (prime): pair terms t_j = v[j] + v[7-j], d_j = v[j] - v[7-j]; X_m = A_m -/+ i B_m with
// A_m = v0 + sum_j cos(2 pi j m / 7) t_j, B_m = sum_j sin(2 pi j m / 7) d_j (forward: X_m = A_m - i B_m, X_{7-m} = A_m + i B_m).
// Used by the prime-factor (Good-Thomas) 2520-point blocks of the matched filter.
template <bool INV> struct DFTD<7, INV> {
    static D4W_HD void run(cpd (&v)[7]) {
        constexpr float c1 = 0.62348980185873353053f, c2 = -0.22252093395631440429f, c3 = -0.90096886790241912624f;
        constexpr float s1 = 0.78183148246802980871f, s2 = 0.97492791218182360702f, s3 = 0.43388373911755812048f;
        const cpd t1 = dadd(v[1], v[6]), d1 = dsub(v[1], v[6]);
        const cpd t2 = dadd(v[2], v[5]), d2 = dsub(v[2], v[5]);
        const cpd t3 = dadd(v[3], v[4]), d3 = dsub(v[3], v[4]);
        const cpd a0 = v[0];
        v[0] = dadd(a0, dadd(t1, dadd(t2, t3)));
        // cos(2 pi j m / 7) for (m, j): m = 1: c1 c2 c3;  m = 2: c2 c3 c1;  m = 3: c3 c1 c2
        // sin(2 pi j m / 7):           m = 1: s1 s2 s3;  m = 2: s2 -s3 -s1; m = 3: s3 -s1 s2
        const cpd A1 = dmake(vfma(t1.x, vbc(c1), vfma(t2.x, vbc(c2), vfma(t3.x, vbc(c3), a0.x))), vfma(t1.y, vbc(c1), vfma(t2.y, vbc(c2), vfma(t3.y, vbc(c3), a0.y))));
        const cpd A2 = dmake(vfma(t1.x, vbc(c2), vfma(t2.x, vbc(c3), vfma(t3.x, vbc(c1), a0.x))), vfma(t1.y, vbc(c2), vfma(t2.y, vbc(c3), vfma(t3.y, vbc(c1), a0.y))));
        const cpd A3 = dmake(vfma(t1.x, vbc(c3), vfma(t2.x, vbc(c1), vfma(t3.x, vbc(c2), a0.x))), vfma(t1.y, vbc(c3), vfma(t2.y, vbc(c1), vfma(t3.y, vbc(c2), a0.y))));
        const cpd B1 = dmake(vfma(d1.x, vbc(s1), vfma(d2.x, vbc(s2), vmul(d3.x, vbc(s3)))), vfma(d1.y, vbc(s1), vfma(d2.y, vbc(s2), vmul(d3.y, vbc(s3)))));
        const cpd B2 = dmake(vfma(d1.x, vbc(s2), vfma(d2.x, vbc(-s3), vmul(d3.x, vbc(-s1)))), vfma(d1.y, vbc(s2), vfma(d2.y, vbc(-s3), vmul(d3.y, vbc(-s1)))));
        const cpd B3 = dmake(vfma(d1.x, vbc(s3), vfma(d2.x, vbc(-s1), vmul(d3.x, vbc(s2)))), vfma(d1.y, vbc(s3), vfma(d2.y, vbc(-s1), vmul(d3.y, vbc(s2)))));
        // forward: A - i B = (A.x + B.y, A.y - B.x);  A + i B = (A.x - B.y, A.y + B.x); inverse swaps the two
        const cpd p1 = dmake(vadd(A1.x, B1.y), vsub(A1.y, B1.x)), q1 = dmake(vsub(A1.x, B1.y), vadd(A1.y, B1.x));
        const cpd p2 = dmake(vadd(A2.x, B2.y), vsub(A2.y, B2.x)), q2 = dmake(vsub(A2.x, B2.y), vadd(A2.y, B2.x));
        const cpd p3 = dmake(vadd(A3.x, B3.y), vsub(A3.y, B3.x)), q3 = dmake(vsub(A3.x, B3.y), vadd(A3.y, B3.x));
        if constexpr (!INV) { v[1] = p1; v[6] = q1; v[2] = p2; v[5] = q2; v[3] = p3; v[4] = q3; }
        else { v[1] = q1; v[6] = p1; v[2] = q2; v[5] = p2; v[3] = q3; v[4] = p3; }
    }
};

// Composite radix, IN PLACE with permuted output: R = R1*R2 (both factors are base radices for every
// radix we use), input v[n] natural; on return X[m] sits at v[outpos<R>(m)].  No second register
// array: the R2 length-R1 column DFTs, the internal twiddles and the R1 length-R2 row DFTs all
// overwrite v, and the transposition is absorbed into the caller's store indices.
template <int R> constexpr int outpos(int m) {
    constexpr int R1 = pick_r1<R>();
    constexpr int R2 = R / R1;
    return (R1 == R) ? m : R2 * (m % R1) + (m / R1);
}

template <int R, bool INV> struct DFTD {
    static constexpr int R1 = pick_r1<R>();
    static constexpr int R2 = R / R1;
    static_assert(R1 != R, "prime radix > 5 is handled by the generic stage");
    static_assert(pick_r1<R2>() == R2 || R2 == 4, "two-level composites only");
    static D4W_HD void run(cpd (&v)[R]) {
        static_for<R2>([&](auto n2c) {
            constexpr int n2 = decltype(n2c)::value;
            cpd a[R1];
            static_for<R1>([&](auto n1c) { constexpr int n1 = decltype(n1c)::value; a[n1] = v[R2 * n1 + n2]; });
            DFTD<R1, INV>::run(a);
            static_for<R1>([&](auto k1c) { constexpr int k1 = decltype(k1c)::value; v[R2 * k1 + n2] = dmul_tw<R, n2 * k1, INV>(a[k1]); });
        });
        static_for<R1>([&](auto k1c) {
            constexpr int k1 = decltype(k1c)::value;
            cpd b[R2];
            static_for<R2>([&](auto n2c) { constexpr int n2 = decltype(n2c)::value; b[n2] = v[R2 * k1 + n2]; });
            DFTD<R2, INV>::run(b);
            static_for<R2>([&](auto k2c) { constexpr int k2 = decltype(k2c)::value; v[R2 * k1 + k2] = b[k2]; });
        });
    }
};

// v[pos(m)] *= w^m (or conj) for m = 1..R-1 with w^m = (w^B)^a * w^j, m = B*a + j: only B + 2 complex
// registers of twiddle state, product depth <= 2 after the short chains (error ~ 5e-7).
template <int R, bool CONJ, bool PERM> D4W_HD void apply_stage_twiddles(cpd (&v)[R], float2 w) {
    constexpr int B = 5;
    float2 bj[B];
    bj[0] = make_float2(1.f, 0.f);
    bj[1] = w;
    static_for<B>([&](auto jc) { constexpr int j = decltype(jc)::value; if constexpr (j >= 2) bj[j] = cmul(bj[j / 2], bj[j - j / 2]); });
    const float2 wB = cmul(bj[B / 2], bj[B - B / 2]);
    float2 g = make_float2(1.f, 0.f);
    static_for<R>([&](auto mc) {
        constexpr int m = decltype(mc)::value;
        if constexpr (m > 0) {
            constexpr int a = m / B, j = m % B;
            if constexpr (j == 0) g = (a == 1) ? wB : cmul(g, wB);
            const float2 t = (a == 0) ? bj[j] : (j == 0 ? g : cmul(g, bj[j]));
            constexpr int pos = PERM ? outpos<R>(m) : m;
            v[pos] = CONJ ? dmulc_s(v[pos], t) : dmul_s(v[pos], t);
        }
    });
}

// ---------------------------------------------------------------- in-place smem stages on cpd elements
template <int R, bool INV>
__host__ __device__ void stage_dual(cpd* __restrict__ s, const float2* __restrict__ tw, int n_total, int ns, int nfft,
                                    int fstride, int tid, int nthr) {
    const int L = ns / R;
    const int per = n_total / R;
    const int twstep = n_total / ns;
    const int total = per * nfft;
    for (int id = tid; id < total; id += nthr) {
        const int f = id / per;
        const int j = id - f * per;
        const int b = j / L;
        const int n = j - b * L;
        cpd* base = s + (size_t)f * fstride + b * ns + n;
        cpd v[R];
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = base[q * L]; });
        if constexpr (!INV) {
            DFTD<R, false>::run(v);                                   // X[m] at v[outpos(m)]
            if (L > 1) apply_stage_twiddles<R, false, true>(v, tw[twstep * n]);
        } else {
            if (L > 1) apply_stage_twiddles<R, true, false>(v, tw[twstep * n]);
            DFTD<R, true>::run(v);
        }
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; base[q * L] = v[outpos<R>(q)]; });
    }
}

// generic prime stage (7..61) on cpd elements; same chunked compute / barrier / write scheme
template <bool INV>
__host__ __device__ void stage_generic_dual(cpd* __restrict__ s, const float2* __restrict__ tw, int n_total, int ns, int p,
                                            int nfft, int fstride, int tid, int nthr) {
    const int L = ns / p;
    const int per = n_total / p;
    const int twstep = n_total / ns;
    const int twp = n_total / p;
    const int total = per * nfft;
#ifdef __CUDA_ARCH__
    const int bpc = nthr / p;
    for (int c0 = 0; c0 < total; c0 += bpc) {
        const int id = c0 + tid / p;
        const int m = tid % p;
        const bool act = (tid < bpc * p) && (id < total);
        cpd acc = dmake(vbc(0.f), vbc(0.f));
        cpd* base = s;
        if (act) {
            const int f = id / per, j = id - f * per, b = j / L, n = j - b * L;
            base = s + (size_t)f * fstride + b * ns + n;
            if (!INV) {
                for (int q = 0; q < p; ++q) acc = dadd(acc, dmul_s(base[q * L], tw[twp * ((q * m) % p)]));
                if (L > 1) acc = dmul_s(acc, tw[(int)(((long long)twstep * n * m) % n_total)]);
            } else {
                for (int q = 0; q < p; ++q) {
                    cpd u = base[q * L];
                    if (L > 1) u = dmulc_s(u, tw[(int)(((long long)twstep * n * q) % n_total)]);
                    acc = dadd(acc, dmulc_s(u, tw[twp * ((q * m) % p)]));
                }
            }
        }
        __syncthreads();
        if (act) base[m * L] = acc;
        __syncthreads();
    }
#else
    if (tid != 0) return;
    for (int id = 0; id < total; ++id) {
        const int f = id / per, j = id - f * per, b = j / L, n = j - b * L;
        cpd* base = s + (size_t)f * fstride + b * ns + n;
        cpd in[64], out[64];
        for (int q = 0; q < p; ++q) in[q] = base[q * L];
        for (int m = 0; m < p; ++m) {
            cpd acc = dmake(vbc(0.f), vbc(0.f));
            if (!INV) {
                for (int q = 0; q < p; ++q) acc = dadd(acc, dmul_s(in[q], tw[twp * ((q * m) % p)]));
                if (L > 1) acc = dmul_s(acc, tw[(int)(((long long)twstep * n * m) % n_total)]);
            } else {
                for (int q = 0; q < p; ++q) {
                    cpd u = in[q];
                    if (L > 1) u = dmulc_s(u, tw[(int)(((long long)twstep * n * q) % n_total)]);
                    acc = dadd(acc, dmulc_s(u, tw[twp * ((q * m) % p)]));
                }
            }
            out[m] = acc;
        }
        for (int m = 0; m < p; ++m) base[m * L] = out[m];
    }
#endif
}

template <bool INV>
__host__ __device__ inline void stage_dispatch_dual(cpd* s, const float2* tw, int n_total, int ns, int r, int nfft,
                                                    int fstride, int tid, int nthr) {
    switch (r) {
#define D4W_CASE(RR) case RR: stage_dual<RR, INV>(s, tw, n_total, ns, nfft, fstride, tid, nthr); break;
        D4W_CASE(2) D4W_CASE(3) D4W_CASE(4) D4W_CASE(5) D4W_CASE(6) D4W_CASE(8) D4W_CASE(10) D4W_CASE(12) D4W_CASE(15) D4W_CASE(16)
        D4W_CASE(20) D4W_CASE(25)
#undef D4W_CASE
        default: stage_generic_dual<INV>(s, tw, n_total, ns, r, nfft, fstride, tid, nthr); break;
    }
}

constexpr int kDualMaxRadix = 25;     // radix > 16 needs ~150-170 registers -> 256-thread kernels

__host__ __device__ inline void fft_forward_stages_dual(cpd* s, const FftPlan& pl, const float2* tw, int nfft, int fstride,
                                                        int tid, int nthr) {
    for (int st = 0; st < pl.nstages; ++st) {
        stage_dispatch_dual<false>(s, tw, pl.n, pl.sub[st], pl.radix[st], nfft, fstride, tid, nthr);
        D4W_SYNC();
    }
}
__host__ __device__ inline void fft_inverse_stages_dual(cpd* s, const FftPlan& pl, const float2* tw, int nfft, int fstride,
                                                        int tid, int nthr) {
    for (int st = pl.nstages - 1; st >= 0; --st) {
        stage_dispatch_dual<true>(s, tw, pl.n, pl.sub[st], pl.radix[st], nfft, fstride, tid, nthr);
        D4W_SYNC();
    }
}

}  // namespace d4w
