// fft_radix.cuh -- in-register radix-R DFT butterflies for the sm_90a FFT engine.
//
// Every butterfly is a fully unrolled template: operands live in registers, twiddles
// W_R^j are compile-time constants (constexpr-evaluated in double, rounded once to fp32),
// composite radices (6, 8, 10, 12, 15, 16, 20, 25) are built by Cooley-Tukey inside the
// register file so a shared-memory pass is only needed once per ~radix-16/25 stage.
// All functions are __host__ __device__ so tests/host_emul can run the very same
// arithmetic on the CPU (there is no GPU in the build container).
#pragma once
#include <cuda_runtime.h>
#include <utility>
#include <type_traits>

#define D4W_HD __host__ __device__ __forceinline__

namespace d4w {

// ---------------------------------------------------------------- complex helpers
D4W_HD float2 cmul(float2 a, float2 b) {
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
D4W_HD float2 cmulc(float2 a, float2 b) {   // a * conj(b)
    return make_float2(fmaf(a.x, b.x, a.y * b.y), fmaf(a.y, b.x, -a.x * b.y));
}
D4W_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
D4W_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
D4W_HD float2 cconj(float2 a) { return make_float2(a.x, -a.y); }
D4W_HD float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }

// ---------------------------------------------------------------- constexpr sin/cos
namespace cx {
constexpr double PI = 3.141592653589793238462643383279502884;
constexpr double sin_taylor(double x) {   // |x| <= pi/2
    double x2 = x * x, term = x, sum = x;
    for (int k = 1; k < 16; ++k) { term *= -x2 / ((2 * k) * (2 * k + 1)); sum += term; }
    return sum;
}
constexpr double cos_taylor(double x) {
    double x2 = x * x, term = 1.0, sum = 1.0;
    for (int k = 1; k < 16; ++k) { term *= -x2 / ((2 * k - 1) * (2 * k)); sum += term; }
    return sum;
}
// cos / sin of 2*pi*j/r with exact integer quadrant reduction
constexpr double cos2pi(int j, int r) {
    j %= r; if (j < 0) j += r;
    // angle = 2*pi*j/r ; reduce by quadrants using 4j vs r
    int q = (4 * j) / r;            // quadrant 0..3
    int rem = 4 * j - q * r;        // 0 <= rem < r ; angle = (pi/2)*(q + rem/r)
    double a = (PI / 2) * ((double)rem / (double)r);
    switch (q) { case 0: return cos_taylor(a); case 1: return -sin_taylor(a);
                 case 2: return -cos_taylor(a); default: return sin_taylor(a); }
}
constexpr double sin2pi(int j, int r) {
    j %= r; if (j < 0) j += r;
    int q = (4 * j) / r;
    int rem = 4 * j - q * r;
    double a = (PI / 2) * ((double)rem / (double)r);
    switch (q) { case 0: return sin_taylor(a); case 1: return cos_taylor(a);
                 case 2: return -sin_taylor(a); default: return -cos_taylor(a); }
}
}  // namespace cx

// W_R^J = exp(-2*pi*i*J/R) (forward) as fp32 constants
template <int R, int J> struct Tw {
    static constexpr float re = (float)cx::cos2pi(J, R);
    static constexpr float im = (float)(-cx::sin2pi(J, R));
};

// a * W_R^E (forward) or a * conj(W_R^E) (inverse), with the trivial cases folded away
template <int R, int E, bool INV> D4W_HD float2 cmul_tw(float2 a) {
    constexpr int e = ((E % R) + R) % R;
    if constexpr (e == 0) {
        return a;
    } else if constexpr (2 * e == R) {
        return make_float2(-a.x, -a.y);
    } else if constexpr (4 * e == R) {            // W = -i (fwd), +i (inv)
        return INV ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x);
    } else if constexpr (4 * e == 3 * R) {        // W = +i (fwd), -i (inv)
        return INV ? make_float2(a.y, -a.x) : make_float2(-a.y, a.x);
    } else {
        constexpr float wr = Tw<R, e>::re;
        constexpr float wi = INV ? -Tw<R, e>::im : Tw<R, e>::im;
        return make_float2(fmaf(a.x, wr, -a.y * wi), fmaf(a.x, wi, a.y * wr));
    }
}

// ---------------------------------------------------------------- static_for
template <class F, int... I>
D4W_HD void static_for_impl(F&& f, std::integer_sequence<int, I...>) {
    (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F> D4W_HD void static_for(F&& f) {
    static_for_impl(static_cast<F&&>(f), std::make_integer_sequence<int, N>{});
}

// ---------------------------------------------------------------- DFT<R, INV>
// In-place on v[0..R): v[k] = sum_n v[n] * exp(-/+ 2*pi*i*n*k/R), natural order in and out.
template <int R, bool INV> struct DFT;

template <bool INV> struct DFT<1, INV> { static D4W_HD void run(float2 (&)[1]) {} };

template <bool INV> struct DFT<2, INV> {
    static D4W_HD void run(float2 (&v)[2]) {
        float2 a = v[0], b = v[1];
        v[0] = cadd(a, b); v[1] = csub(a, b);
    }
};

template <bool INV> struct DFT<3, INV> {
    static D4W_HD void run(float2 (&v)[3]) {
        constexpr float s = INV ? 0.86602540378443864676f : -0.86602540378443864676f;  // Im(W_3)
        float2 t = cadd(v[1], v[2]);
        float2 d = csub(v[1], v[2]);
        float2 m = make_float2(fmaf(-0.5f, t.x, v[0].x), fmaf(-0.5f, t.y, v[0].y));
        v[0] = cadd(v[0], t);
        float2 r = make_float2(-s * d.y, s * d.x);      // i*s*d
        v[1] = cadd(m, r);
        v[2] = csub(m, r);
    }
};

template <bool INV> struct DFT<4, INV> {
    static D4W_HD void run(float2 (&v)[4]) {
        float2 a = cadd(v[0], v[2]), b = csub(v[0], v[2]);
        float2 c = cadd(v[1], v[3]), d = csub(v[1], v[3]);
        // forward: -i*d ; inverse: +i*d
        float2 jd = INV ? make_float2(-d.y, d.x) : make_float2(d.y, -d.x);
        v[0] = cadd(a, c); v[2] = csub(a, c);
        v[1] = cadd(b, jd); v[3] = csub(b, jd);
    }
};

template <bool INV> struct DFT<5, INV> {
    static D4W_HD void run(float2 (&v)[5]) {
        constexpr float c1 = 0.30901699437494742410f;    // cos(2pi/5)
        constexpr float c2 = -0.80901699437494742410f;   // cos(4pi/5)
        constexpr float s1 = INV ? 0.95105651629515357212f : -0.95105651629515357212f;  // -/+ sin(2pi/5)
        constexpr float s2 = INV ? 0.58778525229247312917f : -0.58778525229247312917f;  // -/+ sin(4pi/5)
        float2 t1 = cadd(v[1], v[4]), d1 = csub(v[1], v[4]);
        float2 t2 = cadd(v[2], v[3]), d2 = csub(v[2], v[3]);
        float2 a0 = v[0];
        v[0] = make_float2(a0.x + t1.x + t2.x, a0.y + t1.y + t2.y);
        float2 m1 = make_float2(fmaf(c1, t1.x, fmaf(c2, t2.x, a0.x)), fmaf(c1, t1.y, fmaf(c2, t2.y, a0.y)));
        float2 m2 = make_float2(fmaf(c2, t1.x, fmaf(c1, t2.x, a0.x)), fmaf(c2, t1.y, fmaf(c1, t2.y, a0.y)));
        // i * (s1*d1 + s2*d2) and i * (s2*d1 - s1*d2)
        float2 u1 = make_float2(fmaf(s1, d1.x, s2 * d2.x), fmaf(s1, d1.y, s2 * d2.y));
        float2 u2 = make_float2(fmaf(s2, d1.x, -s1 * d2.x), fmaf(s2, d1.y, -s1 * d2.y));
        float2 r1 = make_float2(-u1.y, u1.x), r2 = make_float2(-u2.y, u2.x);
        v[1] = cadd(m1, r1); v[4] = csub(m1, r1);
        v[2] = cadd(m2, r2); v[3] = csub(m2, r2);
    }
};

template <int R> constexpr int pick_r1() {
    return (R % 4 == 0) ? 4 : (R % 2 == 0) ? 2 : (R % 3 == 0) ? 3 : (R % 5 == 0) ? 5 : R;
}

// Composite radix: R = R1 * R2, decimation with n = R2*n1 + n2, k = k1 + R1*k2.
template <int R, bool INV> struct DFT {
    static constexpr int R1 = pick_r1<R>();
    static constexpr int R2 = R / R1;
    static_assert(R1 != R, "prime radix > 5 has no in-register butterfly (handled by the generic smem stage)");
    static D4W_HD void run(float2 (&v)[R]) {
        float2 t[R];
        static_for<R2>([&](auto n2c) {
            constexpr int n2 = decltype(n2c)::value;
            float2 a[R1];
            static_for<R1>([&](auto n1c) { constexpr int n1 = decltype(n1c)::value; a[n1] = v[R2 * n1 + n2]; });
            DFT<R1, INV>::run(a);
            static_for<R1>([&](auto k1c) {
                constexpr int k1 = decltype(k1c)::value;
                t[n2 * R1 + k1] = cmul_tw<R, n2 * k1, INV>(a[k1]);
            });
        });
        static_for<R1>([&](auto k1c) {
            constexpr int k1 = decltype(k1c)::value;
            float2 b[R2];
            static_for<R2>([&](auto n2c) { constexpr int n2 = decltype(n2c)::value; b[n2] = t[n2 * R1 + k1]; });
            DFT<R2, INV>::run(b);
            static_for<R2>([&](auto k2c) { constexpr int k2 = decltype(k2c)::value; v[k1 + R1 * k2] = b[k2]; });
        });
    }
};

// Powers of a unit twiddle w: p[m] = w^m for m = 1..R-1 by a balanced product tree
// (depth ~log2 m, so rounding stays ~1e-7).  FWD uses w, INV the conjugate.
template <int R> D4W_HD void twiddle_powers(float2 w, float2 (&p)[R]) {
    p[0] = make_float2(1.f, 0.f);
    if constexpr (R > 1) p[1] = w;
    static_for<R>([&](auto mc) {
        constexpr int m = decltype(mc)::value;
        if constexpr (m >= 2) { p[m] = cmul(p[m / 2], p[m - m / 2]); }
    });
}

}  // namespace d4w
