// loc_kernels.cuh -- localisation of many calls at once (d4w_loc_grid / d4w_loc_solve, d4w_loc.cu): the Gauss-Newton
// solver of loc.solve_lq, the covariance rule of loc.calc_covariance_matrix (das4whales/loc.py:57-128, :156-216) and a
// grid-searched first guess, all in FP64.
//
// Call b is the observations [off[b], off[b + 1]) of T (arrival times, s) and pos ([n][3], m).  p = 4 unknowns
// (x, y, z, t0), or 3 with z held (fix_z).
//
// Grid (one CTA per (tile of nodes, call)): node i = (iz * ny + iy) * nx + ix at (gx[ix], gy[iy], gz[iz]); with
// R_j = T_j - d_j / c0 its sum of squares SS = sum (R_j - mean R)^2 and t0* = mean R.  Each thread owns kLocGridNodes
// nodes and sums (R_j - s) and (R_j - s)^2 in double with the node's own shift s = R_0 (the first observation), so
// that SS = S2 - S1^2 / n is a difference of numbers of the size of SS.  Observations are staged through shared memory
// kLocGridChunk at a time; the tile's argmin (ties to the lowest node index) goes to the workspace and loc_pick_body
// reduces the tiles of a call in the same way: nothing depends on timing or on the order CTAs run in.
//
// Gauss-Newton (one CTA per call): every iteration sums the p(p+1)/2 entries of G^T G and the p of G^T dt per thread in
// double, combines them by a fixed tree in shared memory, and thread 0 forms (G^T G + 1e-5 I)^-1 by Gauss-Jordan
// elimination with partial pivoting and steps by 0.7 dn (j < 4) or dn.  G's rows are the reference's:
// theta = atan2(|z - z_c|, r), phi = atan2(y - y_c, x - x_c), [cos th cos ph / c0, cos th sin ph / c0, (sin th / c0), 1].
// Epilogue: the residual variance (NaN when n <= p), G^T G at the final n, its 2-norm condition number from cyclic
// Jacobi (G^T G is symmetric), C = (G^T G)^-1, or (G^T G + 1e-5 I)^-1 when cond > 1 / DBL_EPSILON as the reference
// does, and unc = sqrt(var diag C).
//
// The bodies are __host__ __device__ with (block, tid, nthr, smem) loops, so tests/host_emul/loc_emul.cu runs them on the
// CPU; nthr must be a power of two.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>

#ifndef D4W_SYNC
#ifdef __CUDA_ARCH__
#define D4W_SYNC() __syncthreads()
#else
#define D4W_SYNC() ((void)0)
#endif
#endif

namespace d4w {

constexpr int kLocGridThreads = 256;
constexpr int kLocGridNodes = 4;        // nodes per thread: a tile is kLocGridThreads * kLocGridNodes nodes
constexpr int kLocGridChunk = 512;      // observations per shared-memory stage (16 KB)
constexpr int kLocPickThreads = 128;
constexpr int kLocGnThreads = 256;
constexpr int kLocSums = 14;            // 10 entries of G^T G + 4 of G^T dt
constexpr double kLocLambda = 1e-5;     // loc.py:89 and :185

struct LocBest {
    double ss;                          // sum of squared residuals at t0*
    double t0;                          // t0* = mean(T - d / c0)
    long long idx;                      // node index; -1 for an empty call
};

struct LocGridParams {
    const double* T;
    const double* pos;
    const long long* off;
    const double* gx;
    const double* gy;
    const double* gz;
    int nx, ny, nz;
    long long nnodes;
    long long tile;                     // nodes per tile = nthr * kLocGridNodes
    int ntiles;
    int p;
    double inv_c0;
};

struct LocSolveParams {
    const double* T;
    const double* pos;
    const long long* off;
    const double* n0;                   // [ncalls][4], or null: the reference's [40000, 23000, -60, min T]
    int nbiter, fix_z;
    double c0;
    double* n;                          // [ncalls][4]
    double* var;                        // [ncalls]
    double* unc;                        // [ncalls][p]
    double* cinv;                       // [ncalls][p][p] or null
    double* cond;                       // [ncalls] or null
    double* traj;                       // [ncalls][nbiter][4] or null
    double* n0_used;                    // [ncalls][4] or null: the first guess
};

__host__ __device__ inline bool loc_better(const LocBest& a, const LocBest& b) {
    return a.ss < b.ss || (a.ss == b.ss && a.idx < b.idx);
}

__host__ __device__ inline size_t loc_grid_smem_bytes(int nthr) {
    return (size_t)4 * kLocGridChunk * sizeof(double) + (size_t)nthr * sizeof(LocBest);
}

__host__ __device__ inline size_t loc_gn_smem_bytes(int nthr) {
    return (size_t)(kLocSums * nthr + 4) * sizeof(double);
}

// One (tile, call) of the grid search: ws[call * ntiles + tile] = the tile's best node.
__host__ __device__ inline void loc_grid_body(const LocGridParams& g, int tile, int call, int tid, int nthr, void* smem,
                                              LocBest* __restrict__ ws) {
    double* ox = static_cast<double*>(smem);
    double* oy = ox + kLocGridChunk;
    double* oz = oy + kLocGridChunk;
    double* ot = oz + kLocGridChunk;
    LocBest* red = reinterpret_cast<LocBest*>(ot + kLocGridChunk);
    const long long o0 = g.off[call], n = g.off[call + 1] - o0;
    LocBest* out = ws + (size_t)call * g.ntiles + tile;
    if (n <= 0) {
        if (tid == 0) *out = LocBest{NAN, NAN, -1};
        return;
    }
    const double* T = g.T + o0;
    const double* P = g.pos + 3 * o0;
    double vx[kLocGridNodes], vy[kLocGridNodes], vz[kLocGridNodes], sh[kLocGridNodes], s1[kLocGridNodes], s2[kLocGridNodes];
    const long long base = (long long)tile * g.tile + tid;
    for (int k = 0; k < kLocGridNodes; ++k) {
        long long i = base + (long long)k * nthr;
        if (i >= g.nnodes) i = g.nnodes - 1;             // padding lanes recompute the last node and are ignored below
        const long long ix = i % g.nx, iy = (i / g.nx) % g.ny, iz = i / ((long long)g.nx * g.ny);
        vx[k] = g.gx[ix]; vy[k] = g.gy[iy]; vz[k] = g.gz[iz];
        const double dx = vx[k] - P[0], dy = vy[k] - P[1], dz = vz[k] - P[2];
        sh[k] = T[0] - sqrt(dx * dx + dy * dy + dz * dz) * g.inv_c0;
        s1[k] = 0.0; s2[k] = 0.0;
    }
    for (long long c0 = 0; c0 < n; c0 += kLocGridChunk) {
        const int m = (int)(n - c0 < kLocGridChunk ? n - c0 : kLocGridChunk);
        for (int j = tid; j < m; j += nthr) {
            const double* q = P + 3 * (c0 + j);
            ox[j] = q[0]; oy[j] = q[1]; oz[j] = q[2]; ot[j] = T[c0 + j];
        }
        D4W_SYNC();
        for (int j = 0; j < m; ++j) {
            const double px = ox[j], py = oy[j], pz = oz[j], t = ot[j];
#pragma unroll
            for (int k = 0; k < kLocGridNodes; ++k) {
                const double dx = vx[k] - px, dy = vy[k] - py, dz = vz[k] - pz;
                const double r = (t - sqrt(dx * dx + dy * dy + dz * dz) * g.inv_c0) - sh[k];
                s1[k] += r;
                s2[k] += r * r;
            }
        }
        D4W_SYNC();                                       // the chunk is restaged next pass
    }
    LocBest best{INFINITY, NAN, LLONG_MAX};
    for (int k = 0; k < kLocGridNodes; ++k) {
        const long long i = base + (long long)k * nthr;
        if (i >= g.nnodes) break;
        const LocBest c{s2[k] - s1[k] * s1[k] / (double)n, sh[k] + s1[k] / (double)n, i};
        if (loc_better(c, best)) best = c;
    }
    red[tid] = best;
    D4W_SYNC();
    for (int s = nthr / 2; s > 0; s >>= 1) {
        if (tid < s && loc_better(red[tid + s], red[tid])) red[tid] = red[tid + s];
        D4W_SYNC();
    }
    if (tid == 0) *out = red[0];
}

// One call: the best of its tiles -> index[call], score[call] = SS / (n - p) (NaN when n <= p), n0[call] = node, t0*.
__host__ __device__ inline void loc_pick_body(const LocGridParams& g, const LocBest* __restrict__ ws, int call, int tid, int nthr,
                                              void* smem, long long* __restrict__ index, double* __restrict__ score,
                                              double* __restrict__ n0) {
    LocBest* red = static_cast<LocBest*>(smem);
    LocBest best{INFINITY, NAN, LLONG_MAX};
    for (int t = tid; t < g.ntiles; t += nthr) {
        const LocBest c = ws[(size_t)call * g.ntiles + t];
        if (loc_better(c, best)) best = c;
    }
    red[tid] = best;
    D4W_SYNC();
    for (int s = nthr / 2; s > 0; s >>= 1) {
        if (tid < s && loc_better(red[tid + s], red[tid])) red[tid] = red[tid + s];
        D4W_SYNC();
    }
    if (tid != 0) return;
    const long long n = g.off[call + 1] - g.off[call];
    best = red[0];
    double* o = n0 + 4 * (size_t)call;
    if (n <= 0 || best.idx == LLONG_MAX) {               // empty call (or every score NaN)
        index[call] = -1; score[call] = NAN;
        o[0] = o[1] = o[2] = o[3] = NAN;
        return;
    }
    const long long i = best.idx;
    index[call] = i;
    score[call] = n > g.p ? best.ss / (double)(n - g.p) : NAN;
    o[0] = g.gx[i % g.nx]; o[1] = g.gy[(i / g.nx) % g.ny]; o[2] = g.gz[i / ((long long)g.nx * g.ny)]; o[3] = best.t0;
}

// The row of G at observation (x, y, z) for the estimate v = (x, y, z, t0) (loc.py:92-110), packed to the p unknowns, and
// dt = T - (t0 + d / c0) (loc.py:94, :23).
__host__ __device__ inline void loc_g_row(const double* v, const double* q, double t, double c0, int fix_z, double* g, double* dt) {
    const double ex = q[0] - v[0], ey = q[1] - v[1], ez = q[2] - v[2];
    const double r = sqrt(ex * ex + ey * ey);
    const double th = atan2(fabs(v[2] - q[2]), r);
    const double ph = atan2(v[1] - q[1], v[0] - q[0]);
    const double ct = cos(th), st = sin(th), cp = cos(ph), sp = sin(ph);
    g[0] = ct * cp / c0;
    g[1] = ct * sp / c0;
    if (fix_z) {
        g[2] = 1.0;
    } else {
        g[2] = st / c0;
        g[3] = 1.0;
    }
    *dt = t - (v[3] + sqrt(ex * ex + ey * ey + ez * ez) / c0);
}

// out = M^-1 of the p x p matrix M (row-major, destroyed), Gauss-Jordan with partial pivoting.  A zero pivot gives inf/NaN,
// as numpy's inv would raise; G^T G + 1e-5 I never has one.
__host__ __device__ inline void loc_inverse(int p, double* M, double* out) {
    for (int i = 0; i < p; ++i)
        for (int j = 0; j < p; ++j) out[i * p + j] = i == j ? 1.0 : 0.0;
    for (int c = 0; c < p; ++c) {
        int piv = c;
        for (int r = c + 1; r < p; ++r)
            if (fabs(M[r * p + c]) > fabs(M[piv * p + c])) piv = r;
        if (piv != c)
            for (int j = 0; j < p; ++j) {
                double t = M[c * p + j]; M[c * p + j] = M[piv * p + j]; M[piv * p + j] = t;
                t = out[c * p + j]; out[c * p + j] = out[piv * p + j]; out[piv * p + j] = t;
            }
        const double d = M[c * p + c];
        for (int j = 0; j < p; ++j) { M[c * p + j] /= d; out[c * p + j] /= d; }
        for (int r = 0; r < p; ++r) {
            if (r == c) continue;
            const double f = M[r * p + c];
            if (f == 0.0) continue;
            for (int j = 0; j < p; ++j) { M[r * p + j] -= f * M[c * p + j]; out[r * p + j] -= f * out[c * p + j]; }
        }
    }
}

// 2-norm condition number of the symmetric p x p matrix A (row-major, destroyed): max |lambda| / min |lambda| by cyclic
// Jacobi rotations; inf when an eigenvalue is exactly 0 (np.linalg.cond's SVD gives the same ratio for a symmetric matrix).
__host__ __device__ inline double loc_cond_sym(int p, double* A) {
    for (int sweep = 0; sweep < 16; ++sweep) {
        double off = 0.0, dia = 0.0;
        for (int i = 0; i < p; ++i) {
            dia += A[i * p + i] * A[i * p + i];
            for (int j = i + 1; j < p; ++j) off += A[i * p + j] * A[i * p + j];
        }
        if (off <= 1e-34 * dia) break;
        for (int a = 0; a < p; ++a)
            for (int b = a + 1; b < p; ++b) {
                const double apq = A[a * p + b];
                if (apq == 0.0) continue;
                const double th = (A[b * p + b] - A[a * p + a]) / (2.0 * apq);
                const double t = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < p; ++k) {                    // A <- J^T A J on columns a, b, then rows a, b
                    const double ka = A[k * p + a], kb = A[k * p + b];
                    A[k * p + a] = c * ka - s * kb;
                    A[k * p + b] = s * ka + c * kb;
                }
                for (int k = 0; k < p; ++k) {
                    const double ak = A[a * p + k], bk = A[b * p + k];
                    A[a * p + k] = c * ak - s * bk;
                    A[b * p + k] = s * ak + c * bk;
                }
            }
    }
    double lo = INFINITY, hi = 0.0;
    for (int i = 0; i < p; ++i) {
        const double e = fabs(A[i * p + i]);
        lo = e < lo ? e : lo;
        hi = e > hi ? e : hi;
    }
    return lo == 0.0 ? INFINITY : hi / lo;
}

// sum part[v * nthr + t] over t into part[v * nthr], for v < nv, by a fixed tree
__host__ __device__ inline void loc_block_sum(double* part, int nv, int tid, int nthr) {
    D4W_SYNC();
    for (int s = nthr / 2; s > 0; s >>= 1) {
        if (tid < s)
            for (int v = 0; v < nv; ++v) part[v * nthr + tid] += part[v * nthr + tid + s];
        D4W_SYNC();
    }
}

// One call of the Gauss-Newton solve and its epilogue; p = 3 (fix_z) or 4 unknowns, so that the sums stay in registers.
template <int p>
__host__ __device__ inline void loc_gn_body_p(const LocSolveParams& sp, int call, int tid, int nthr, void* smem) {
    double* part = static_cast<double*>(smem);           // [kLocSums][nthr]
    double* nv = part + (size_t)kLocSums * nthr;         // [4] the estimate
    constexpr int na = p * (p + 1) / 2;                  // lower triangle of G^T G, row by row
    const long long o0 = sp.off[call], n = sp.off[call + 1] - o0;
    const double* T = sp.T + o0;
    const double* P = sp.pos + 3 * o0;
    if (n <= 0) {
        if (tid != 0) return;
        for (int k = 0; k < 4; ++k) sp.n[4 * (size_t)call + k] = NAN;
        sp.var[call] = NAN;
        for (int k = 0; k < p; ++k) sp.unc[(size_t)call * p + k] = NAN;
        if (sp.cinv) for (int k = 0; k < p * p; ++k) sp.cinv[(size_t)call * p * p + k] = NAN;
        if (sp.cond) sp.cond[call] = NAN;
        if (sp.traj) for (int k = 0; k < 4 * sp.nbiter; ++k) sp.traj[(size_t)call * sp.nbiter * 4 + k] = NAN;
        if (sp.n0_used) for (int k = 0; k < 4; ++k) sp.n0_used[4 * (size_t)call + k] = NAN;
        return;
    }
    if (sp.n0) {
        if (tid == 0) for (int k = 0; k < 4; ++k) nv[k] = sp.n0[4 * (size_t)call + k];
    } else {                                             // loc.py:86: [40000, 23000, -60, min(Ti)]
        double m = INFINITY;
        for (long long i = tid; i < n; i += nthr) m = T[i] < m ? T[i] : m;
        part[tid] = m;
        D4W_SYNC();
        for (int s = nthr / 2; s > 0; s >>= 1) {
            if (tid < s && part[tid + s] < part[tid]) part[tid] = part[tid + s];
            D4W_SYNC();
        }
        if (tid == 0) { nv[0] = 40000.0; nv[1] = 23000.0; nv[2] = -60.0; nv[3] = part[0]; }
    }
    if (tid == 0 && sp.n0_used)
        for (int k = 0; k < 4; ++k) sp.n0_used[4 * (size_t)call + k] = nv[k];
    D4W_SYNC();
    const int upd[4] = {0, 1, p == 3 ? 3 : 2, 3};        // unknown k -> index in (x, y, z, t0)
    for (int j = 0; j <= sp.nbiter; ++j) {
        const bool last = j == sp.nbiter;                // the epilogue pass: G^T G without lambda and sum dt^2
        double v[4] = {nv[0], nv[1], nv[2], nv[3]};
        double acc[na + p];
#pragma unroll
        for (int k = 0; k < na + p; ++k) acc[k] = 0.0;
        for (long long i = tid; i < n; i += nthr) {
            double g[4], dt;
            loc_g_row(v, P + 3 * i, T[i], sp.c0, p == 3, g, &dt);
#pragma unroll
            for (int a = 0; a < p; ++a)
#pragma unroll
                for (int b = 0; b <= a; ++b) acc[a * (a + 1) / 2 + b] += g[a] * g[b];
            if (last) {
                acc[na] += dt * dt;
            } else {
#pragma unroll
                for (int a = 0; a < p; ++a) acc[na + a] += g[a] * dt;
            }
        }
        const int nsum = last ? na + 1 : na + p;
#pragma unroll
        for (int k = 0; k < na + p; ++k)
            if (k < nsum) part[k * nthr + tid] = acc[k];
        loc_block_sum(part, nsum, tid, nthr);
        if (tid == 0) {
            double A[16], Ai[16];
            int e = 0;
            for (int a = 0; a < p; ++a)
                for (int b = 0; b <= a; ++b) { A[a * p + b] = A[b * p + a] = part[(e++) * nthr]; }
            if (!last) {
                for (int a = 0; a < p; ++a) A[a * p + a] += kLocLambda;
                loc_inverse(p, A, Ai);
                const double step = j < 4 ? 0.7 : 1.0;   // loc.py:117-120
                for (int a = 0; a < p; ++a) {
                    double dn = 0.0;
                    for (int b = 0; b < p; ++b) dn += Ai[a * p + b] * part[(na + b) * nthr];
                    nv[upd[a]] += step * dn;
                }
                if (sp.traj)
                    for (int k = 0; k < 4; ++k) sp.traj[((size_t)call * sp.nbiter + j) * 4 + k] = nv[k];
            } else {
                const double var = n > p ? part[na * nthr] / (double)(n - p) : NAN;   // loc.py:148-153
                double B[16];
                for (int k = 0; k < p * p; ++k) B[k] = A[k];
                const double cond = loc_cond_sym(p, B);
                if (cond > 1.0 / DBL_EPSILON)                                          // loc.py:183-187
                    for (int a = 0; a < p; ++a) A[a * p + a] += kLocLambda;
                loc_inverse(p, A, Ai);
                for (int k = 0; k < 4; ++k) sp.n[4 * (size_t)call + k] = nv[k];
                sp.var[call] = var;
                for (int a = 0; a < p; ++a) sp.unc[(size_t)call * p + a] = sqrt(var * Ai[a * p + a]);
                if (sp.cinv) for (int k = 0; k < p * p; ++k) sp.cinv[(size_t)call * p * p + k] = Ai[k];
                if (sp.cond) sp.cond[call] = cond;
            }
        }
        D4W_SYNC();                                      // nv and part are read / rewritten next pass
    }
}

__host__ __device__ inline void loc_gn_body(const LocSolveParams& sp, int call, int tid, int nthr, void* smem) {
    if (sp.fix_z) loc_gn_body_p<3>(sp, call, tid, nthr, smem);
    else loc_gn_body_p<4>(sp, call, tid, nthr, smem);
}

}  // namespace d4w
