// assoc_kernels.cuh -- pick association by back-projection over a source grid (d4w_loc_associate, d4w_assoc.cu), in FP64.
//
// Picks are a CSR by channel: channel c holds samples s[off[c] .. off[c + 1]), at cable_pos[c] (m).  For node g and pick p
// of channel c: T_p = s_p / fs, tau(g, c) = sqrt(dx dx + dy dy + dz dz) / c0 with dx = cable_pos[c].x - g_x, o = T_p - tau
// and the bin j = floor(o r), r = 1 / h, h = tol / 2.  Every operation is rounded on its own (no fused multiply-add; the
// __d*_rn intrinsics on the device, contraction off on the host), so a float64 NumPy restatement gives the same bins.
//
// Extraction k: the vote counts the unassigned picks per (node, bin) and scores (g, j) by n(g, j) + n(g, j + 1); the best
// (score, then lowest node, then lowest j) becomes call k when its score reaches min_picks, and its picks are labelled k.
//
// Kernels, all deterministic (integer counts, fixed-order reductions):
//   assoc_prep_body    one CTA: T_p into the workspace, labels = -1, the range of samples and the bounding boxes of the
//                      picked channels and of the grid (assoc_bin_range turns them into the bin range [jlo, jlo + nbins))
//   assoc_vote_body    one CTA per kAssocNodes nodes: counts in shared memory (one row of nbins + 1 ints per node), tau once
//                      per (node, picked channel), then the tile's best (score, node, j) into the workspace
//   assoc_pick_body    one CTA: the best of the tiles; writes call k when it qualifies
//   assoc_assign_body  one thread per channel: labels the winning window's picks
//
// The bodies are __host__ __device__ with (block, tid, nthr, smem) loops, so tests/host_emul/assoc_emul.cu runs them on the
// CPU; nthr must be a power of two.
#pragma once
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

constexpr int kAssocThreads = 256;
constexpr int kAssocNodes = 4;                 // nodes per vote CTA: one load of a channel's position and picks serves all
constexpr int kAssocPrepThreads = 256;
constexpr int kAssocPickThreads = 256;
constexpr int kAssocSmemMax = 227 * 1024;      // opt-in shared memory of an sm_90 block

struct AssocBest {
    long long node;                            // LLONG_MAX: none
    long long j;                               // absolute bin
    int score;                                 // -1: none
    int bad;                                   // a bin fell outside [jlo, jlo + nbins): the caller's range is wrong
};

struct AssocRange {
    int smin, smax;                            // sample range (smin < 0 flags a negative sample)
    int bad_offsets;                           // off[0] != 0, off[nch] != npicks or a decreasing offset
    int pad;
    double box[12];                            // picked cable min x, y, z, max x, y, z; grid min x, y, z, max x, y, z
};

struct AssocParams {
    const int* off;                            // [nch + 1]
    const int* s;                              // [npicks] samples
    int nch;
    long long npicks;
    double fs;
    const double* pos;                         // [>= nch][3]
    double c0;
    const double* gx;
    const double* gy;
    const double* gz;
    int nx, ny, nz;
    long long nnodes;
    int ntiles;
    double h, r;
    long long jlo;
    int nbins;
    int min_picks;
    double* T;                                 // [npicks] workspace: s / fs
    long long* labels;                         // [npicks]
};

__host__ __device__ inline bool assoc_better(const AssocBest& a, const AssocBest& b) {
    return a.score > b.score || (a.score == b.score && (a.node < b.node || (a.node == b.node && a.j < b.j)));
}

// tau(g, c): left to right, each operation rounded on its own
__host__ __device__ inline double assoc_tau(double gx, double gy, double gz, const double* q, double c0) {
#ifdef __CUDA_ARCH__
    const double dx = __dsub_rn(q[0], gx), dy = __dsub_rn(q[1], gy), dz = __dsub_rn(q[2], gz);
    return __ddiv_rn(__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))), c0);
#else
    const double dx = q[0] - gx, dy = q[1] - gy, dz = q[2] - gz;
    return sqrt(dx * dx + dy * dy + dz * dz) / c0;
#endif
}

__host__ __device__ inline long long assoc_bin(double T, double tau, double r) {
#ifdef __CUDA_ARCH__
    return (long long)floor(__dmul_rn(__dsub_rn(T, tau), r));
#else
    return (long long)floor((T - tau) * r);
#endif
}

__host__ __device__ inline void assoc_node(const AssocParams& P, long long i, double* g) {
    g[0] = P.gx[i % P.nx];
    g[1] = P.gy[(i / P.nx) % P.ny];
    g[2] = P.gz[i / ((long long)P.nx * P.ny)];
}

__host__ __device__ inline size_t assoc_vote_smem_bytes(int nbins, int nthr) {
    return (size_t)kAssocNodes * (size_t)(nbins + 1) * sizeof(int) + (size_t)nthr * sizeof(AssocBest);
}

// The largest bin count whose vote fits shared memory.
__host__ __device__ inline int assoc_max_bins() {
    return (int)((kAssocSmemMax - (size_t)kAssocThreads * sizeof(AssocBest)) / (kAssocNodes * sizeof(int))) - 1;
}

// [jlo, jlo + nbins) covers every bin: tau lies between the distances of the two bounding boxes (each axis' gap and
// span) over c0, with a relative margin far above the few rounding errors of assoc_tau / assoc_bin and two bins either side.
// false when the bounds are not finite or the range does not fit an int.
inline bool assoc_bin_range(double tmin, double tmax, const double* box, double c0, double r, long long* jlo,
                            long long* nbins) {
    double lo2 = 0.0, hi2 = 0.0;
    for (int a = 0; a < 3; ++a) {
        const double cmin = box[a], cmax = box[3 + a], gmin = box[6 + a], gmax = box[9 + a];
        const double gap = fmax(0.0, fmax(cmin - gmax, gmin - cmax));
        const double span = fmax(fabs(gmax - cmin), fabs(cmax - gmin));
        lo2 += gap * gap;
        hi2 += span * span;
    }
    const double tau_lo = sqrt(lo2) / c0, tau_hi = sqrt(hi2) / c0;
    const double m = 2.0 + 1e-9 * (fabs(tmin) + fabs(tmax) + tau_hi) * r;
    const double a = floor((tmin - tau_hi) * r - m), b = floor((tmax - tau_lo) * r + m);
    if (!(std::isfinite(a) && std::isfinite(b)) || fabs(a) > 4.0e18 || fabs(b) > 4.0e18 || b - a + 1.0 > (double)INT_MAX)
        return false;
    *jlo = (long long)a;
    *nbins = (long long)b - (long long)a + 1;
    return true;
}

// One CTA: T_p = s_p / fs, labels = -1, the sample range and the two bounding boxes.
__host__ __device__ inline void assoc_prep_body(const AssocParams& P, int tid, int nthr, void* smem, AssocRange* out) {
    double* red = static_cast<double*>(smem);                     // [12][nthr]
    int* ired = reinterpret_cast<int*>(red + 12 * (size_t)nthr);  // [3][nthr]
    int smin = INT_MAX, smax = INT_MIN, badoff = 0;
    for (long long p = tid; p < P.npicks; p += nthr) {
        const int s = P.s[p];
#ifdef __CUDA_ARCH__
        P.T[p] = __ddiv_rn((double)s, P.fs);
#else
        P.T[p] = (double)s / P.fs;
#endif
        P.labels[p] = -1;
        smin = s < smin ? s : smin;
        smax = s > smax ? s : smax;
    }
    double b[12];
    for (int a = 0; a < 3; ++a) { b[a] = INFINITY; b[3 + a] = -INFINITY; }
    for (int c = tid; c < P.nch; c += nthr) {
        const int o0 = P.off[c], o1 = P.off[c + 1];
        if (o1 < o0) badoff = 1;
        if (o1 <= o0) continue;
        for (int a = 0; a < 3; ++a) {
            const double v = P.pos[3 * (size_t)c + a];
            b[a] = fmin(b[a], v);
            b[3 + a] = fmax(b[3 + a], v);
        }
    }
    if (tid == 0 && (P.off[0] != 0 || (long long)P.off[P.nch] != P.npicks)) badoff = 1;
    const double* ax[3] = {P.gx, P.gy, P.gz};
    const int na[3] = {P.nx, P.ny, P.nz};
    for (int a = 0; a < 3; ++a) {
        double lo = INFINITY, hi = -INFINITY;
        for (int i = tid; i < na[a]; i += nthr) { lo = fmin(lo, ax[a][i]); hi = fmax(hi, ax[a][i]); }
        b[6 + a] = lo;
        b[9 + a] = hi;
    }
    for (int k = 0; k < 12; ++k) red[k * nthr + tid] = b[k];
    ired[tid] = smin; ired[nthr + tid] = smax; ired[2 * nthr + tid] = badoff;
    D4W_SYNC();
    for (int st = nthr / 2; st > 0; st >>= 1) {
        if (tid < st) {
            for (int k = 0; k < 12; ++k) {
                double& x = red[k * nthr + tid];
                const double y = red[k * nthr + tid + st];
                x = (k % 6) < 3 ? fmin(x, y) : fmax(x, y);
            }
            int* m = ired;
            m[tid] = m[tid + st] < m[tid] ? m[tid + st] : m[tid];
            m[nthr + tid] = m[nthr + tid + st] > m[nthr + tid] ? m[nthr + tid + st] : m[nthr + tid];
            m[2 * nthr + tid] |= m[2 * nthr + tid + st];
        }
        D4W_SYNC();
    }
    if (tid != 0) return;
    out->smin = ired[0];
    out->smax = ired[nthr];
    out->bad_offsets = ired[2 * nthr];
    out->pad = 0;
    for (int k = 0; k < 12; ++k) out->box[k] = red[k * nthr];
}

__host__ __device__ inline void assoc_count(int* c) {
#ifdef __CUDA_ARCH__
    atomicAdd(c, 1);
#else
    ++*c;
#endif
}

// One tile of kAssocNodes nodes: ws[tile] = its best (score, node, j) over the unassigned picks.
__host__ __device__ inline void assoc_vote_body(const AssocParams& P, int tile, int tid, int nthr, void* smem,
                                                AssocBest* __restrict__ ws) {
    const int stride = P.nbins + 1;                               // bin nbins stays 0: the partner of the last bin
    int* cnt = static_cast<int*>(smem);                           // [kAssocNodes][nbins + 1]
    AssocBest* red = reinterpret_cast<AssocBest*>(cnt + (size_t)kAssocNodes * stride);
    for (int k = tid; k < kAssocNodes * stride; k += nthr) cnt[k] = 0;
    const long long n0 = (long long)tile * kAssocNodes;
    int nn = 0;
    double g[kAssocNodes][3];
    for (int k = 0; k < kAssocNodes; ++k) {
        if (n0 + k < P.nnodes) { assoc_node(P, n0 + k, g[k]); nn = k + 1; }
        else { g[k][0] = g[k][1] = g[k][2] = 0.0; }
    }
    D4W_SYNC();
    int bad = 0;
    for (int c = tid; c < P.nch; c += nthr) {
        const int o0 = P.off[c], o1 = P.off[c + 1];
        if (o1 <= o0) continue;                                   // a channel with no pick
        const double* q = P.pos + 3 * (size_t)c;
        double tau[kAssocNodes];
#pragma unroll
        for (int k = 0; k < kAssocNodes; ++k) tau[k] = assoc_tau(g[k][0], g[k][1], g[k][2], q, P.c0);
        for (int p = o0; p < o1; ++p) {
            if (P.labels[p] >= 0) continue;
            const double T = P.T[p];
#pragma unroll
            for (int k = 0; k < kAssocNodes; ++k) {
                if (k >= nn) break;
                const long long j = assoc_bin(T, tau[k], P.r) - P.jlo;
                if (j < 0 || j >= P.nbins) { bad = 1; continue; }
                assoc_count(&cnt[k * stride + j]);
            }
        }
    }
    D4W_SYNC();
    AssocBest best{LLONG_MAX, LLONG_MAX, -1, bad};
    for (int k = 0; k < nn; ++k)
        for (int j = tid; j < P.nbins; j += nthr) {
            const AssocBest c{n0 + k, P.jlo + j, cnt[k * stride + j] + cnt[k * stride + j + 1], 0};
            if (assoc_better(c, best)) { best.node = c.node; best.j = c.j; best.score = c.score; }
        }
    red[tid] = best;
    D4W_SYNC();
    for (int s = nthr / 2; s > 0; s >>= 1) {
        if (tid < s) {
            const int b = red[tid].bad | red[tid + s].bad;
            if (assoc_better(red[tid + s], red[tid])) red[tid] = red[tid + s];
            red[tid].bad = b;
        }
        D4W_SYNC();
    }
    if (tid == 0) ws[tile] = red[0];
}

// The best of the tiles into *rec; when its score reaches min_picks it is call k: node[k], t0[k] = (j + 1) h, count[k].
__host__ __device__ inline void assoc_pick_body(const AssocParams& P, const AssocBest* __restrict__ ws, int k, int tid,
                                                int nthr, void* smem, AssocBest* rec, long long* node, double* t0,
                                                long long* count) {
    AssocBest* red = static_cast<AssocBest*>(smem);
    AssocBest best{LLONG_MAX, LLONG_MAX, -1, 0};
    int bad = 0;
    for (int t = tid; t < P.ntiles; t += nthr) {
        const AssocBest c = ws[t];
        bad |= c.bad;
        if (assoc_better(c, best)) best = c;
    }
    best.bad = bad;
    red[tid] = best;
    D4W_SYNC();
    for (int s = nthr / 2; s > 0; s >>= 1) {
        if (tid < s) {
            const int b = red[tid].bad | red[tid + s].bad;
            if (assoc_better(red[tid + s], red[tid])) red[tid] = red[tid + s];
            red[tid].bad = b;
        }
        D4W_SYNC();
    }
    if (tid != 0) return;
    best = red[0];
    *rec = best;
    if (best.bad || best.score < P.min_picks) return;
    node[k] = best.node;
#ifdef __CUDA_ARCH__
    t0[k] = __dmul_rn((double)(best.j + 1), P.h);
#else
    t0[k] = (double)(best.j + 1) * P.h;
#endif
    count[k] = best.score;
}

// Channel c = block * nthr + tid: its unassigned picks in bins j and j + 1 of the winning node become call k.
__host__ __device__ inline void assoc_assign_body(const AssocParams& P, const AssocBest* rec, int k, int block, int tid,
                                                  int nthr) {
    const AssocBest b = *rec;
    if (b.bad || b.score < P.min_picks) return;
    const int c = block * nthr + tid;
    if (c >= P.nch) return;
    const int o0 = P.off[c], o1 = P.off[c + 1];
    if (o1 <= o0) return;
    double g[3];
    assoc_node(P, b.node, g);
    const double tau = assoc_tau(g[0], g[1], g[2], P.pos + 3 * (size_t)c, P.c0);
    for (int p = o0; p < o1; ++p) {
        if (P.labels[p] >= 0) continue;
        const long long j = assoc_bin(P.T[p], tau, P.r);
        if (j == b.j || j == b.j + 1) P.labels[p] = k;
    }
}

}  // namespace d4w
