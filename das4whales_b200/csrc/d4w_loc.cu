// d4w_loc.cu -- localisation of a batch of calls (C ABI d4w_loc_* in include/d4w.h): the grid-searched first guess
// (k_loc_grid, k_loc_pick) and the Gauss-Newton solve of loc.solve_lq with its covariance epilogue (k_loc_gn).  The CTA
// bodies are loc_kernels.cuh.
#include <climits>
#include <string>
#include "d4w_common.hpp"
#include "loc_kernels.cuh"

using namespace d4w;

namespace {

__global__ void __launch_bounds__(kLocGridThreads)
k_loc_grid(LocGridParams g, LocBest* __restrict__ ws) {
    extern __shared__ __align__(16) double loc_grid_smem[];
    loc_grid_body(g, (int)blockIdx.x, (int)blockIdx.y, threadIdx.x, blockDim.x, loc_grid_smem, ws);
}

__global__ void __launch_bounds__(kLocPickThreads)
k_loc_pick(LocGridParams g, const LocBest* __restrict__ ws, long long* __restrict__ index, double* __restrict__ score,
           double* __restrict__ n0) {
    __shared__ LocBest red[kLocPickThreads];
    loc_pick_body(g, ws, (int)blockIdx.x, threadIdx.x, blockDim.x, red, index, score, n0);
}

__global__ void __launch_bounds__(kLocGnThreads)
k_loc_gn(LocSolveParams sp) {
    __shared__ double gn_smem[kLocSums * kLocGnThreads + 4];
    loc_gn_body(sp, (int)blockIdx.x, threadIdx.x, blockDim.x, gn_smem);
}

long long loc_tiles(long long nnodes) { return (nnodes + (long long)kLocGridThreads * kLocGridNodes - 1) / ((long long)kLocGridThreads * kLocGridNodes); }

std::string loc_grid_args(int ncalls, int nx, int ny, int nz) {
    if (ncalls < 1) return "ncalls must be >= 1";
    if (nx < 1 || ny < 1 || nz < 1) return "nx, ny and nz must be >= 1";
    if (loc_tiles((long long)nx * ny * nz) > INT_MAX) return "too many grid nodes";
    return "";
}

}  // namespace

extern "C" size_t d4w_loc_grid_workspace_bytes(int ncalls, int nx, int ny, int nz) {
    if (!loc_grid_args(ncalls, nx, ny, nz).empty()) return 0;
    return (size_t)ncalls * (size_t)loc_tiles((long long)nx * ny * nz) * sizeof(LocBest);
}

extern "C" int d4w_loc_grid(const double* T, const double* pos, const long long* offsets, int ncalls, double c0, int fix_z,
                            const double* gx, int nx, const double* gy, int ny, const double* gz, int nz, void* ws,
                            long long* index, double* score, double* n0, void* stream_v) {
    const std::string bad = loc_grid_args(ncalls, nx, ny, nz);
    if (!bad.empty()) return fail(D4W_ERR_ARG, "d4w_loc_grid: " + bad);
    if (!(c0 > 0.0)) return fail(D4W_ERR_ARG, "d4w_loc_grid: c0 must be > 0");
    if (fix_z && nz != 1) return fail(D4W_ERR_ARG, "d4w_loc_grid: fix_z needs nz = 1");
    if (!T || !pos || !offsets || !gx || !gy || !gz || !ws || !index || !score || !n0)
        return fail(D4W_ERR_ARG, "d4w_loc_grid: null pointer");
    LocGridParams g{};
    g.T = T; g.pos = pos; g.off = offsets; g.gx = gx; g.gy = gy; g.gz = gz;
    g.nx = nx; g.ny = ny; g.nz = nz;
    g.nnodes = (long long)nx * ny * nz;
    g.tile = (long long)kLocGridThreads * kLocGridNodes;
    g.ntiles = (int)loc_tiles(g.nnodes);
    g.p = fix_z ? 3 : 4;
    g.inv_c0 = 1.0 / c0;
    cudaStream_t st = (cudaStream_t)stream_v;
    const size_t smem = loc_grid_smem_bytes(kLocGridThreads);
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_loc_grid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LocBest* w = static_cast<LocBest*>(ws);
    return for_row_blocks(ncalls, kMaxGridRows, [&](size_t c, int m) -> int {         // one call per blockIdx.y
        LocGridParams gc = g;
        gc.off = offsets + c;
        LocBest* wc = w + c * g.ntiles;
        k_loc_grid<<<dim3((unsigned)g.ntiles, (unsigned)m), kLocGridThreads, smem, st>>>(gc, wc);
        D4W_CHECK_LAUNCH("k_loc_grid");
        k_loc_pick<<<(unsigned)m, kLocPickThreads, 0, st>>>(gc, wc, index + c, score + c, n0 + 4 * c);
        D4W_CHECK_LAUNCH("k_loc_pick");
        return D4W_OK;
    });
}

extern "C" int d4w_loc_solve(const double* T, const double* pos, const long long* offsets, int ncalls, double c0, int nbiter,
                             int fix_z, const double* n0, double* n, double* var, double* unc, double* cinv, double* cond,
                             double* traj, double* n0_used, void* stream_v) {
    if (ncalls < 1) return fail(D4W_ERR_ARG, "d4w_loc_solve: ncalls must be >= 1");
    if (nbiter < 0) return fail(D4W_ERR_ARG, "d4w_loc_solve: nbiter must be >= 0");
    if (!(c0 > 0.0)) return fail(D4W_ERR_ARG, "d4w_loc_solve: c0 must be > 0");
    if (!T || !pos || !offsets || !n || !var || !unc) return fail(D4W_ERR_ARG, "d4w_loc_solve: null pointer");
    LocSolveParams sp{};
    sp.T = T; sp.pos = pos; sp.off = offsets; sp.n0 = n0;
    sp.nbiter = nbiter; sp.fix_z = fix_z ? 1 : 0; sp.c0 = c0;
    sp.n = n; sp.var = var; sp.unc = unc; sp.cinv = cinv; sp.cond = cond; sp.traj = traj; sp.n0_used = n0_used;
    k_loc_gn<<<(unsigned)ncalls, kLocGnThreads, 0, (cudaStream_t)stream_v>>>(sp);
    D4W_CHECK_LAUNCH("k_loc_gn");
    return D4W_OK;
}
