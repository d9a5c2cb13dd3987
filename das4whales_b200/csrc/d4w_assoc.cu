// d4w_assoc.cu -- pick association by back-projection (C ABI d4w_loc_assoc_* / d4w_loc_associate in include/d4w.h): a
// prep kernel (arrival times, labels, bin range), then per call a vote over nodes x picks with the assigned picks masked
// (k_assoc_vote), the best window (k_assoc_pick) and the labelling of its picks (k_assoc_assign).  The CTA bodies are
// assoc_kernels.cuh.
#include <climits>
#include <string>
#include "d4w_common.hpp"
#include "assoc_kernels.cuh"

using namespace d4w;

namespace {

__global__ void __launch_bounds__(kAssocPrepThreads)
k_assoc_prep(AssocParams P, AssocRange* __restrict__ out) {
    __shared__ __align__(16) double prep_smem[12 * kAssocPrepThreads + 2 * kAssocPrepThreads];
    assoc_prep_body(P, threadIdx.x, blockDim.x, prep_smem, out);
}

__global__ void __launch_bounds__(kAssocThreads)
k_assoc_vote(AssocParams P, AssocBest* __restrict__ ws) {
    extern __shared__ __align__(16) int assoc_vote_smem[];
    assoc_vote_body(P, (int)blockIdx.x, threadIdx.x, blockDim.x, assoc_vote_smem, ws);
}

__global__ void __launch_bounds__(kAssocPickThreads)
k_assoc_pick(AssocParams P, const AssocBest* __restrict__ ws, int k, AssocBest* rec, long long* node, double* t0,
             long long* count) {
    __shared__ AssocBest red[kAssocPickThreads];
    assoc_pick_body(P, ws, k, threadIdx.x, blockDim.x, red, rec, node, t0, count);
}

__global__ void __launch_bounds__(kAssocThreads)
k_assoc_assign(AssocParams P, const AssocBest* __restrict__ rec, int k) {
    assoc_assign_body(P, rec, k, (int)blockIdx.x, threadIdx.x, blockDim.x);
}

long long assoc_tiles(long long nnodes) { return (nnodes + kAssocNodes - 1) / kAssocNodes; }

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// workspace: T [npicks] | tile bests [ntiles] | record | range
struct AssocWs {
    double* T;
    AssocBest* tiles;
    AssocBest* rec;
    AssocRange* range;
    size_t bytes;
};

AssocWs assoc_ws(void* base, long long npicks, long long ntiles) {
    char* p = static_cast<char*>(base);
    AssocWs w{};
    size_t o = 0;
    w.T = reinterpret_cast<double*>(p + o);          o += align256((size_t)npicks * sizeof(double));
    w.tiles = reinterpret_cast<AssocBest*>(p + o);   o += align256((size_t)ntiles * sizeof(AssocBest));
    w.rec = reinterpret_cast<AssocBest*>(p + o);     o += align256(sizeof(AssocBest));
    w.range = reinterpret_cast<AssocRange*>(p + o);  o += align256(sizeof(AssocRange));
    w.bytes = o;
    return w;
}

std::string assoc_args(long long npicks, int nx, int ny, int nz) {
    if (npicks < 0 || npicks > INT_MAX) return "n_picks must be in [0, 2^31)";
    if (nx < 1 || ny < 1 || nz < 1) return "nx, ny and nz must be >= 1";
    if (assoc_tiles((long long)nx * ny * nz) > INT_MAX) return "too many grid nodes";
    return "";
}

}  // namespace

extern "C" int d4w_loc_assoc_bins(double t_min, double t_max, const double* host_box, double c0, double r,
                                  long long* jlo, int* nbins) {
    if (!host_box || !jlo || !nbins) return fail(D4W_ERR_ARG, "d4w_loc_assoc_bins: null pointer");
    if (!(c0 > 0.0) || !(r > 0.0)) return fail(D4W_ERR_ARG, "d4w_loc_assoc_bins: c0 and r must be > 0");
    long long lo = 0, n = 0;
    const int lim = assoc_max_bins();
    if (!assoc_bin_range(t_min, t_max, host_box, c0, r, &lo, &n) || n > lim)
        return fail(D4W_ERR_UNSUPPORTED, "the back-projected origin times span " +
                    (n > 0 ? std::to_string(n) : std::string("too many")) + " bins of tol / 2; at most " +
                    std::to_string(lim) + " fit one block's shared memory");
    *jlo = lo;
    *nbins = (int)n;
    return D4W_OK;
}

extern "C" size_t d4w_loc_assoc_workspace_bytes(long long n_picks, int nx, int ny, int nz) {
    if (!assoc_args(n_picks, nx, ny, nz).empty()) return 0;
    return assoc_ws(nullptr, n_picks, assoc_tiles((long long)nx * ny * nz)).bytes;
}

extern "C" int d4w_loc_associate(const int* offsets, const int* samples, int n_channels, long long n_picks, double fs,
                                 const double* cable_pos, double c0, const double* gx, int nx, const double* gy, int ny,
                                 const double* gz, int nz, double h, double r, int min_picks, int max_calls, void* ws,
                                 long long* labels, long long* node, double* t0, long long* count, int* n_calls,
                                 void* stream_v) {
    const std::string bad = assoc_args(n_picks, nx, ny, nz);
    if (!bad.empty()) return fail(D4W_ERR_ARG, "d4w_loc_associate: " + bad);
    if (n_channels < 1) return fail(D4W_ERR_ARG, "d4w_loc_associate: n_channels must be >= 1");
    if (!(fs > 0.0) || !(c0 > 0.0) || !(h > 0.0) || !(r > 0.0))
        return fail(D4W_ERR_ARG, "d4w_loc_associate: fs, c0, h and r must be > 0");
    if (min_picks < 1 || max_calls < 1) return fail(D4W_ERR_ARG, "d4w_loc_associate: min_picks and max_calls must be >= 1");
    if (!n_calls) return fail(D4W_ERR_ARG, "d4w_loc_associate: null pointer");
    *n_calls = 0;
    if (n_picks == 0) return D4W_OK;                   // no pick, no call (empty arrays may come with null pointers)
    if (!offsets || !samples || !cable_pos || !gx || !gy || !gz || !ws || !labels || !node || !t0 || !count)
        return fail(D4W_ERR_ARG, "d4w_loc_associate: null pointer");
    cudaStream_t st = (cudaStream_t)stream_v;
    AssocParams P{};
    P.off = offsets; P.s = samples; P.nch = n_channels; P.npicks = n_picks; P.fs = fs; P.pos = cable_pos; P.c0 = c0;
    P.gx = gx; P.gy = gy; P.gz = gz; P.nx = nx; P.ny = ny; P.nz = nz;
    P.nnodes = (long long)nx * ny * nz;
    P.ntiles = (int)assoc_tiles(P.nnodes);
    P.h = h; P.r = r; P.min_picks = min_picks;
    P.labels = labels;
    const AssocWs w = assoc_ws(ws, n_picks, P.ntiles);
    P.T = w.T;

    k_assoc_prep<<<1, kAssocPrepThreads, 0, st>>>(P, w.range);
    D4W_CHECK_LAUNCH("k_assoc_prep");
    AssocRange rg;
    D4W_CUDA_TRY(cudaMemcpyAsync(&rg, w.range, sizeof(rg), cudaMemcpyDeviceToHost, st));
    D4W_CUDA_TRY(cudaStreamSynchronize(st));
    if (rg.bad_offsets) return fail(D4W_ERR_ARG, "d4w_loc_associate: offsets must rise from 0 to n_picks");
    if (rg.smin < 0) return fail(D4W_ERR_ARG, "d4w_loc_associate: a pick has a negative sample");
    int nbins = 0;
    const int rc = d4w_loc_assoc_bins((double)rg.smin / fs, (double)rg.smax / fs, rg.box, c0, r, &P.jlo, &nbins);
    if (rc != D4W_OK) return rc;
    P.nbins = nbins;

    const size_t smem = assoc_vote_smem_bytes(nbins, kAssocThreads);
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_assoc_vote, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned assign_blocks = (unsigned)((n_channels + kAssocThreads - 1) / kAssocThreads);
    for (int k = 0; k < max_calls; ++k) {
        k_assoc_vote<<<(unsigned)P.ntiles, kAssocThreads, smem, st>>>(P, w.tiles);
        D4W_CHECK_LAUNCH("k_assoc_vote");
        k_assoc_pick<<<1, kAssocPickThreads, 0, st>>>(P, w.tiles, k, w.rec, node, t0, count);
        D4W_CHECK_LAUNCH("k_assoc_pick");
        AssocBest b;
        D4W_CUDA_TRY(cudaMemcpyAsync(&b, w.rec, sizeof(b), cudaMemcpyDeviceToHost, st));
        D4W_CUDA_TRY(cudaStreamSynchronize(st));
        if (b.bad) return fail(D4W_ERR_ARG, "d4w_loc_associate: an origin time fell outside the bin range (non-finite input?)");
        if (b.score < min_picks) break;
        k_assoc_assign<<<assign_blocks, kAssocThreads, 0, st>>>(P, w.rec, k);
        D4W_CHECK_LAUNCH("k_assoc_assign");
        *n_calls = k + 1;
    }
    return D4W_OK;
}
