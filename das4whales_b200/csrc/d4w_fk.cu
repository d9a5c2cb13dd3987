// d4w_fk.cu -- host side of the f-k filter: plans, mask descriptors, the five launches.
// C ABI declared in include/d4w.h; replaces dsp.fk_filter_filt / fk_filter_sparsefilt /
// taper_data and the device side of the mask design functions
// (/root/reference/src/das4whales/dsp.py:85-171, :308-454, :705-786).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cstdint>
#include <cuda.h>
#include "d4w_common.hpp"
#include "fk_hostplan.hpp"
#include "fk_kernels.cuh"

using namespace d4w;

namespace d4w {
std::string& last_error_ref() { static thread_local std::string e; return e; }
std::atomic<long long>& launch_counter() { static std::atomic<long long> c{0}; return c; }
}  // namespace d4w

extern "C" const char* d4w_last_error(void) { return last_error_ref().c_str(); }
extern "C" int d4w_version(void) { return 100; }
extern "C" long long d4w_launch_count(void) { return launch_counter().load(); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_tiled() {
    static PFN_encodeTiled fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
        else
            (void)cudaGetLastError();
    }
    return fn;
}

// 2-D fp32 tensor map over a [nx][ns] row-major matrix, box = 4 samples x 256 channels
static bool make_tile_map(CUtensorMap* map, const float* base, int nx, int ns) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)ns, (cuuint64_t)nx};
    const cuuint64_t strides[1] = {(cuuint64_t)ns * sizeof(float)};
    const cuuint32_t box[2] = {4, (cuuint32_t)kTmaBoxRows};
    const cuuint32_t estr[2] = {1, 1};
    // L2 promotion: one DRAM access brings a 128/256-byte line into L2, so the neighbouring tiles (other
    // SMs, microseconds later) hit in L2 instead of opening the same DRAM page again for 32 bytes
    static const int promo = env_int("D4W_TMA_L2PROMO", 3);
    const CUtensorMapL2promotion l2 = promo == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE
                                    : promo == 1 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
                                    : promo == 2 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                                 : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct d4w_fk_plan {
    int nx = 0, ns = 0, device = 0;
    int num_sms = 0;                          // cudaDeviceProp::multiProcessorCount
    int t1 = 1, t2 = 0;
    ColParams col{};
    RowParams row{};
    float2 *d_tw_col = nullptr, *d_tw_row = nullptr, *d_twT = nullptr;
    int *d_k2pos = nullptr, *d_pos2k = nullptr, *d_pos2k_row = nullptr;
    float* d_taper = nullptr;
    unsigned long long* d_dbg = nullptr;      // 8 phase-cycle counters (D4W_FK_DEBUG=1)
    // two-level column transform
    int two_level = 0;
    Col2Params col2{};
    float2* d_tw_x2 = nullptr;
    size_t colb_smem = 0;
    int colb_threads = 128;
    PipeParams pipe{};                        // pipe.nchunks > 0: single-launch pipelined level A+B
    int czt = 0;                              // chirp-z column kernels (nx with a prime factor > 61)
    CztParams cz{};
    float2 *d_czt_chirp = nullptr, *d_czt_bhat = nullptr;
    FkHostPlan hostplan;                     // kept for mask-time table building
    std::vector<int> h_k2pos;
    int col_threads = 256, row_threads = 256;
    size_t col_smem = 0, row_smem = 0;
};

struct d4w_fk_mask {
    d4w_fk_plan* plan = nullptr;
    int device = 0;
    MaskParams mp{};
    double* d_h = nullptr;
    int nact = 0;
    std::vector<int> act_k;
    int *d_act_k = nullptr, *d_k2slot = nullptr;
    int2* d_need = nullptr;
    int2* d_slot_pos = nullptr;
    int* d_plane_ptr = nullptr;
    Col2Entry* d_ents = nullptr;
    float* d_table = nullptr;      // caller-owned
};

extern "C" int d4w_fk_plan_create(d4w_fk_plan** out, int nx, int ns, int device) {
    if (!out) return fail(D4W_ERR_ARG, "d4w_fk_plan_create: null output pointer");
    *out = nullptr;
    if (nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_fk_plan_create: nx and ns must be >= 1");
    int ndev = 0;
    D4W_CUDA_TRY(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(D4W_ERR_ARG, "d4w_fk_plan_create: no such CUDA device");
    DeviceGuard guard(device);
    cudaDeviceProp prop;
    D4W_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    const size_t smem_cap = prop.sharedMemPerBlockOptin;
    const int num_sms = prop.multiProcessorCount;

    FkHostPlan hp;
    std::string err;
    if (build_fk_hostplan(nx, ns, smem_cap, hp, err)) return fail(D4W_ERR_UNSUPPORTED, err);
    auto pl = new d4w_fk_plan();
    pl->nx = nx; pl->ns = ns; pl->device = device; pl->num_sms = num_sms;
    pl->col.pl = hp.colpl; pl->col.nx = nx; pl->col.ns = ns; pl->col.nc = hp.nc; pl->col.nc_shift = hp.nc_shift;
    pl->col.fstride = hp.fstride; pl->col.aligned = hp.aligned;
    pl->col.tma = hp.tma;
    pl->col.dual = hp.dual; pl->col.npair = hp.npair; pl->col.npair_shift = hp.npair_shift; pl->col.aligned16 = hp.aligned16;
    pl->col_smem = hp.col_smem;
    pl->col_threads = std::min(1024, std::max(32, env_int("D4W_COL_THREADS", 512) / 32 * 32));
    if (hp.dual && hp.col_max_radix > 16) pl->col_threads = std::min(pl->col_threads, env_int("D4W_COL_THREADS_R25", 256));   // register budget of radix 20/25
    pl->t1 = hp.t1; pl->t2 = hp.t2;
    pl->row.pl = hp.rowpl; pl->row.t1 = hp.t1; pl->row.t2 = hp.t2; pl->row.dual = hp.row_dual;
    pl->row_smem = hp.row_smem;
    pl->row_threads = std::min(256, std::max(32, env_int("D4W_ROW_THREADS", 256)));
    const auto &twc = hp.tw_col, &twr = hp.tw_row, &twT = hp.twT;
    const auto &p2k = hp.pos2k, &k2p = hp.k2pos, &p2kr = hp.pos2k_row_tab;
    const auto& tap = hp.taper;
    pl->h_k2pos = hp.k2pos;
    pl->hostplan = hp;
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = upload(&pl->d_tw_col, twc);
    if (e == cudaSuccess) e = upload(&pl->d_tw_row, twr);
    if (e == cudaSuccess) e = upload(&pl->d_twT, twT);
    if (e == cudaSuccess) e = upload(&pl->d_pos2k, p2k);
    if (e == cudaSuccess) e = upload(&pl->d_k2pos, k2p);
    if (e == cudaSuccess) e = upload(&pl->d_pos2k_row, p2kr);
    if (e == cudaSuccess) e = upload(&pl->d_taper, tap);
    if (e == cudaSuccess && hp.two_level) e = upload(&pl->d_tw_x2, hp.tw_x2);
    if (e == cudaSuccess && hp.czt) e = upload(&pl->d_czt_chirp, hp.czt_chirp);
    if (e == cudaSuccess && hp.czt) e = upload(&pl->d_czt_bhat, hp.czt_bhat);
    if (e == cudaSuccess && hp.czt) e = cudaFuncSetAttribute(k_col_fwd_czt, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess && hp.czt) e = cudaFuncSetAttribute(k_col_inv_czt, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess && env_int("D4W_FK_DEBUG", 0)) { e = cudaMalloc((void**)&pl->d_dbg, 64); if (e == cudaSuccess) e = cudaMemset(pl->d_dbg, 0, 64); }
    // the attribute is per-kernel global state: always raise it to the device maximum, never to a plan's own size
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd_dual<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv_dual<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd_dual<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv_dual<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd_tma<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap - 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv_tma<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap - 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd_tma<416>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap - 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv_tma<416>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap - 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd_tma<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap - 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv_tma<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap - 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_fwd<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_col_inv<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid_dual, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    if (e != cudaSuccess) {
        std::string msg = std::string("d4w_fk_plan_create: ") + cudaGetErrorString(e);
        d4w_fk_plan_destroy(pl);
        return fail(D4W_ERR_CUDA, msg);
    }
    pl->col.tw = pl->d_tw_col; pl->col.k2pos = pl->d_k2pos; pl->col.pos2k = pl->d_pos2k;
    pl->row.tw = pl->d_tw_row; pl->row.twT = pl->d_twT;
    if (hp.czt) {
        pl->czt = 1;
        pl->col_threads = 512;
        CztParams& cz = pl->cz;
        cz.pl = hp.colpl; cz.tw = pl->d_tw_col; cz.chirp = pl->d_czt_chirp; cz.bhat = pl->d_czt_bhat;
        cz.nx = nx; cz.ns = ns; cz.m = hp.czt_m;
        cz.nc = hp.nc; cz.nc_shift = hp.nc_shift; cz.fstride = hp.fstride; cz.aligned = hp.aligned;
    }
    if (hp.two_level) {
        pl->two_level = 1; pl->colb_smem = hp.colb_smem;
        pl->col2.plb = hp.plb; pl->col2.twb = pl->d_tw_x2; pl->col2.twn = pl->d_tw_col;
        pl->col2.nx = nx; pl->col2.ns = ns; pl->col2.x1 = hp.x1; pl->col2.x2 = hp.x2; pl->col2.planes = hp.planes;
        pl->col2.np = hp.np2; pl->col2.fstride = hp.fstride2;
        pl->col2.np_shift = hp.np2 == 8 ? 3 : hp.np2 == 4 ? 2 : hp.np2 == 2 ? 1 : 0;
        pl->colb_threads = hp.colb_threads;
        pl->col2.vhp = hp.chunk_pairs; pl->col2.tpb = 0; pl->col2.tpn = hp.chunk_pairs;
        if (hp.pipe) {
            PipeParams& pp = pl->pipe;
            pp.nchunks = (ns / 2 + hp.chunk_pairs - 1) / hp.chunk_pairs;
            pp.lag = hp.pipe_lag; pp.nbuf = hp.pipe_lag + std::max(2, env_int("D4W_PIPE_SLACK", 2));
            pp.cq = hp.pipe_cq; pp.rpc = (hp.fused3 ? hp.colb_threads : 160) / hp.pipe_cq;
            pp.nA = (hp.x2 + pp.rpc - 1) / pp.rpc;
            pp.tiles = hp.chunk_pairs / hp.np2; pp.nB = hp.planes * pp.tiles;
            pp.hints = env_int("D4W_PIPE_HINTS", 1);
            pp.vbuf_elems = (size_t)hp.planes * hp.x2 * hp.chunk_pairs;
        }
        cudaFuncSetAttribute(k_colB_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
        cudaFuncSetAttribute(k_colB_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
    }
    *out = pl;
    return D4W_OK;
}

extern "C" int d4w_fk_plan_destroy(d4w_fk_plan* pl) {
    if (!pl) return D4W_OK;
    DeviceGuard guard(pl->device);
    cudaFree(pl->d_tw_col); cudaFree(pl->d_tw_row); cudaFree(pl->d_twT);
    cudaFree(pl->d_k2pos); cudaFree(pl->d_pos2k); cudaFree(pl->d_pos2k_row); cudaFree(pl->d_taper); cudaFree(pl->d_dbg); cudaFree(pl->d_tw_x2);
    cudaFree(pl->d_czt_chirp); cudaFree(pl->d_czt_bhat);
    delete pl;
    return D4W_OK;
}

extern "C" int d4w_fk_debug_phases(d4w_fk_plan* pl, unsigned long long* host8) {
    if (!pl || !host8) return fail(D4W_ERR_ARG, "d4w_fk_debug_phases: null argument");
    if (!pl->d_dbg) return fail(D4W_ERR_ARG, "d4w_fk_debug_phases: create the plan with D4W_FK_DEBUG=1");
    DeviceGuard guard(pl->device);
    D4W_CUDA_TRY(cudaMemcpy(host8, pl->d_dbg, 64, cudaMemcpyDeviceToHost));
    D4W_CUDA_TRY(cudaMemset(pl->d_dbg, 0, 64));
    return D4W_OK;
}

extern "C" int d4w_fk_plan_info(const d4w_fk_plan* pl, int* info) {
    if (!pl || !info) return fail(D4W_ERR_ARG, "d4w_fk_plan_info: null argument");
    info[0] = pl->t1; info[1] = pl->t2; info[2] = 2 * pl->col.nc; info[3] = pl->col.pl.nstages;
    info[4] = pl->row.pl.nstages; info[5] = pl->col_threads; info[6] = pl->row_threads;
    info[7] = pl->czt ? 4 : pl->pipe.nchunks ? 3 : pl->two_level ? 2 : pl->col.tma ? 1 : 0;
    return D4W_OK;
}

// ------------------------------------------------------------------------------- masks
// eps_arg < 0: exact pruning unless the environment variable D4W_MASK_EPS says otherwise
static int mask_finish_support(d4w_fk_mask* m, void* stream_v, double eps_arg = -1.0) {
    d4w_fk_plan* pl = m->plan;
    cudaStream_t stream = (cudaStream_t)stream_v;
    const int nrows = pl->nx / 2 + 1;
    unsigned int* d_rowmax = nullptr;
    D4W_CUDA_TRY(cudaMalloc((void**)&d_rowmax, nrows * sizeof(unsigned int)));
    cudaError_t e = cudaMemsetAsync(d_rowmax, 0, nrows * sizeof(unsigned int), stream);
    if (e == cudaSuccess) {
        const int fchunk = 8192;
        dim3 grid((pl->ns + fchunk - 1) / fchunk, nrows);
        k_mask_rowmax<<<grid, 256, 0, stream>>>(m->mp, d_rowmax, fchunk);
        e = cudaGetLastError();
        count_launch();
    }
    std::vector<unsigned int> rowmax((size_t)nrows);
    if (e == cudaSuccess) e = cudaMemcpyAsync(rowmax.data(), d_rowmax, nrows * sizeof(unsigned int), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    cudaFree(d_rowmax);
    if (e != cudaSuccess) return fail(D4W_ERR_CUDA, std::string("mask support scan: ") + cudaGetErrorString(e));
    // exact pruning by default; D4W_MASK_EPS > 0 additionally drops rows whose folded mask never exceeds eps
    const char* eps_s = std::getenv("D4W_MASK_EPS");
    const float eps = eps_arg >= 0.0 ? (float)eps_arg : (eps_s && *eps_s) ? (float)std::atof(eps_s) : 0.0f;
    cudaFree(m->d_act_k); cudaFree(m->d_k2slot); cudaFree(m->d_slot_pos); cudaFree(m->d_plane_ptr); cudaFree(m->d_ents); cudaFree(m->d_need);
    m->d_act_k = m->d_k2slot = nullptr; m->d_slot_pos = nullptr; m->d_plane_ptr = nullptr; m->d_ents = nullptr; m->d_need = nullptr;
    std::vector<int> k2slot((size_t)nrows, -1);
    m->act_k.clear();
    for (int k = 0; k < nrows; ++k) {
        float v; std::memcpy(&v, &rowmax[k], 4);
        if (v > eps) { k2slot[k] = (int)m->act_k.size(); m->act_k.push_back(k); }
    }
    m->nact = (int)m->act_k.size();
    D4W_CUDA_TRY(upload(&m->d_act_k, m->act_k));
    D4W_CUDA_TRY(upload(&m->d_k2slot, k2slot));
    std::vector<int2> slot_pos((size_t)m->nact);
    for (int sl = 0; sl < m->nact; ++sl) {
        const int k = m->act_k[sl];
        slot_pos[sl] = make_int2(pl->h_k2pos[k], pl->h_k2pos[k == 0 ? 0 : pl->nx - k]);
    }
    D4W_CUDA_TRY(upload(&m->d_slot_pos, slot_pos));
    if (pl->two_level) {
        std::vector<int> plane_ptr; std::vector<Col2EntryHost> ents;
        build_col2_entries(pl->hostplan, k2slot, plane_ptr, ents);
        static_assert(sizeof(Col2EntryHost) == sizeof(Col2Entry), "entry layout");
        std::vector<Col2Entry> dev((size_t)ents.size());
        for (size_t i = 0; i < ents.size(); ++i) dev[i] = Col2Entry{ents[i].pos, ents[i].slot, ents[i].flags, 0};
        D4W_CUDA_TRY(upload(&m->d_plane_ptr, plane_ptr));
        D4W_CUDA_TRY(upload(&m->d_ents, dev));
        if (pl->hostplan.fused_ra || pl->hostplan.fused3) {
            std::vector<int2> need;
            build_col2_need(pl->hostplan, k2slot, need);
            D4W_CUDA_TRY(upload(&m->d_need, need));
        }
    }
    return D4W_OK;
}

static int mask_create_common(d4w_fk_mask** out, d4w_fk_plan* plan, const MaskParams& mp, const double* host_h,
                              void* stream) {
    if (!out || !plan) return fail(D4W_ERR_ARG, "mask create: null argument");
    *out = nullptr;
    DeviceGuard guard(plan->device);
    auto m = new d4w_fk_mask();
    m->plan = plan; m->device = plan->device; m->mp = mp; m->mp.nx = plan->nx; m->mp.ns = plan->ns;
    if (host_h) {
        cudaError_t e = cudaMalloc((void**)&m->d_h, (size_t)plan->ns * sizeof(double));
        if (e == cudaSuccess) e = cudaMemcpy(m->d_h, host_h, (size_t)plan->ns * sizeof(double), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { d4w_fk_mask_destroy(m); return fail(D4W_ERR_CUDA, std::string("mask H upload: ") + cudaGetErrorString(e)); }
        m->mp.h = m->d_h;
    }
    int rc = mask_finish_support(m, stream);
    if (rc != D4W_OK) { d4w_fk_mask_destroy(m); return rc; }
    *out = m;
    return D4W_OK;
}

extern "C" int d4w_fk_mask_create_fan(d4w_fk_mask** out, d4w_fk_plan* plan, double kval, double fval, double cs_min,
                                      double cp_min, double cp_max, double cs_max) {
    MaskParams mp{};
    mp.kind = MASK_FAN; mp.kval = kval; mp.fval = fval;
    mp.c0 = cs_min; mp.c1 = cp_min; mp.c2 = cp_max; mp.c3 = cs_max;
    return mask_create_common(out, plan, mp, nullptr, nullptr);
}

extern "C" int d4w_fk_mask_create_hybrid_ninf(d4w_fk_mask** out, d4w_fk_plan* plan, double kval, double fval,
                                              double cs_min, double cp_min, double cp_max, double cs_max,
                                              const double* host_H, int col_lo, int col_hi) {
    if (!host_H) return fail(D4W_ERR_ARG, "hybrid mask: null H profile");
    MaskParams mp{};
    mp.kind = MASK_HYBRID_NINF; mp.kval = kval; mp.fval = fval;
    mp.c0 = cs_min; mp.c1 = cp_min; mp.c2 = cp_max; mp.c3 = cs_max;
    mp.col_lo = col_lo; mp.col_hi = col_hi;
    return mask_create_common(out, plan, mp, host_H, nullptr);
}

extern "C" int d4w_fk_mask_create_dense(d4w_fk_mask** out, d4w_fk_plan* plan, const float* dev_mask, void* stream) {
    if (!dev_mask) return fail(D4W_ERR_ARG, "dense mask: null device pointer");
    MaskParams mp{};
    mp.kind = MASK_DENSE; mp.dense = dev_mask;
    return mask_create_common(out, plan, mp, nullptr, stream);
}

extern "C" int d4w_fk_mask_destroy(d4w_fk_mask* m) {
    if (!m) return D4W_OK;
    DeviceGuard guard(m->device);
    cudaFree(m->d_h); cudaFree(m->d_act_k); cudaFree(m->d_k2slot); cudaFree(m->d_slot_pos); cudaFree(m->d_plane_ptr); cudaFree(m->d_ents); cudaFree(m->d_need);
    delete m;
    return D4W_OK;
}

extern "C" int d4w_fk_mask_prune(d4w_fk_mask* m, double eps, void* stream) {
    if (!m) return fail(D4W_ERR_ARG, "d4w_fk_mask_prune: null mask");
    if (!(eps >= 0.0)) return fail(D4W_ERR_ARG, "d4w_fk_mask_prune: eps must be >= 0");
    DeviceGuard guard(m->device);
    m->d_table = nullptr;                       // the transform-order table must be rebuilt for the new support
    return mask_finish_support(m, stream, eps);
}

extern "C" int d4w_fk_mask_rows(const d4w_fk_mask* m) { return m ? m->nact : 0; }

extern "C" size_t d4w_fk_mask_table_bytes(const d4w_fk_mask* m) {
    if (!m) return 0;
    return std::max<size_t>((size_t)m->nact * m->plan->ns * sizeof(float), 16);
}

extern "C" int d4w_fk_mask_build(d4w_fk_mask* m, float* dev_table, void* stream_v) {
    if (!m || !dev_table) return fail(D4W_ERR_ARG, "d4w_fk_mask_build: null argument");
    d4w_fk_plan* pl = m->plan;
    DeviceGuard guard(pl->device);
    cudaStream_t stream = (cudaStream_t)stream_v;
    m->d_table = dev_table;
    const size_t total = (size_t)m->nact * pl->ns;
    if (total == 0) return D4W_OK;
    const double scale = 1.0 / ((double)pl->nx * (double)pl->ns);
    const size_t blocks = (total + 255) / 256;
    if (blocks > 0x7fffffffull) return fail(D4W_ERR_UNSUPPORTED, "mask table too large for one launch");
    k_mask_build<<<(unsigned)blocks, 256, 0, stream>>>(m->mp, dev_table, m->d_act_k, pl->d_pos2k_row, pl->t1, pl->t2,
                                                      scale, total);
    D4W_CHECK_LAUNCH("k_mask_build");
    return D4W_OK;
}

extern "C" int d4w_fk_mask_materialize(const d4w_fk_mask* m, double* dev_out, void* stream_v) {
    if (!m || !dev_out) return fail(D4W_ERR_ARG, "d4w_fk_mask_materialize: null argument");
    DeviceGuard guard(m->plan->device);
    const size_t total = (size_t)m->plan->nx * m->plan->ns;
    const size_t blocks = (total + 255) / 256;
    if (blocks > 0x7fffffffull) return fail(D4W_ERR_UNSUPPORTED, "mask too large for one launch");
    k_mask_materialize<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream_v>>>(m->mp, dev_out, total);
    D4W_CHECK_LAUNCH("k_mask_materialize");
    return D4W_OK;
}

// ------------------------------------------------------------------------------- apply
extern "C" size_t d4w_fk_workspace_bytes(const d4w_fk_plan* pl, const d4w_fk_mask* m) {
    if (!pl || !m) return 0;
    size_t b = std::max<size_t>((size_t)m->nact * pl->ns * sizeof(float2), 16);
    b = (b + 255) / 256 * 256;
    if (pl->two_level) {
        const int nbuf = pl->pipe.nchunks ? pl->pipe.nbuf : 1;
        b += (size_t)nbuf * pl->col2.planes * pl->col2.x2 * pl->col2.vhp * sizeof(cpd);     // level-A/B intermediate V (chunk ring)
        if (pl->pipe.nchunks) b += (size_t)(2 * pl->pipe.nchunks + 1 + 63) / 64 * 64 * sizeof(unsigned);   // ticket + chunk counters
    }
    return b;
}

template <bool INV>
static int launch_row_split(const d4w_fk_plan* pl, float2* w, int nact, cudaStream_t stream) {
    const int threads = 128;
    dim3 grid((pl->t2 + threads - 1) / threads, nact);
    const size_t ldw = (size_t)pl->ns;
    switch (pl->t1) {
#define D4W_T1CASE(T) case T: k_row_split<T, INV><<<grid, threads, 0, stream>>>(w, ldw, pl->t2, pl->d_twT); break;
        D4W_T1CASE(2) D4W_T1CASE(3) D4W_T1CASE(4) D4W_T1CASE(5) D4W_T1CASE(6) D4W_T1CASE(8) D4W_T1CASE(10)
        D4W_T1CASE(12) D4W_T1CASE(15) D4W_T1CASE(16) D4W_T1CASE(20) D4W_T1CASE(25)
#undef D4W_T1CASE
        default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
    }
    D4W_CHECK_LAUNCH("k_row_split");
    return D4W_OK;
}

// Geometry `pl` may be a different plan than the mask's when a matrix is sharded over GPUs:
//  * passes 1 / 5 run on a time slab [nx][pl->ns] that starts at global sample t_offset (all kept rows);
//  * passes 2-4 run on `slot_count` kept rows starting at slot `slot_begin` (full time axis), `ws`
//    pointing at the first local row.
// fused two-stage level B: (ra, rb) in {16, 20, 25}^2
template <bool INV, typename V2>
static bool launch_colB_fused(const d4w_fk_plan* pl, const Col2Params& c2, const d4w_fk_mask* m, dim3 gb, V2 v2, float2* w, size_t ldw, cudaStream_t stream) {
    const int ra = pl->hostplan.fused_ra, rb = pl->hostplan.fused_rb;
    const size_t smem = (size_t)pl->col2.np * pl->col2.fstride * sizeof(cpd);
#define D4W_FUSED(RA, RB)                                                                                              \
    if (ra == RA && rb == RB) {                                                                                        \
        static bool attr_done_dev[64] = {};   /* opt in to > 48 KB dynamic shared memory once per instantiation and device */ \
        bool& attr_done = attr_done_dev[pl->device & 63];                                                              \
        if (!attr_done) {                                                                                              \
            if constexpr (!INV) cudaFuncSetAttribute(k_colB_fwd_fused<RA, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
            else cudaFuncSetAttribute(k_colB_inv_fused<RA, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);               \
            attr_done = true;                                                                                          \
        }                                                                                                              \
        if constexpr (!INV) k_colB_fwd_fused<RA, RB><<<gb, pl->colb_threads, smem, stream>>>(c2, v2, w, ldw, m->d_need); \
        else k_colB_inv_fused<RA, RB><<<gb, pl->colb_threads, smem, stream>>>(c2, v2, w, ldw, m->d_need);       \
        return true;                                                                                                   \
    }
    D4W_FUSED(16, 16) D4W_FUSED(16, 20) D4W_FUSED(16, 25) D4W_FUSED(20, 16) D4W_FUSED(20, 20) D4W_FUSED(20, 25)
    D4W_FUSED(25, 16) D4W_FUSED(25, 20) D4W_FUSED(25, 25)
#undef D4W_FUSED
    return false;
}

// single-launch pipelined level A + level B (forward: x -> kept rows W; inverse: W -> y)
template <bool INV>
static int launch_col2_pipe(const d4w_fk_plan* pl, const d4w_fk_mask* m, const float* x, float* y, cpd* v2, float2* w, size_t ldw,
                            const float* tap, cudaStream_t stream) {
    PipeParams pp = pl->pipe;
    pp.cnt = reinterpret_cast<unsigned*>(v2 + (size_t)pp.nbuf * pp.vbuf_elems);
    cudaError_t e = cudaMemsetAsync(pp.cnt, 0, (size_t)(2 * pp.nchunks + 1) * sizeof(unsigned), stream);
    if (e != cudaSuccess) return fail(D4W_ERR_CUDA, std::string("pipe counters: ") + cudaGetErrorString(e));
    const size_t smem = (size_t)pl->col2.np * pl->col2.fstride * sizeof(cpd);
    const unsigned grid = (unsigned)(pp.nchunks + pp.lag) * (unsigned)(pp.nA + pp.nB);
    const int ra = pl->hostplan.fused_ra, x1 = pl->col2.x1;
    bool done = false;
    if (pl->hostplan.fused3) {
        const int* r3 = pl->hostplan.r3;
        const int occ3 = env_int("D4W_PIPE3_OCC", 3);
#define D4W_PIPE3(R0, R1, R2, OCC)                                                                                        \
        if (!done && r3[0] == R0 && r3[1] == R1 && r3[2] == R2 && occ3 == OCC) {                                          \
            static bool attr_done_dev[64] = {};                                                                           \
            bool& attr_done = attr_done_dev[pl->device & 63];                                                             \
            if (!attr_done) { cudaFuncSetAttribute(k_col3_pipe<10, R0, R1, R2, INV, OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr_done = true; } \
            k_col3_pipe<10, R0, R1, R2, INV, OCC><<<grid, pl->colb_threads, smem, stream>>>(pl->col2, pp, x, y, v2, w, ldw, m->d_need, tap); \
            done = true;                                                                                                  \
        }
        D4W_PIPE3(10, 10, 10, 3) D4W_PIPE3(10, 10, 10, 4) D4W_PIPE3(10, 10, 10, 2) D4W_PIPE3(5, 5, 4, 3)
#undef D4W_PIPE3
        if (!done) return fail(D4W_ERR_UNSUPPORTED, "three-stage pipelined column kernel: unsupported split / occupancy");
        D4W_CHECK_LAUNCH("k_col3_pipe");
        return D4W_OK;
    }
    const int occ = env_int("D4W_PIPE_OCC", 3);       // CTAs per SM the kernel is compiled for: 3 = 128 registers (default), 4 = 96 (spills), 2 = 200
#define D4W_PIPE_OCC(X1, RA, RB, OCC)                                                                                     \
    if (!done && x1 == X1 && ra == RA && occ == OCC) {                                                                    \
        static bool attr_done_dev[64] = {};                                                                               \
        bool& attr_done = attr_done_dev[pl->device & 63];                                                                 \
        if (!attr_done) { cudaFuncSetAttribute(k_col2_pipe<X1, RA, RB, INV, OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr_done = true; } \
        k_col2_pipe<X1, RA, RB, INV, OCC><<<grid, 160, smem, stream>>>(pl->col2, pp, x, y, v2, w, ldw, m->d_need, tap);   \
        done = true;                                                                                                      \
    }
    D4W_PIPE_OCC(25, 20, 20, 4) D4W_PIPE_OCC(25, 20, 20, 2)
#define D4W_PIPE(X1, RA, RB)                                                                                              \
    if (!done && x1 == X1 && ra == RA) {                                                                                  \
        static bool attr_done_dev[64] = {};                                                                               \
        bool& attr_done = attr_done_dev[pl->device & 63];                                                                 \
        if (!attr_done) { cudaFuncSetAttribute(k_col2_pipe<X1, RA, RB, INV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr_done = true; } \
        k_col2_pipe<X1, RA, RB, INV><<<grid, 160, smem, stream>>>(pl->col2, pp, x, y, v2, w, ldw, m->d_need, tap);        \
        done = true;                                                                                                      \
    }
    D4W_PIPE(25, 20, 20) D4W_PIPE(25, 16, 25) D4W_PIPE(20, 20, 20) D4W_PIPE(20, 16, 25) D4W_PIPE(16, 20, 20) D4W_PIPE(16, 16, 25)
#undef D4W_PIPE_OCC
#undef D4W_PIPE
    if (!done) return fail(D4W_ERR_UNSUPPORTED, "pipelined column kernel: unsupported split");
    D4W_CHECK_LAUNCH("k_col2_pipe");
    return D4W_OK;
}

extern "C" int d4w_fk_apply_pass_ex(d4w_fk_plan* pl, d4w_fk_mask* m, const float* x, float* y, void* ws, int taper,
                                    int pass, int slot_begin, int slot_count, int t_offset, void* stream_v) {
    if (!pl || !m || !ws) return fail(D4W_ERR_ARG, "d4w_fk_apply: null argument");
    d4w_fk_plan* mp = m->plan;
    if (!m->d_table) return fail(D4W_ERR_ARG, "d4w_fk_apply: call d4w_fk_mask_build first");
    if (pl->device != mp->device) return fail(D4W_ERR_ARG, "d4w_fk_apply: plan and mask live on different devices");
    DeviceGuard guard(pl->device);
    cudaStream_t stream = (cudaStream_t)stream_v;
    float2* w = (float2*)ws;
    const size_t ldw = (size_t)pl->ns;
    const int nact = m->nact;
    if (pass == 1 || pass == 5) {
        if (pl->nx != mp->nx) return fail(D4W_ERR_ARG, "d4w_fk_apply: column passes need the mask's channel count");
        if (t_offset < 0 || (long long)t_offset + pl->ns > mp->ns) return fail(D4W_ERR_ARG, "d4w_fk_apply: time slab outside the mask's time axis");
    } else {
        if (pl->ns != mp->ns) return fail(D4W_ERR_ARG, "d4w_fk_apply: time passes need the mask's full time axis");
        if (slot_begin < 0 || slot_count < 0 || slot_begin + slot_count > nact) return fail(D4W_ERR_ARG, "d4w_fk_apply: bad slot range");
    }
    const int tile = pl->col.dual ? 4 * pl->col.npair : 2 * pl->col.nc;
    const int ntiles = (pl->ns + tile - 1) / tile;
    const float* tap = taper ? mp->d_taper + t_offset : nullptr;
    // the per-plane tables of the mask were built for its own plan; a time-slab plan of the same channel axis has the very
    // same two-level split (it depends on nx only), so the slab runs the two-level / pipelined kernels as well
    const bool same_split = pl == mp || (pl->nx == mp->nx && pl->two_level && mp->two_level && pl->col2.x1 == mp->col2.x1 &&
                                         pl->col2.x2 == mp->col2.x2 && pl->hostplan.fused_ra == mp->hostplan.fused_ra &&
                                         pl->hostplan.fused_rb == mp->hostplan.fused_rb && pl->hostplan.pos_x2 == mp->hostplan.pos_x2);
    const bool two = pl->two_level && same_split && m->d_ents && ((uintptr_t)ws % 16 == 0);
    cpd* v2 = nullptr;
    if (two) {
        size_t wb = std::max<size_t>((size_t)nact * pl->ns * sizeof(float2), 16);
        wb = (wb + 255) / 256 * 256;
        v2 = reinterpret_cast<cpd*>(reinterpret_cast<char*>(ws) + wb);
    }
    switch (pass) {
        case 1:
            if (!x) return fail(D4W_ERR_ARG, "d4w_fk_apply: null input");
            if (nact == 0) return D4W_OK;
            if (pl->czt || mp->czt) {
                if (!(pl->czt && mp->czt)) return fail(D4W_ERR_UNSUPPORTED, "d4w_fk_apply: chirp-z plan mixed with a mixed-radix plan");
                k_col_fwd_czt<<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->cz, x, w, ldw, m->d_slot_pos, nact, tap);
                D4W_CHECK_LAUNCH("k_col_fwd_czt");
                return D4W_OK;
            }
            if (two && ((uintptr_t)x % 16 == 0)) {
                if (pl->pipe.nchunks && m->d_need) return launch_col2_pipe<false>(pl, m, x, nullptr, v2, w, ldw, tap, stream);
                for (int tpb = 0; tpb < pl->ns / 2; tpb += pl->col2.vhp) {        // time chunks: V stays in L2 from A to B
                    Col2Params c2 = pl->col2;
                    c2.tpb = tpb; c2.tpn = std::min(c2.vhp, pl->ns / 2 - tpb);
                    dim3 ga((c2.tpn / 2 + 127) / 128, c2.x2);
                    switch (c2.x1) {
                        case 25: k_colA_fwd<25><<<ga, 128, 0, stream>>>(c2, x, v2, tap); break;
                        case 20: k_colA_fwd<20><<<ga, 128, 0, stream>>>(c2, x, v2, tap); break;
                        default: k_colA_fwd<16><<<ga, 128, 0, stream>>>(c2, x, v2, tap); break;
                    }
                    D4W_CHECK_LAUNCH("k_colA_fwd");
                    dim3 gb((c2.tpn + c2.np - 1) / c2.np, c2.planes);
                    if (!(m->d_need && launch_colB_fused<false>(pl, c2, m, gb, (const cpd*)v2, w, ldw, stream)))
                        k_colB_fwd<<<gb, pl->colb_threads, pl->colb_smem, stream>>>(c2, v2, w, ldw, m->d_plane_ptr, m->d_ents);
                    D4W_CHECK_LAUNCH("k_colB_fwd");
                }
                return D4W_OK;
            }
            if (pl->col.tma && ((uintptr_t)x % 16 == 0)) {
                CUtensorMap tm;
                if (make_tile_map(&tm, x, pl->nx, pl->ns)) {
                    const int grid = std::min(ntiles, pl->num_sms);
                    const int nbox = (pl->nx + kTmaBoxRows - 1) / kTmaBoxRows;
                    const int tma_boxes = std::min(nbox, std::max(0, nbox * env_int("D4W_TMA_LOAD_PCT", 100) / 100));
                    if (pl->col_threads <= 256)
                        k_col_fwd_tma<256><<<grid, pl->col_threads, pl->col_smem, stream>>>(tm, pl->col, x, w, ldw, m->d_slot_pos, nact, tap,
                                                                                            ntiles, tma_boxes, pl->d_dbg);
                    else if (pl->col_threads <= 416)
                        k_col_fwd_tma<416><<<grid, pl->col_threads, pl->col_smem, stream>>>(tm, pl->col, x, w, ldw, m->d_slot_pos, nact, tap,
                                                                                            ntiles, tma_boxes, pl->d_dbg);
                    else
                        k_col_fwd_tma<512><<<grid, std::min(pl->col_threads, 512), pl->col_smem, stream>>>(
                            tm, pl->col, x, w, ldw, m->d_slot_pos, nact, tap, ntiles, tma_boxes, pl->d_dbg);
                    D4W_CHECK_LAUNCH("k_col_fwd_tma");
                    return D4W_OK;
                }
            }
            if (pl->col.dual && pl->col_threads <= 256)
                k_col_fwd_dual<256><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, x, w, ldw, m->d_slot_pos, nact, tap);
            else if (pl->col.dual)
                k_col_fwd_dual<512><<<ntiles, std::min(pl->col_threads, 512), pl->col_smem, stream>>>(pl->col, x, w, ldw, m->d_slot_pos, nact, tap);
            else if (pl->col_threads <= 256)
                k_col_fwd<256><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, x, w, ldw, m->d_slot_pos, nact, tap);
            else if (pl->col_threads <= 512)
                k_col_fwd<512><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, x, w, ldw, m->d_slot_pos, nact, tap);
            else
                k_col_fwd<1024><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, x, w, ldw, m->d_slot_pos, nact, tap);
            D4W_CHECK_LAUNCH("k_col_fwd");
            return D4W_OK;
        case 2:
            if (pl->t1 == 1 || slot_count == 0) return D4W_OK;
            return launch_row_split<false>(pl, w, slot_count, stream);
        case 3: {
            if (slot_count == 0) return D4W_OK;
            if (pl->row.dual) {
                dim3 grid(pl->t1, (slot_count + 1) / 2);
                k_row_mid_dual<<<grid, env_int("D4W_ROW_DUAL_THREADS", 128), pl->row_smem, stream>>>(pl->row, w, ldw, m->d_table + (size_t)slot_begin * pl->ns,
                                                                    (size_t)pl->ns, slot_count);
                D4W_CHECK_LAUNCH("k_row_mid_dual");
                return D4W_OK;
            }
            dim3 grid(pl->t1, slot_count);
            if (pl->hostplan.row_fused)
                k_row_mid_fused<<<grid, pl->row_threads, pl->row_smem, stream>>>(pl->row, w, ldw, m->d_table + (size_t)slot_begin * pl->ns,
                                                                                 (size_t)pl->ns);
            else
                k_row_mid<<<grid, pl->row_threads, pl->row_smem, stream>>>(pl->row, w, ldw, m->d_table + (size_t)slot_begin * pl->ns,
                                                                           (size_t)pl->ns);
            D4W_CHECK_LAUNCH("k_row_mid");
            return D4W_OK;
        }
        case 4:
            if (pl->t1 == 1 || slot_count == 0) return D4W_OK;
            return launch_row_split<true>(pl, w, slot_count, stream);
        case 5:
            if (!y) return fail(D4W_ERR_ARG, "d4w_fk_apply: null output");
            if (pl->czt || mp->czt) {
                if (!(pl->czt && mp->czt)) return fail(D4W_ERR_UNSUPPORTED, "d4w_fk_apply: chirp-z plan mixed with a mixed-radix plan");
                k_col_inv_czt<<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->cz, w, ldw, m->d_slot_pos, nact, y);
                D4W_CHECK_LAUNCH("k_col_inv_czt");
                return D4W_OK;
            }
            if (two && ((uintptr_t)y % 16 == 0)) {
                if (pl->pipe.nchunks && m->d_need) return launch_col2_pipe<true>(pl, m, nullptr, y, v2, w, ldw, nullptr, stream);
                for (int tpb = 0; tpb < pl->ns / 2; tpb += pl->col2.vhp) {
                    Col2Params c2 = pl->col2;
                    c2.tpb = tpb; c2.tpn = std::min(c2.vhp, pl->ns / 2 - tpb);
                    dim3 gb((c2.tpn + c2.np - 1) / c2.np, c2.planes);
                    if (!(m->d_need && launch_colB_fused<true>(pl, c2, m, gb, (cpd*)v2, w, ldw, stream)))
                        k_colB_inv<<<gb, pl->colb_threads, pl->colb_smem, stream>>>(c2, v2, w, ldw, m->d_plane_ptr, m->d_ents);
                    D4W_CHECK_LAUNCH("k_colB_inv");
                    dim3 ga((c2.tpn / 2 + 127) / 128, c2.x2);
                    switch (c2.x1) {
                        case 25: k_colA_inv<25><<<ga, 128, 0, stream>>>(c2, v2, y); break;
                        case 20: k_colA_inv<20><<<ga, 128, 0, stream>>>(c2, v2, y); break;
                        default: k_colA_inv<16><<<ga, 128, 0, stream>>>(c2, v2, y); break;
                    }
                    D4W_CHECK_LAUNCH("k_colA_inv");
                }
                return D4W_OK;
            }
            if (pl->col.tma && ((uintptr_t)y % 16 == 0)) {
                CUtensorMap tm;
                if (make_tile_map(&tm, y, pl->nx, pl->ns)) {
                    const int grid = std::min(ntiles, pl->num_sms);
                    const int nbox = (pl->nx + kTmaBoxRows - 1) / kTmaBoxRows;
                    const int tma_boxes = std::min(nbox, std::max(0, nbox * env_int("D4W_TMA_STORE_PCT", 100) / 100));
                    if (pl->col_threads <= 256)
                        k_col_inv_tma<256><<<grid, pl->col_threads, pl->col_smem, stream>>>(tm, pl->col, w, ldw, m->d_slot_pos, nact, ntiles, y,
                                                                                            tma_boxes, pl->d_dbg);
                    else if (pl->col_threads <= 416)
                        k_col_inv_tma<416><<<grid, pl->col_threads, pl->col_smem, stream>>>(tm, pl->col, w, ldw, m->d_slot_pos, nact, ntiles, y,
                                                                                            tma_boxes, pl->d_dbg);
                    else
                        k_col_inv_tma<512><<<grid, std::min(pl->col_threads, 512), pl->col_smem, stream>>>(
                            tm, pl->col, w, ldw, m->d_slot_pos, nact, ntiles, y, tma_boxes, pl->d_dbg);
                    D4W_CHECK_LAUNCH("k_col_inv_tma");
                    return D4W_OK;
                }
            }
            if (pl->col.dual && pl->col_threads <= 256)
                k_col_inv_dual<256><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, w, ldw, m->d_slot_pos, nact, y);
            else if (pl->col.dual)
                k_col_inv_dual<512><<<ntiles, std::min(pl->col_threads, 512), pl->col_smem, stream>>>(pl->col, w, ldw, m->d_slot_pos, nact, y);
            else if (pl->col_threads <= 256)
                k_col_inv<256><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, w, ldw, m->d_slot_pos, nact, y);
            else if (pl->col_threads <= 512)
                k_col_inv<512><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, w, ldw, m->d_slot_pos, nact, y);
            else
                k_col_inv<1024><<<ntiles, pl->col_threads, pl->col_smem, stream>>>(pl->col, w, ldw, m->d_slot_pos, nact, y);
            D4W_CHECK_LAUNCH("k_col_inv");
            return D4W_OK;
        default:
            return fail(D4W_ERR_ARG, "d4w_fk_apply_pass: pass must be 1..5");
    }
}

extern "C" int d4w_fk_apply_pass(d4w_fk_plan* pl, d4w_fk_mask* m, const float* x, float* y, void* ws, int taper,
                                 int pass, void* stream) {
    if (!pl || !m) return fail(D4W_ERR_ARG, "d4w_fk_apply: null argument");
    if (m->plan != pl) return fail(D4W_ERR_ARG, "d4w_fk_apply: mask was built for a different plan");
    return d4w_fk_apply_pass_ex(pl, m, x, y, ws, taper, pass, 0, m->nact, 0, stream);
}

extern "C" int d4w_fk_apply(d4w_fk_plan* pl, d4w_fk_mask* m, const float* x, float* y, void* ws, int taper,
                            void* stream) {
    for (int pass = 1; pass <= 5; ++pass) {
        int rc = d4w_fk_apply_pass(pl, m, x, y, ws, taper, pass, stream);
        if (rc != D4W_OK) return rc;
    }
    return D4W_OK;
}
