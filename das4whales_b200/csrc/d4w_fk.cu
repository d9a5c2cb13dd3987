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
#include "fk_spectrum.cuh"

using namespace d4w;

namespace d4w {
std::string& last_error_ref() { static thread_local std::string e; return e; }
std::atomic<long long>& launch_counter() { static std::atomic<long long> c{0}; return c; }
// mask-bank kernels (d4w_fk_bank.cu)
int launch_row_mid_oop(bool dual, bool fused, dim3 grid, int threads, size_t smem, const RowParams& rp, float2* w, size_t ldw,
                       const float* tab, size_t tab_slot_stride, int nslots, float2* dst, int device, cudaStream_t stream);
int launch_bank_gather(const float* src, float* dst, const int* src_row, int ns, size_t total, cudaStream_t stream);
// f-k spectrum power pass (d4w_fk_spectrum.cu)
int launch_fk_power(dim3 grid, int threads, size_t smem, const RowParams& rp, const SpecParams& sp, const float2* w, size_t ldw,
                    float* out, int device, cudaStream_t stream);
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
            // three ring slots beyond the lag (5 chunks, 33 MB of V at 10 000 channels, still inside the 50 MB L2): a producer
            // waits less often for the consumers of the slot it re-uses; measured on the H100 against two, P1 5.08 -> 4.97 ms
            pp.lag = hp.pipe_lag; pp.nbuf = hp.pipe_lag + std::max(2, env_int("D4W_PIPE_SLACK", 3));
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
static int build_support_tables(d4w_fk_mask* m, const std::vector<int>& act_k);

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
    std::vector<int> act_k;
    for (int k = 0; k < nrows; ++k) {
        float v; std::memcpy(&v, &rowmax[k], 4);
        if (v > eps) act_k.push_back(k);
    }
    return build_support_tables(m, act_k);
}

// Per-slot column tables for the kept wavenumber rows act_k (ascending, in [0, nx/2]): slot positions, the two-level
// plane entries and need tables.  Used for a mask's own support and for the union support of a mask bank.
static int build_support_tables(d4w_fk_mask* m, const std::vector<int>& act_k) {
    d4w_fk_plan* pl = m->plan;
    const int nrows = pl->nx / 2 + 1;
    cudaFree(m->d_act_k); cudaFree(m->d_k2slot); cudaFree(m->d_slot_pos); cudaFree(m->d_plane_ptr); cudaFree(m->d_ents); cudaFree(m->d_need);
    m->d_act_k = m->d_k2slot = nullptr; m->d_slot_pos = nullptr; m->d_plane_ptr = nullptr; m->d_ents = nullptr; m->d_need = nullptr;
    std::vector<int> k2slot((size_t)nrows, -1);
    m->act_k = act_k;
    for (size_t sl = 0; sl < act_k.size(); ++sl) k2slot[act_k[sl]] = (int)sl;
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
// bytes of one block of kept rows W (|support| x ns complex samples), rounded up so that what follows stays aligned
static size_t kept_rows_bytes(const d4w_fk_plan* pl, int nact) {
    const size_t b = std::max<size_t>((size_t)nact * pl->ns * sizeof(float2), 16);
    return (b + 255) / 256 * 256;
}

// bytes of the level-A/B intermediate V of a two-level plan (chunk ring and its counters), 0 for other plans
static size_t col2_ring_bytes(const d4w_fk_plan* pl) {
    if (!pl->two_level) return 0;
    const int nbuf = pl->pipe.nchunks ? pl->pipe.nbuf : 1;
    size_t b = (size_t)nbuf * pl->col2.planes * pl->col2.x2 * pl->col2.vhp * sizeof(cpd);     // level-A/B intermediate V (chunk ring)
    if (pl->pipe.nchunks) b += (size_t)(2 * pl->pipe.nchunks + 1 + 63) / 64 * 64 * sizeof(unsigned);   // ticket + chunk counters
    return b;
}

extern "C" size_t d4w_fk_workspace_bytes(const d4w_fk_plan* pl, const d4w_fk_mask* m) {
    if (!pl || !m) return 0;
    return kept_rows_bytes(pl, m->nact) + col2_ring_bytes(pl);
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
    // CTAs per SM the kernel is compiled for: 3 = 128 registers, 4 = 96 (spills), 2 = 200.  Only 25 x (20 x 20) is built at
    // 2 and 4; other splits run at 3.  The forward 25 x (20 x 20) kernel runs at 2: capped at 128 registers it spills, at 2
    // CTAs/SM it takes 158 and none, and P1 at 10 000 x 120 000 fell from 5.50 to 5.08 ms on the H100.  The inverse takes
    // 128 registers either way and runs at 3 (4.40 ms at both)
    const int occ = env_int("D4W_PIPE_OCC", INV ? 3 : 2);
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

// The column kernels move whole rows of x and y with 16-byte accesses when ns % 4 == 0 (cp.async, TMA tiles, the two-level
// kernels) and 8-byte ones when ns is even, so a matrix must start on that boundary.  Checked before any launch: a
// misaligned base would otherwise fault inside a kernel.
static int check_matrix_alignment(const float* p, int ns, const char* what) {
    const uintptr_t align = ns % 4 == 0 ? 16 : ns % 2 == 0 ? 8 : sizeof(float);
    if (p && (uintptr_t)p % align)
        return fail(D4W_ERR_ARG, std::string(what) + " must be " + std::to_string(align) + "-byte aligned for " + std::to_string(ns) +
                                     " samples per row");
    return D4W_OK;
}

// One pass on explicit buffers, arguments already checked (x and y aligned as check_matrix_alignment requires).
// w: the kept rows of m's support; v2: the two-level intermediate (nullptr: the single-level column kernels); tab: P3's table for the `slot_count` rows at w; w3: P3's
// destination (nullptr: in place, the single-mask filter; otherwise a second kept-row block of the same layout).
static int fk_run_pass(const d4w_fk_plan* pl, const d4w_fk_mask* m, const float* x, float* y, float2* w, cpd* v2,
                       const float* tab, float2* w3, const float* tap, int pass, int slot_count, cudaStream_t stream) {
    const d4w_fk_plan* mp = m->plan;
    const size_t ldw = (size_t)pl->ns;
    const int nact = m->nact;
    const int tile = pl->col.dual ? 4 * pl->col.npair : 2 * pl->col.nc;
    const int ntiles = (pl->ns + tile - 1) / tile;
    const bool two = v2 != nullptr;
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
            if (two) {
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
            if (pl->col.tma) {
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
                const int threads = env_int("D4W_ROW_DUAL_THREADS", 128);
                if (w3) return launch_row_mid_oop(true, false, grid, threads, pl->row_smem, pl->row, w, ldw, tab, (size_t)pl->ns,
                                                  slot_count, w3, pl->device, stream);
                k_row_mid_dual<<<grid, threads, pl->row_smem, stream>>>(pl->row, w, ldw, tab, (size_t)pl->ns, slot_count);
                D4W_CHECK_LAUNCH("k_row_mid_dual");
                return D4W_OK;
            }
            dim3 grid(pl->t1, slot_count);
            if (w3) return launch_row_mid_oop(false, pl->hostplan.row_fused, grid, pl->row_threads, pl->row_smem, pl->row, w, ldw,
                                              tab, (size_t)pl->ns, slot_count, w3, pl->device, stream);
            if (pl->hostplan.row_fused)
                return launch_row_mid_fused(grid, pl->row_threads, pl->row_smem, pl->row, w, ldw, tab, (size_t)pl->ns, nullptr,
                                            pl->device, stream);
            k_row_mid<<<grid, pl->row_threads, pl->row_smem, stream>>>(pl->row, w, ldw, tab, (size_t)pl->ns);
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
            if (two) {
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
            if (pl->col.tma) {
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

// the two-level kernels need their per-plane tables built for this channel split, and a 16-byte aligned workspace
static bool use_two_level(const d4w_fk_plan* pl, const d4w_fk_mask* m, const void* ws) {
    const d4w_fk_plan* mp = m->plan;
    // the per-plane tables of the mask were built for its own plan; a time-slab plan of the same channel axis has the very
    // same two-level split (it depends on nx only), so the slab runs the two-level / pipelined kernels as well
    const bool same_split = pl == mp || (pl->nx == mp->nx && pl->two_level && mp->two_level && pl->col2.x1 == mp->col2.x1 &&
                                         pl->col2.x2 == mp->col2.x2 && pl->hostplan.fused_ra == mp->hostplan.fused_ra &&
                                         pl->hostplan.fused_rb == mp->hostplan.fused_rb && pl->hostplan.pos_x2 == mp->hostplan.pos_x2);
    return pl->two_level && same_split && m->d_ents && ((uintptr_t)ws % 16 == 0);
}

extern "C" int d4w_fk_apply_pass_ex(d4w_fk_plan* pl, d4w_fk_mask* m, const float* x, float* y, void* ws, int taper,
                                    int pass, int slot_begin, int slot_count, int t_offset, void* stream_v) {
    if (!pl || !m || !ws) return fail(D4W_ERR_ARG, "d4w_fk_apply: null argument");
    d4w_fk_plan* mp = m->plan;
    if (!m->d_table) return fail(D4W_ERR_ARG, "d4w_fk_apply: call d4w_fk_mask_build first");
    if (pl->device != mp->device) return fail(D4W_ERR_ARG, "d4w_fk_apply: plan and mask live on different devices");
    DeviceGuard guard(pl->device);
    if (pass == 1 || pass == 5) {
        if (pl->nx != mp->nx) return fail(D4W_ERR_ARG, "d4w_fk_apply: column passes need the mask's channel count");
        if (t_offset < 0 || (long long)t_offset + pl->ns > mp->ns) return fail(D4W_ERR_ARG, "d4w_fk_apply: time slab outside the mask's time axis");
    } else {
        if (pl->ns != mp->ns) return fail(D4W_ERR_ARG, "d4w_fk_apply: time passes need the mask's full time axis");
        if (slot_begin < 0 || slot_count < 0 || slot_begin + slot_count > m->nact) return fail(D4W_ERR_ARG, "d4w_fk_apply: bad slot range");
    }
    if (pass == 1 && check_matrix_alignment(x, pl->ns, "d4w_fk_apply: input") != D4W_OK) return D4W_ERR_ARG;
    if (pass == 5 && check_matrix_alignment(y, pl->ns, "d4w_fk_apply: output") != D4W_OK) return D4W_ERR_ARG;
    const float* tap = taper ? mp->d_taper + t_offset : nullptr;
    cpd* v2 = use_two_level(pl, m, ws) ? reinterpret_cast<cpd*>(reinterpret_cast<char*>(ws) + kept_rows_bytes(pl, m->nact)) : nullptr;
    return fk_run_pass(pl, m, x, y, (float2*)ws, v2, m->d_table + (size_t)slot_begin * pl->ns, nullptr, tap, pass, slot_count,
                       (cudaStream_t)stream_v);
}

extern "C" int d4w_fk_apply_pass(d4w_fk_plan* pl, d4w_fk_mask* m, const float* x, float* y, void* ws, int taper,
                                 int pass, void* stream) {
    if (!pl || !m) return fail(D4W_ERR_ARG, "d4w_fk_apply: null argument");
    if (m->plan != pl) return fail(D4W_ERR_ARG, "d4w_fk_apply: mask was built for a different plan");
    return d4w_fk_apply_pass_ex(pl, m, x, y, ws, taper, pass, 0, m->nact, 0, stream);
}

extern "C" int d4w_fk_apply(d4w_fk_plan* pl, d4w_fk_mask* m, const float* x, float* y, void* ws, int taper,
                            void* stream) {
    if (pl && (check_matrix_alignment(x, pl->ns, "d4w_fk_apply: input") != D4W_OK ||
               check_matrix_alignment(y, pl->ns, "d4w_fk_apply: output") != D4W_OK)) return D4W_ERR_ARG;   // before P1 runs
    for (int pass = 1; pass <= 5; ++pass) {
        int rc = d4w_fk_apply_pass(pl, m, x, y, ws, taper, pass, stream);
        if (rc != D4W_OK) return rc;
    }
    return D4W_OK;
}

// ------------------------------------------------------------------------------- mask banks
// Several masks over one plan and one forward transform (scripts/main_fkcomp.py:66-95 filters the same band-passed
// matrix with four masks).  The bank's slots are the union U of the masks' kept rows in ascending wavenumber order,
// so P1, P2 and P4 and the kept-row layout are those of a mask with support U.  Each mask gets a [|U|][ns] table
// holding its own table's rows at its own slots and exact zeros elsewhere, which keeps a mask's arithmetic on every
// row it keeps and leaves the rows it drops at zero.
struct d4w_fk_bank {
    d4w_fk_plan* plan = nullptr;
    std::vector<d4w_fk_mask*> masks;
    std::vector<std::vector<int>> supports;   // each mask's kept rows when the bank was made
    d4w_fk_mask* sup = nullptr;               // the union support: its slot and column tables (no mask table)
    int* d_src_row = nullptr;                 // [nmasks][|U|]: row of mask i's own table for slot u, -1 where it keeps none
    float* d_table = nullptr;                 // caller-owned [nmasks][|U|][ns], set by d4w_fk_bank_build
};

extern "C" int d4w_fk_bank_destroy(d4w_fk_bank* b) {
    if (!b) return D4W_OK;
    DeviceGuard guard(b->plan->device);
    d4w_fk_mask_destroy(b->sup);
    cudaFree(b->d_src_row);
    delete b;
    return D4W_OK;
}

extern "C" int d4w_fk_bank_create(d4w_fk_bank** out, d4w_fk_plan* plan, d4w_fk_mask* const* masks, int nmasks) {
    if (!out) return fail(D4W_ERR_ARG, "d4w_fk_bank_create: null output pointer");
    *out = nullptr;
    if (!plan || !masks) return fail(D4W_ERR_ARG, "d4w_fk_bank_create: null argument");
    if (nmasks < 1) return fail(D4W_ERR_ARG, "d4w_fk_bank_create: a bank needs at least one mask");
    for (int i = 0; i < nmasks; ++i) {
        if (!masks[i]) return fail(D4W_ERR_ARG, "d4w_fk_bank_create: null mask " + std::to_string(i));
        if (masks[i]->plan != plan) return fail(D4W_ERR_ARG, "d4w_fk_bank_create: mask " + std::to_string(i) + " was built for another plan");
    }
    DeviceGuard guard(plan->device);
    const int nrows = plan->nx / 2 + 1;
    std::vector<char> kept((size_t)nrows, 0);
    for (int i = 0; i < nmasks; ++i)
        for (int k : masks[i]->act_k) kept[k] = 1;
    std::vector<int> uni;
    for (int k = 0; k < nrows; ++k)
        if (kept[k]) uni.push_back(k);
    auto b = new d4w_fk_bank();
    b->plan = plan;
    b->masks.assign(masks, masks + nmasks);
    b->sup = new d4w_fk_mask();
    b->sup->plan = plan; b->sup->device = plan->device;
    int rc = build_support_tables(b->sup, uni);
    if (rc != D4W_OK) { d4w_fk_bank_destroy(b); return rc; }
    const size_t nu = uni.size();
    std::vector<int> src_row((size_t)nmasks * nu, -1);
    for (int i = 0; i < nmasks; ++i) {
        const std::vector<int>& s = masks[i]->act_k;
        b->supports.push_back(s);
        size_t j = 0;                                   // both lists ascend, and s is a subset of uni
        for (size_t u = 0; u < nu && j < s.size(); ++u)
            if (uni[u] == s[j]) src_row[(size_t)i * nu + u] = (int)j++;
    }
    cudaError_t e = upload(&b->d_src_row, src_row);
    if (e != cudaSuccess) { d4w_fk_bank_destroy(b); return fail(D4W_ERR_CUDA, std::string("bank row map: ") + cudaGetErrorString(e)); }
    *out = b;
    return D4W_OK;
}

extern "C" int d4w_fk_bank_rows(const d4w_fk_bank* b) { return b ? b->sup->nact : 0; }

extern "C" size_t d4w_fk_bank_table_bytes(const d4w_fk_bank* b) {
    if (!b) return 0;
    return std::max<size_t>(b->masks.size() * (size_t)b->sup->nact * b->plan->ns * sizeof(float), 16);
}

extern "C" int d4w_fk_bank_build(d4w_fk_bank* b, float* dev_table, void* stream_v) {
    if (!b || !dev_table) return fail(D4W_ERR_ARG, "d4w_fk_bank_build: null argument");
    DeviceGuard guard(b->plan->device);
    cudaStream_t stream = (cudaStream_t)stream_v;
    for (size_t i = 0; i < b->masks.size(); ++i) {
        const d4w_fk_mask* m = b->masks[i];
        if (m->act_k != b->supports[i])
            return fail(D4W_ERR_ARG, "d4w_fk_bank_build: mask " + std::to_string(i) + " was pruned again after the bank was made");
        if (!m->d_table) return fail(D4W_ERR_ARG, "d4w_fk_bank_build: call d4w_fk_mask_build on mask " + std::to_string(i) + " first");
    }
    const int nu = b->sup->nact, ns = b->plan->ns;
    const size_t total = (size_t)nu * ns;
    for (size_t i = 0; i < b->masks.size() && total; ++i) {
        const int rc = launch_bank_gather(b->masks[i]->d_table, dev_table + i * total, b->d_src_row + i * nu, ns, total, stream);
        if (rc != D4W_OK) return rc;
    }
    b->d_table = dev_table;
    return D4W_OK;
}

extern "C" size_t d4w_fk_bank_workspace_bytes(const d4w_fk_plan* pl, const d4w_fk_bank* b) {
    if (!pl || !b) return 0;
    return 2 * kept_rows_bytes(pl, b->sup->nact) + col2_ring_bytes(pl);
}

extern "C" int d4w_fk_bank_apply_pass(d4w_fk_plan* pl, d4w_fk_bank* b, const float* x, float* const* ys, void* ws, int taper,
                                      int pass, int mask, void* stream_v) {
    if (!pl || !b || !ys || !ws) return fail(D4W_ERR_ARG, "d4w_fk_bank_apply: null argument");
    if (b->plan != pl) return fail(D4W_ERR_ARG, "d4w_fk_bank_apply: bank was built for a different plan");
    if (!b->d_table) return fail(D4W_ERR_ARG, "d4w_fk_bank_apply: call d4w_fk_bank_build first");
    const int nm = (int)b->masks.size();
    if (pass >= 3 && (mask < 0 || mask >= nm)) return fail(D4W_ERR_ARG, "d4w_fk_bank_apply: mask index out of range");
    // each output is written by its own P5 while the other masks still run, so no two outputs may overlap; an output
    // may alias x, which is last read in P1
    const size_t bytes = (size_t)pl->nx * pl->ns * sizeof(float);
    for (int i = 0; i < nm; ++i) {
        if (!ys[i]) return fail(D4W_ERR_ARG, "d4w_fk_bank_apply: null output " + std::to_string(i));
        if (check_matrix_alignment(ys[i], pl->ns, ("d4w_fk_bank_apply: output " + std::to_string(i)).c_str()) != D4W_OK) return D4W_ERR_ARG;
        for (int j = 0; j < i; ++j) {
            const char *a = (const char*)ys[i], *c = (const char*)ys[j];
            if (a < c + bytes && c < a + bytes) return fail(D4W_ERR_ARG, "d4w_fk_bank_apply: outputs " + std::to_string(j) + " and " + std::to_string(i) + " overlap");
        }
    }
    if (pass == 1 && check_matrix_alignment(x, pl->ns, "d4w_fk_bank_apply: input") != D4W_OK) return D4W_ERR_ARG;
    DeviceGuard guard(pl->device);
    const d4w_fk_mask* sup = b->sup;
    const int nu = sup->nact;
    float2* w = (float2*)ws;                                                          // W: the forward transform
    float2* w3 = (float2*)((char*)ws + kept_rows_bytes(pl, nu));                      // W': one mask's filtered rows
    cpd* v2 = use_two_level(pl, sup, ws) ? reinterpret_cast<cpd*>((char*)ws + 2 * kept_rows_bytes(pl, nu)) : nullptr;
    cudaStream_t stream = (cudaStream_t)stream_v;
    switch (pass) {
        case 1: return fk_run_pass(pl, sup, x, nullptr, w, v2, nullptr, nullptr, taper ? pl->d_taper : nullptr, 1, nu, stream);
        case 2: return fk_run_pass(pl, sup, nullptr, nullptr, w, v2, nullptr, nullptr, nullptr, 2, nu, stream);
        case 3: return fk_run_pass(pl, sup, nullptr, nullptr, w, v2, b->d_table + (size_t)mask * nu * pl->ns, w3, nullptr, 3, nu, stream);
        case 4: return fk_run_pass(pl, sup, nullptr, nullptr, w3, v2, nullptr, nullptr, nullptr, 4, nu, stream);
        case 5: return fk_run_pass(pl, sup, nullptr, ys[mask], w3, v2, nullptr, nullptr, nullptr, 5, nu, stream);
        default: return fail(D4W_ERR_ARG, "d4w_fk_bank_apply_pass: pass must be 1..5");
    }
}

extern "C" int d4w_fk_bank_apply(d4w_fk_plan* pl, d4w_fk_bank* b, const float* x, float* const* ys, void* ws, int taper,
                                 void* stream) {
    int rc = d4w_fk_bank_apply_pass(pl, b, x, ys, ws, taper, 1, 0, stream);
    if (rc == D4W_OK) rc = d4w_fk_bank_apply_pass(pl, b, x, ys, ws, taper, 2, 0, stream);
    for (int i = 0; rc == D4W_OK && b && i < (int)b->masks.size(); ++i)
        for (int pass = 3; rc == D4W_OK && pass <= 5; ++pass) rc = d4w_fk_bank_apply_pass(pl, b, x, ys, ws, taper, pass, i, stream);
    return rc;
}

// ------------------------------------------------------------------------------- f-k power spectrum
// |fftshift(fft2(x))|^2 over a band of the shifted plane: P1 and P2 of the filter on the band's half-plane rows, then the
// forward-only power pass (fk_spectrum.cuh) in place of P3's mask multiply and inverse; no P4 or P5.  The rows are the
// k' in [0, nx/2] with +k' or -k' inside the band, kept in a support object (slot and column tables, no mask table) as
// a mask bank keeps its union support.
struct d4w_fk_spectrum {
    d4w_fk_plan* plan = nullptr;
    d4w_fk_mask* sup = nullptr;
    int k_lo = 0, k_hi = 0, f_lo = 0, f_hi = 0;
    int* d_k2pos_row = nullptr;               // natural T2-point frequency -> position after the forward stages
};

extern "C" int d4w_fk_spectrum_destroy(d4w_fk_spectrum* s) {
    if (!s) return D4W_OK;
    DeviceGuard guard(s->plan->device);
    d4w_fk_mask_destroy(s->sup);
    cudaFree(s->d_k2pos_row);
    delete s;
    return D4W_OK;
}

extern "C" int d4w_fk_spectrum_create(d4w_fk_spectrum** out, d4w_fk_plan* plan, int k_lo, int k_hi, int f_lo, int f_hi) {
    if (!out) return fail(D4W_ERR_ARG, "d4w_fk_spectrum_create: null output pointer");
    *out = nullptr;
    if (!plan) return fail(D4W_ERR_ARG, "d4w_fk_spectrum_create: null plan");
    const int nx = plan->nx, ns = plan->ns;
    if (k_lo < 0 || k_hi > nx || k_lo >= k_hi)
        return fail(D4W_ERR_ARG, "d4w_fk_spectrum_create: wavenumber rows [" + std::to_string(k_lo) + ", " + std::to_string(k_hi) +
                                     ") empty or outside [0, " + std::to_string(nx) + ")");
    if (f_lo < 0 || f_hi > ns || f_lo >= f_hi)
        return fail(D4W_ERR_ARG, "d4w_fk_spectrum_create: frequency columns [" + std::to_string(f_lo) + ", " + std::to_string(f_hi) +
                                     ") empty or outside [0, " + std::to_string(ns) + ")");
    DeviceGuard guard(plan->device);
    std::vector<int> rows;
    for (int k = 0; k <= nx / 2; ++k) {
        const int rp = (k + nx / 2) % nx, rn = (nx - k + nx / 2) % nx;
        if ((rp >= k_lo && rp < k_hi) || (rn >= k_lo && rn < k_hi)) rows.push_back(k);
    }
    const std::vector<int>& p2k = plan->hostplan.pos2k_row;
    std::vector<int> k2p(p2k.size());
    for (size_t p = 0; p < p2k.size(); ++p) k2p[p2k[p]] = (int)p;
    auto s = new d4w_fk_spectrum();
    s->plan = plan; s->k_lo = k_lo; s->k_hi = k_hi; s->f_lo = f_lo; s->f_hi = f_hi;
    s->sup = new d4w_fk_mask();
    s->sup->plan = plan; s->sup->device = plan->device;
    int rc = build_support_tables(s->sup, rows);
    if (rc == D4W_OK) {
        cudaError_t e = upload(&s->d_k2pos_row, k2p);
        if (e != cudaSuccess) rc = fail(D4W_ERR_CUDA, std::string("spectrum frequency map: ") + cudaGetErrorString(e));
    }
    if (rc != D4W_OK) { d4w_fk_spectrum_destroy(s); return rc; }
    *out = s;
    return D4W_OK;
}

extern "C" int d4w_fk_spectrum_rows(const d4w_fk_spectrum* s) { return s ? s->sup->nact : 0; }

extern "C" size_t d4w_fk_spectrum_workspace_bytes(const d4w_fk_plan* pl, const d4w_fk_spectrum* s) {
    if (!pl || !s) return 0;
    return kept_rows_bytes(pl, s->sup->nact) + col2_ring_bytes(pl);
}

extern "C" int d4w_fk_spectrum_apply(d4w_fk_plan* pl, d4w_fk_spectrum* s, const float* x, float* out, void* ws, int taper,
                                     float scale, int accumulate, void* stream_v) {
    if (!pl || !s || !x || !out || !ws) return fail(D4W_ERR_ARG, "d4w_fk_spectrum_apply: null argument");
    if (s->plan->device != pl->device) return fail(D4W_ERR_ARG, "d4w_fk_spectrum_apply: plan and spectrum live on different devices");
    if (s->plan != pl) return fail(D4W_ERR_ARG, "d4w_fk_spectrum_apply: spectrum was made for a different plan");
    if (accumulate != 0 && accumulate != 1) return fail(D4W_ERR_ARG, "d4w_fk_spectrum_apply: accumulate must be 0 or 1");
    if (check_matrix_alignment(x, pl->ns, "d4w_fk_spectrum_apply: input") != D4W_OK) return D4W_ERR_ARG;
    DeviceGuard guard(pl->device);
    cudaStream_t stream = (cudaStream_t)stream_v;
    const d4w_fk_mask* sup = s->sup;
    const int nact = sup->nact;
    float2* w = (float2*)ws;
    cpd* v2 = use_two_level(pl, sup, ws) ? reinterpret_cast<cpd*>((char*)ws + kept_rows_bytes(pl, nact)) : nullptr;
    int rc = fk_run_pass(pl, sup, x, nullptr, w, v2, nullptr, nullptr, taper ? pl->d_taper : nullptr, 1, nact, stream);
    if (rc == D4W_OK) rc = fk_run_pass(pl, sup, nullptr, nullptr, w, v2, nullptr, nullptr, nullptr, 2, nact, stream);
    if (rc != D4W_OK) return rc;
    SpecParams sp{};
    sp.act_k = sup->d_act_k; sp.k2pos_row = s->d_k2pos_row; sp.nx = pl->nx; sp.ns = pl->ns;
    sp.k_lo = s->k_lo; sp.k_hi = s->k_hi; sp.f_lo = s->f_lo; sp.f_hi = s->f_hi; sp.scale = scale; sp.accumulate = accumulate;
    return launch_fk_power(dim3(pl->t1, nact), pl->row_threads, pl->row_smem, pl->row, sp, w, (size_t)pl->ns, out, pl->device,
                           stream);
}
