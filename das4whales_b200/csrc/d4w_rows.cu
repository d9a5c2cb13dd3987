// d4w_rows.cu -- host side of the per-channel operators (C ABI in include/d4w.h).
#include <algorithm>
#include <cmath>
#include <cstring>
#include "d4w_common.hpp"
#include "fk_hostplan.hpp"
#include "row_plan.hpp"
#include "rows_kernels.cuh"
#include "xcorr_launch.cuh"

using namespace d4w;

// ------------------------------------------------------------------ generic smem FFT plan (xcorr blocks, STFT frames)
// struct d4w_fft_plan: xcorr_launch.cuh

extern "C" int d4w_fft_plan_create(d4w_fft_plan** out, int n, int device) {
    if (!out) return fail(D4W_ERR_ARG, "d4w_fft_plan_create: null output");
    *out = nullptr;
    if (n < 2) return fail(D4W_ERR_ARG, "d4w_fft_plan_create: n must be >= 2");
    DeviceGuard guard(device);
    cudaDeviceProp prop;
    D4W_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    auto p = new d4w_fft_plan();
    p->n = n; p->device = device; p->smem_cap = prop.sharedMemPerBlockOptin;
    std::string err;
    // overlap-save block lengths (rows.py _pick_block): big even radix first, small odd radix last suits k_xcorr_fused
    const char* forced = std::getenv("D4W_BLOCK_PLAN");
    // dual-lane matched filter (default): radices <= 10 only (register budget of two 256-thread CTAs per SM)
    const bool dual_blocks = env_int("D4W_XCORR_DUAL", 1) != 0;
    const char* pref = dual_blocks ? (n == 1250 ? "10,5,5,5" : n == 2500 ? "10,10,5,5" : n == 5000 ? "10,10,10,5" : n == 10000 ? "10,10,10,10" : nullptr)
                                   : (n == 1250 ? "10,25,5" : n == 2500 ? "20,25,5" : n == 5000 ? "20,10,25" : n == 10000 ? "20,20,25" : nullptr);
    bool have = false;
    if (forced && *forced) have = make_plan_from_string(n, forced, p->pl);
    if (!have && pref && env_int("D4W_XCORR_FUSED", 1)) have = make_plan_from_string(n, pref, p->pl);
    if (!have && !make_plan(n, env_int("D4W_BLOCK_MAX_RADIX", 25), p->pl, err, 128, 16)) { delete p; return fail(D4W_ERR_UNSUPPORTED, err); }
    p->pos2k = make_pos2freq(p->pl);
    p->tab2k = p->pos2k;
    {
        const int nst = p->pl.nstages;
        if (env_int("D4W_XCORR_FUSED", 1) && nst >= 2 && row_radix_inreg(p->pl.radix[0]) && row_radix_inreg(p->pl.radix[nst - 1])) {
            p->fused = 1;
            const int rl = p->pl.radix[nst - 1], G = n / rl;
            for (int m = 0; m < rl; ++m)
                for (int j = 0; j < G; ++j) p->tab2k[(size_t)m * G + j] = p->pos2k[(size_t)j * rl + m];
        }
    }
    std::vector<int> tpos;
    if (n == kPfaN && env_int("D4W_XCORR_PFA", 1)) {
        // prime-factor plan: positions are [5][7][8][9] digits; table order of the fused last dimension (radix 9)
        p->pfa = 1; p->fused = 0;
        pfa_build_maps(tpos, p->pos2k);
        p->tab2k.assign((size_t)n, 0);
        const int G = n / 9;
        for (int m = 0; m < 9; ++m)
            for (int j = 0; j < G; ++j) p->tab2k[(size_t)m * G + j] = p->pos2k[(size_t)j * 9 + m];
    }
    std::vector<int> k2pos((size_t)n);
    for (int i = 0; i < n; ++i) k2pos[p->pos2k[i]] = i;
    cudaError_t e = upload(&p->d_tw, make_twiddles(n));
    if (e == cudaSuccess) e = upload(&p->d_k2pos, k2pos);
    if (e == cudaSuccess && p->pfa) e = upload(&p->d_tpos, tpos);
    if (e == cudaSuccess && n <= 4096) {
        std::vector<float2> wn((size_t)n);
        for (int j = 0; j < n; ++j) { const double a = -2.0 * M_PI * (double)j / (double)n; wn[j] = make_float2((float)std::cos(a), (float)std::sin(a)); }
        e = upload(&p->d_wn, wn);
    }
    if (e != cudaSuccess) { d4w_fft_plan_destroy(p); return fail(D4W_ERR_CUDA, std::string("fft plan: ") + cudaGetErrorString(e)); }
    *out = p;
    return D4W_OK;
}

extern "C" int d4w_fft_plan_destroy(d4w_fft_plan* p) {
    if (!p) return D4W_OK;
    DeviceGuard guard(p->device);
    cudaFree(p->d_tw); cudaFree(p->d_k2pos); cudaFree(p->d_tpos); cudaFree(p->d_wn);
    delete p;
    return D4W_OK;
}

extern "C" int d4w_fft_plan_order(const d4w_fft_plan* p, int* host_pos2freq) {
    if (!p || !host_pos2freq) return fail(D4W_ERR_ARG, "d4w_fft_plan_order: null argument");
    std::memcpy(host_pos2freq, p->pos2k.data(), (size_t)p->n * sizeof(int));
    return D4W_OK;
}

extern "C" int d4w_fft_plan_table_order(const d4w_fft_plan* p, int* host_tab2freq) {
    if (!p || !host_tab2freq) return fail(D4W_ERR_ARG, "d4w_fft_plan_table_order: null argument");
    std::memcpy(host_tab2freq, p->tab2k.data(), (size_t)p->n * sizeof(int));
    return D4W_OK;
}

// ------------------------------------------------------------------ row statistics / plain SNR
extern "C" int d4w_row_stats(const float* x, int nx, int ns, int seglen, double* stats, double* segpre, void* stream) {
    if (!x || !stats || nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_row_stats: bad argument");
    int nseg = 0;
    if (segpre) {
        if (seglen < 1) return fail(D4W_ERR_ARG, "d4w_row_stats: seglen must be >= 1 when segpre is given");
        nseg = (ns + seglen - 1) / seglen;
        if (nseg > kMaxSeg) return fail(D4W_ERR_UNSUPPORTED, "d4w_row_stats: more than 512 segments per row");
    }
    k_row_stats<<<nx, 256, 0, (cudaStream_t)stream>>>(x, ns, seglen, nseg, stats, segpre);
    D4W_CHECK_LAUNCH("k_row_stats");
    return D4W_OK;
}

extern "C" int d4w_snr(const float* x, float* out, int nx, int ns, const double* stats, void* stream) {
    if (!x || !out || !stats) return fail(D4W_ERR_ARG, "d4w_snr: null argument");
    const size_t total = (size_t)nx * ns;
    const size_t blocks = (total + 255) / 256;
    if (blocks > 0x7fffffffull) return fail(D4W_ERR_UNSUPPORTED, "d4w_snr: matrix too large");
    k_snr_plain<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, out, ns, stats, total);
    D4W_CHECK_LAUNCH("k_snr_plain");
    return D4W_OK;
}

// ------------------------------------------------------------------ overlap-save matched filter
extern "C" int d4w_xcorr(d4w_fft_plan* p, const float* x, int nx, int ns, int valid, int ntpl, const void* dev_tabs,
                         const double* dev_mu_over_m, const double* dev_stats, const double* dev_segpre, float* out,
                         void* stream) {
    if (!p || !x || !dev_tabs || !out) return fail(D4W_ERR_ARG, "d4w_xcorr: null argument");
    if (valid < 1 || valid > p->n || ntpl < 1) return fail(D4W_ERR_ARG, "d4w_xcorr: bad valid / ntpl");
    const bool normalize = dev_stats != nullptr;
    if (normalize && (!dev_segpre || !dev_mu_over_m)) return fail(D4W_ERR_ARG, "d4w_xcorr: normalisation needs stats, segpre and mu");
    return xcorr_launch<false>(p, x, nx, ns, valid, ntpl, dev_tabs, dev_mu_over_m, dev_stats, dev_segpre, nullptr, 0, out, stream);
}

// ------------------------------------------------------------------ Hilbert envelope / envelope SNR
// struct d4w_row_plan: row_plan.hpp

// plan for a row length the time-axis planner rejects: chirp-z transform over an m-point convolution
static int row_plan_create_czt(d4w_row_plan** out, int ns, int device, const cudaDeviceProp& prop) {
    RowCztPlan cz; std::string err;
    if (plan_czt_rows(ns, prop.sharedMemPerBlockOptin, cz, err)) return fail(D4W_ERR_UNSUPPORTED, err);
    const FkHostPlan& hp = cz.hp;
    auto p = new d4w_row_plan();
    p->ns = ns; p->device = device; p->t1 = hp.t1; p->t2 = hp.t2; p->row_smem = hp.row_smem;
    p->row.pl = hp.rowpl; p->row.t1 = hp.t1; p->row.t2 = hp.t2;
    p->fused = cz.fused; p->czt_m = cz.m;
    p->pair = (hp.t1 > 1 && env_int("D4W_HILBERT_PAIR", 1)) ? 1 : 0;
    std::vector<float2> bc(cz.bhat.size());
    for (size_t i = 0; i < bc.size(); ++i) bc[i] = make_float2(cz.bhat[i].x, -cz.bhat[i].y);
    cudaError_t e = upload(&p->d_tw, hp.tw_row);
    if (e == cudaSuccess) e = upload(&p->d_twT, hp.twT);
    if (e == cudaSuccess) e = upload(&p->d_chirp, cz.chirp);
    if (e == cudaSuccess) e = upload(&p->d_bhat, cz.bhat);
    if (e == cudaSuccess) e = upload(&p->d_bhatc, bc);
    const int smax = (int)prop.sharedMemPerBlockOptin;
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid_c, cudaFuncAttributeMaxDynamicSharedMemorySize, smax);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid_fused_c, cudaFuncAttributeMaxDynamicSharedMemorySize, smax);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_hczt_row, cudaFuncAttributeMaxDynamicSharedMemorySize, smax);
    if (e != cudaSuccess) { d4w_row_plan_destroy(p); return fail(D4W_ERR_CUDA, std::string("row plan: ") + cudaGetErrorString(e)); }
    p->row.tw = p->d_tw; p->row.twT = p->d_twT;
    *out = p;
    return D4W_OK;
}

extern "C" int d4w_row_plan_create(d4w_row_plan** out, int ns, int device) {
    if (!out) return fail(D4W_ERR_ARG, "d4w_row_plan_create: null output");
    *out = nullptr;
    if (ns < 1) return fail(D4W_ERR_ARG, "d4w_row_plan_create: ns must be >= 1");
    DeviceGuard guard(device);
    cudaDeviceProp prop;
    D4W_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    FkHostPlan hp; std::string err;
    // the envelope keeps k_row_mid_fused: 10 000 x 120 000 on an H100 took 15.5 ms with it and 16.9 ms with k_row_mid
    // (two rows per transform both ways; one row per transform: 25.1 ms)
    // a length with no T1 x T2 split (a prime factor > 61, or T2 too long) goes through the chirp-z rows
    if (build_fk_hostplan(1, ns, prop.sharedMemPerBlockOptin, hp, err, /*allow_row_dual=*/false, /*row_fused_default=*/1))
        return row_plan_create_czt(out, ns, device, prop);
    auto p = new d4w_row_plan();
    p->ns = ns; p->device = device; p->t1 = hp.t1; p->t2 = hp.t2; p->row_smem = hp.row_smem;
    p->row.pl = hp.rowpl; p->row.t1 = hp.t1; p->row.t2 = hp.t2;
    // analytic-signal weights of scipy.signal.hilbert (N = ns, no padding), scaled by 1/ns, transform order
    std::vector<float> h((size_t)ns);
    p->fused = (hp.t1 > 1 && hp.row_fused) ? 1 : 0;
    const std::vector<int>& order = p->fused ? hp.pos2k_row_tab : hp.pos2k_row;
    for (int kt1 = 0; kt1 < hp.t1; ++kt1)
        for (int pos = 0; pos < hp.t2; ++pos) {
            const int f = kt1 + hp.t1 * order[pos];
            double wgt;
            if (ns % 2 == 0) wgt = (f == 0 || f == ns / 2) ? 1.0 : (f < ns / 2 ? 2.0 : 0.0);
            else wgt = (f == 0) ? 1.0 : (f <= (ns - 1) / 2 ? 2.0 : 0.0);
            h[(size_t)kt1 * hp.t2 + pos] = (float)(wgt / ns);
        }
    // two real rows per complex transform; sg inherits h's table order, so either middle-pass kernel can apply it
    std::vector<float> sg;
    if (hp.t1 > 1 && env_int("D4W_HILBERT_PAIR", 1)) {
        sg.resize((size_t)ns);
        for (size_t i = 0; i < sg.size(); ++i) sg[i] = h[i] - (float)(1.0 / ns);      // h - 1: 0 at DC / Nyquist, +-1 elsewhere
    }
    cudaError_t e = upload(&p->d_tw, hp.tw_row);
    if (e == cudaSuccess) e = upload(&p->d_twT, hp.twT);
    if (e == cudaSuccess) e = upload(&p->d_hilbert, h);
    if (e == cudaSuccess && !sg.empty()) e = upload(&p->d_sgn, sg);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_row_mid_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_hilbert_row, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin);
    if (e != cudaSuccess) { d4w_row_plan_destroy(p); return fail(D4W_ERR_CUDA, std::string("row plan: ") + cudaGetErrorString(e)); }
    p->row.tw = p->d_tw; p->row.twT = p->d_twT;
    *out = p;
    return D4W_OK;
}

extern "C" int d4w_row_plan_destroy(d4w_row_plan* p) {
    if (!p) return D4W_OK;
    DeviceGuard guard(p->device);
    cudaFree(p->d_tw); cudaFree(p->d_twT); cudaFree(p->d_hilbert); cudaFree(p->d_sgn);
    cudaFree(p->d_chirp); cudaFree(p->d_bhat); cudaFree(p->d_bhatc);
    delete p;
    return D4W_OK;
}

extern "C" size_t d4w_row_workspace_bytes(const d4w_row_plan* p, int nx) {
    if (!p || p->t1 == 1) return 16;
    const bool pair = p->czt_m ? p->pair != 0 : p->d_sgn != nullptr;
    const size_t rows = pair ? (size_t)(nx + 1) / 2 : (size_t)nx;      // two real rows share one complex workspace row
    return rows * (size_t)(p->czt_m ? p->czt_m : p->ns) * sizeof(float2);
}

extern "C" int d4w_row_plan_info(const d4w_row_plan* p, int* t1, int* t2, int* czt_m) {
    if (!p) return fail(D4W_ERR_ARG, "d4w_row_plan_info: null plan");
    if (t1) *t1 = p->t1;
    if (t2) *t2 = p->t2;
    if (czt_m) *czt_m = p->czt_m;
    return D4W_OK;
}

// chirp-z rows: one CTA per row (t1 == 1), or the five split launches of hilbert_czt.cuh
static int hilbert_czt(d4w_row_plan* p, const float* x, float* out, int nx, void* workspace, int mode, const double* dev_stats,
                       cudaStream_t stream) {
    HcztParams hz{};
    hz.n = p->ns; hz.m = p->czt_m; hz.t2 = p->t2; hz.nx = nx; hz.pair = p->pair; hz.invn = (float)(1.0 / p->ns);
    hz.chirp = p->d_chirp; hz.twT = p->d_twT;
    if (p->t1 == 1) {
        k_hczt_row<<<nx, 256, p->row_smem, stream>>>(p->row, hz, p->d_bhat, p->d_bhatc, x, out, mode, dev_stats);
        D4W_CHECK_LAUNCH("k_hczt_row");
        return D4W_OK;
    }
    if (!workspace) return fail(D4W_ERR_ARG, "d4w_hilbert: workspace required for split rows");
    float2* w = (float2*)workspace;
    const int nrow = p->pair ? (nx + 1) / 2 : nx, thr = 128;
    const dim3 g((p->t2 + thr - 1) / thr, nrow), gm(p->t1, nrow);
    auto mid = [&](const float2* tab) {
        if (p->fused) k_row_mid_fused_c<<<gm, 256, p->row_smem, stream>>>(p->row, w, (size_t)p->czt_m, tab, (size_t)0);
        else k_row_mid_c<<<gm, 256, p->row_smem, stream>>>(p->row, w, (size_t)p->czt_m, tab, (size_t)0);
    };
    switch (p->t1) {
#define D4W_HC(T) case T: k_hczt_fwd<T><<<g, thr, 0, stream>>>(hz, x, w); break;
        D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
        default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
    }
    D4W_CHECK_LAUNCH("k_hczt_fwd");
    mid(p->d_bhat);
    D4W_CHECK_LAUNCH("k_row_mid_c");
    switch (p->t1) {
#define D4W_HC(T) case T: k_hczt_turn<T><<<g, thr, 0, stream>>>(hz, w); break;
        D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
        default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
    }
    D4W_CHECK_LAUNCH("k_hczt_turn");
    mid(p->d_bhatc);
    D4W_CHECK_LAUNCH("k_row_mid_c");
    switch (p->t1) {
#define D4W_HC(T) case T: k_hczt_inv<T><<<g, thr, 0, stream>>>(hz, w, x, out, mode, dev_stats); break;
        D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
        default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
    }
    D4W_CHECK_LAUNCH("k_hczt_inv");
    return D4W_OK;
}

extern "C" int d4w_hilbert(d4w_row_plan* p, const float* x, float* out, int nx, void* workspace, int mode,
                           const double* dev_stats, void* stream_v) {
    if (!p || !x || !out || nx < 1) return fail(D4W_ERR_ARG, "d4w_hilbert: bad argument");
    if (mode < 0 || mode > EPI_ENVSTD) return fail(D4W_ERR_ARG, "d4w_hilbert: mode must be 0..3");
    if ((mode == EPI_SNR || mode == EPI_ENVSTD) && !dev_stats) return fail(D4W_ERR_ARG, "d4w_hilbert: this mode needs row statistics");
    if (nx > 65535 && p->t1 > 1) return fail(D4W_ERR_UNSUPPORTED, "d4w_hilbert: more than 65535 rows per call");
    DeviceGuard guard(p->device);
    cudaStream_t stream = (cudaStream_t)stream_v;
    if (p->czt_m) return hilbert_czt(p, x, out, nx, workspace, mode, dev_stats, stream);
    if (p->t1 == 1) {
        k_hilbert_row<<<nx, 256, p->row_smem, stream>>>(p->row, x, out, p->d_hilbert, mode, dev_stats);
        D4W_CHECK_LAUNCH("k_hilbert_row");
        return D4W_OK;
    }
    if (!workspace) return fail(D4W_ERR_ARG, "d4w_hilbert: workspace required for split rows");
    if (p->d_sgn) {                                              // two real rows per complex transform
        float2* w2 = (float2*)workspace;
        const int npair = (nx + 1) / 2, thr = 128;
        dim3 g2((p->t2 + thr - 1) / thr, npair);
        switch (p->t1) {
#define D4W_HC(T) case T: k_hsplit_fwd2<T><<<g2, thr, 0, stream>>>(x, nx, p->ns, w2, p->t2, p->d_twT); break;
            D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
            default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
        }
        D4W_CHECK_LAUNCH("k_hsplit_fwd2");
        dim3 gm(p->t1, npair);
        if (p->fused) k_row_mid_fused<<<gm, 256, p->row_smem, stream>>>(p->row, w2, (size_t)p->ns, p->d_sgn, (size_t)0);
        else k_row_mid<<<gm, 256, p->row_smem, stream>>>(p->row, w2, (size_t)p->ns, p->d_sgn, (size_t)0);
        D4W_CHECK_LAUNCH("k_row_mid");
        switch (p->t1) {
#define D4W_HC(T) case T: k_hsplit_inv2<T><<<g2, thr, 0, stream>>>(w2, x, nx, p->ns, out, p->t2, p->d_twT, mode, dev_stats); break;
            D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
            default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
        }
        D4W_CHECK_LAUNCH("k_hsplit_inv2");
        return D4W_OK;
    }
    float2* w = (float2*)workspace;
    const int threads = 128;
    dim3 grid((p->t2 + threads - 1) / threads, nx);
    switch (p->t1) {
#define D4W_HC(T) case T: k_hsplit_fwd<T><<<grid, threads, 0, stream>>>(x, p->ns, w, p->t2, p->d_twT); break;
        D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
        default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
    }
    D4W_CHECK_LAUNCH("k_hsplit_fwd");
    dim3 gmid(p->t1, nx);
    if (p->fused) k_row_mid_fused<<<gmid, 256, p->row_smem, stream>>>(p->row, w, (size_t)p->ns, p->d_hilbert, (size_t)0);
    else k_row_mid<<<gmid, 256, p->row_smem, stream>>>(p->row, w, (size_t)p->ns, p->d_hilbert, (size_t)0);
    D4W_CHECK_LAUNCH("k_row_mid");
    switch (p->t1) {
#define D4W_HC(T) case T: k_hsplit_inv<T><<<grid, threads, 0, stream>>>(w, p->ns, out, p->t2, p->d_twT, mode, dev_stats); break;
        D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
        default: return fail(D4W_ERR_UNSUPPORTED, "row split radix not built");
    }
    D4W_CHECK_LAUNCH("k_hsplit_inv");
    return D4W_OK;
}

// ------------------------------------------------------------------ forward-backward SOS IIR
extern "C" int d4w_sosfiltfilt(const float* x, float* y, float* tmp, int nx, int ns, const double* host_sos,
                               const double* host_zi, int nsec, int padlen, void* stream_v) {
    if (!x || !y || !tmp || !host_sos || !host_zi) return fail(D4W_ERR_ARG, "d4w_sosfiltfilt: null argument");
    if (nsec < 1 || nsec > kMaxSections) return fail(D4W_ERR_UNSUPPORTED, "d4w_sosfiltfilt: 1..16 sections supported");
    if (padlen < 0 || ns <= padlen) return fail(D4W_ERR_ARG, "The length of the input vector x must be greater than padlen");
    SosParams sp{};
    for (int s = 0; s < nsec; ++s) {
        const double* c = host_sos + 6 * s;
        const double a0 = c[3];
        sp.b0[s] = c[0] / a0; sp.b1[s] = c[1] / a0; sp.b2[s] = c[2] / a0; sp.a1[s] = c[4] / a0; sp.a2[s] = c[5] / a0;
        sp.zi0[s] = host_zi[2 * s]; sp.zi1[s] = host_zi[2 * s + 1];
    }
    sp.nsec = nsec; sp.pad = padlen; sp.ns = ns;
    cudaStream_t stream = (cudaStream_t)stream_v;
    const int blocks = (nx + 31) / 32;
    // time chunking with a warm-up chosen from the slowest pole: |p|^warm < 1e-9 (exact at fp32 precision)
    double rmax = 0.0;
    for (int s = 0; s < nsec; ++s) {
        const double a1 = sp.a1[s], a2 = sp.a2[s];
        const double disc = a1 * a1 - 4.0 * a2;
        const double r = disc < 0 ? std::sqrt(std::fabs(a2)) : std::max(std::fabs((-a1 + std::sqrt(disc)) / 2), std::fabs((-a1 - std::sqrt(disc)) / 2));
        rmax = std::max(rmax, r);
    }
    const int next = ns + 2 * padlen;
    int chunk = 0, warm = 0;
    if (env_int("D4W_IIR_CHUNKED", 1) && rmax > 0.0 && rmax < 0.9995) {
        warm = (int)std::ceil(std::log(1e-9) / std::log(rmax)) + 32;
        warm = (warm + 31) / 32 * 32;
        chunk = std::max(4 * warm, 4096);
        chunk = (chunk + 31) / 32 * 32;
        if (next < 2 * chunk) chunk = 0;          // short signals: plain sequential recursion
    }
    const int nchunks = chunk > 0 ? (next + chunk - 1) / chunk : 1;
    // four warps per block (one 32-channel group each); with time chunking every warp walks two chunks at once
    const int nch = (nchunks >= 2 && env_int("D4W_IIR_NCH", 2) >= 2) ? 2 : 1;
    dim3 grid((blocks + 3) / 4, (nchunks + nch - 1) / nch);
#define D4W_SOS(NS_, NCH_)                                                                               \
    do {                                                                                                 \
        const size_t sm_ = (size_t)4 * 2 * NCH_ * 32 * 33 * sizeof(float);                               \
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_sos_pass<1, NS_, NCH_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_));   \
        D4W_CUDA_TRY(cudaFuncSetAttribute(k_sos_pass<-1, NS_, NCH_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_));  \
        k_sos_pass<1, NS_, NCH_><<<grid, 128, sm_, stream>>>(sp, x, tmp, y, nx, chunk, warm, nchunks);   \
        D4W_CHECK_LAUNCH("k_sos_pass<fwd>");                                                             \
        k_sos_pass<-1, NS_, NCH_><<<grid, 128, sm_, stream>>>(sp, x, tmp, y, nx, chunk, warm, nchunks);  \
        D4W_CHECK_LAUNCH("k_sos_pass<bwd>");                                                             \
    } while (0)
    if (nch == 2) {
        switch (nsec) {
            case 1: D4W_SOS(1, 2); break; case 2: D4W_SOS(2, 2); break; case 3: D4W_SOS(3, 2); break; case 4: D4W_SOS(4, 2); break;
            case 5: D4W_SOS(5, 2); break; case 6: D4W_SOS(6, 2); break; case 8: D4W_SOS(8, 2); break;
            default: D4W_SOS(0, 1); break;
        }
    } else {
        switch (nsec) {
            case 1: D4W_SOS(1, 1); break; case 2: D4W_SOS(2, 1); break; case 3: D4W_SOS(3, 1); break; case 4: D4W_SOS(4, 1); break;
            case 5: D4W_SOS(5, 1); break; case 6: D4W_SOS(6, 1); break; case 8: D4W_SOS(8, 1); break;
            default: D4W_SOS(0, 1); break;
        }
    }
#undef D4W_SOS
    return D4W_OK;
}

// ------------------------------------------------------------------ batched STFT magnitude
extern "C" int d4w_stft_mag(d4w_fft_plan* p, const float* x, float* out, int nx, int ns, int hop, const float* dev_window,
                            int bin_lo, int bin_hi, void* stream_v) {
    if (!p || !x || !out || !dev_window) return fail(D4W_ERR_ARG, "d4w_stft_mag: null argument");
    if (p->n % 2 || hop < 1) return fail(D4W_ERR_ARG, "d4w_stft_mag: n_fft must be even and hop >= 1");
    if (nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_stft_mag: more than 65535 rows per call");
    DeviceGuard guard(p->device);
    StftParams sp{};
    sp.pl = p->pl; sp.tw = p->d_tw; sp.k2pos = p->d_k2pos;
    if (bin_lo < 0 || bin_hi > p->n / 2 || bin_lo > bin_hi) return fail(D4W_ERR_ARG, "d4w_stft_mag: bad bin range");
    sp.nfft = p->n; sp.hop = hop; sp.ns = ns; sp.nframes = 1 + ns / hop; sp.nbins = bin_hi - bin_lo + 1; sp.bin_lo = bin_lo;
    int fpb = 32;
    while (fpb > 2 && (size_t)(fpb / 2) * (p->n + 1) * sizeof(float2) > 96 * 1024) fpb >>= 1;
    sp.fpb = fpb;
    const size_t smem = (size_t)(fpb / 2) * (p->n + 1) * sizeof(float2);
    if (smem > p->smem_cap) return fail(D4W_ERR_UNSUPPORTED, "d4w_stft_mag: n_fft too large for shared memory");
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_stft_mag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_cap));
    dim3 grid((sp.nframes + fpb - 1) / fpb, nx);
    k_stft_mag<<<grid, 256, smem, (cudaStream_t)stream_v>>>(sp, x, dev_window, out);
    D4W_CHECK_LAUNCH("k_stft_mag");
    return D4W_OK;
}

// sliding-DFT variant for a band of bins of heavily overlapping Hann frames (k_stft_slide); n_fft = hop * P
template <int H, int P, int G>
static int launch_stft_slide_g(d4w_fft_plan* p, const float* x, float* out, int nx, SlideParams sp, cudaStream_t st) {
    auto bytes = [&](int Q) {
        return (size_t)G * slide_run_stride(P * Q * H, H * P) * sizeof(float) + (size_t)G * P * sp.nYp * sizeof(float2);
    };
    while (sp.Q > 1 && bytes(sp.Q) > 110 * 1024) --sp.Q;          // two CTAs per SM (the register budget allows no more)
    const int R = P * sp.Q;
    const size_t smem = bytes(sp.Q);
    if (smem > p->smem_cap) return fail(D4W_ERR_UNSUPPORTED, "d4w_stft_slide: tile does not fit shared memory");
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_stft_slide<H, P, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_cap));
    const int threads = std::min(kSlideMaxThreads, std::max((G * sp.nY + 31) / 32 * 32, 320));
    dim3 grid((sp.nframes + G * R - 1) / (G * R), nx);
    k_stft_slide<H, P, G><<<grid, threads, smem, st>>>(sp, x, p->d_wn, out);
    D4W_CHECK_LAUNCH("k_stft_slide");
    return D4W_OK;
}

// runs per CTA: narrow bands take more runs so that runs x (bins + 2) threads fill the CTA
template <int H, int P>
static int launch_stft_slide(d4w_fft_plan* p, const float* x, float* out, int nx, const SlideParams& sp, cudaStream_t st) {
    // measured on 1000 x 120 000 (scripts/gpu_slide_tune.py): 16 runs only pay below ~10 bins (0.69 vs 0.86 ms for 7 bins);
    // at 13 bins their larger sample buffer forces shorter runs and loses (1.15 vs 0.94 ms)
    int G = sp.nY <= 10 ? 16 : 8;
    const int forced = env_int("D4W_SLIDE_G", 0);                 // tuning override; must keep G * nY <= 320
    if ((forced == 8 || forced == 16) && forced * sp.nY <= kSlideMaxThreads) G = forced;
    if (G == 16) return launch_stft_slide_g<H, P, 16>(p, x, out, nx, sp, st);
    return launch_stft_slide_g<H, P, 8>(p, x, out, nx, sp, st);
}

extern "C" int d4w_stft_slide_supported(int nfft, int hop, int nbins) {
    if (!env_int("D4W_STFT_SLIDE", 1)) return 0;
    if (nbins < 1 || 8 * (nbins + 2) > kSlideMaxThreads) return 0;
    return (nfft == 160 && hop == 8) || (nfft == 128 && hop == 8) || (nfft == 256 && hop == 16);
}

extern "C" int d4w_stft_slide(d4w_fft_plan* p, const float* x, float* out, int nx, int ns, int hop, int bin_lo, int bin_hi,
                              void* stream_v) {
    if (!p || !x || !out) return fail(D4W_ERR_ARG, "d4w_stft_slide: null argument");
    if (bin_lo < 0 || bin_hi > p->n / 2 || bin_lo > bin_hi) return fail(D4W_ERR_ARG, "d4w_stft_slide: bad bin range");
    if (nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_stft_slide: empty input");
    if (nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_stft_slide: more than 65535 rows per call");
    const int nbins = bin_hi - bin_lo + 1;
    if (!d4w_stft_slide_supported(p->n, hop, nbins) || !p->d_wn)
        return fail(D4W_ERR_UNSUPPORTED, "d4w_stft_slide: (n_fft, hop, band) not covered, use d4w_stft_mag");
    DeviceGuard guard(p->device);
    SlideParams sp{};
    sp.ns = ns; sp.nframes = 1 + ns / hop; sp.nbins = nbins; sp.bin_lo = bin_lo;
    sp.nY = nbins + 2; sp.nYp = sp.nY | 1;                   // odd pitch: conflict-free 8-byte reads along frames
    sp.Q = std::max(1, env_int("D4W_SLIDE_Q", 8));
    cudaStream_t st = (cudaStream_t)stream_v;
    if (p->n == 160) return launch_stft_slide<8, 20>(p, x, out, nx, sp, st);
    if (p->n == 128) return launch_stft_slide<8, 16>(p, x, out, nx, sp, st);
    return launch_stft_slide<16, 16>(p, x, out, nx, sp, st);
}

// ------------------------------------------------------------------ per-channel FFT magnitude (dsp.get_fx)
extern "C" int d4w_row_fft_mag(d4w_fft_plan* p, const float* x, int nx, size_t ld, int ncopy, double scale, float* out, void* stream_v) {
    if (!p || !x || !out || nx < 1 || ncopy < 0) return fail(D4W_ERR_ARG, "d4w_row_fft_mag: bad argument");
    if (ncopy > p->n) ncopy = p->n;                      // numpy.fft.fft(a, n) crops rows longer than n
    const size_t smem = (size_t)p->n * sizeof(float2);
    if (smem > p->smem_cap) return fail(D4W_ERR_UNSUPPORTED, "d4w_row_fft_mag: nfft too large for shared memory (max ~28 000)");
    DeviceGuard guard(p->device);
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_row_fftmag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_cap));
    k_row_fftmag<<<nx, 256, smem, (cudaStream_t)stream_v>>>(p->pl, p->d_tw, p->d_k2pos, x, ld, ncopy, (float)scale, out);
    D4W_CHECK_LAUNCH("k_row_fftmag");
    return D4W_OK;
}

// ------------------------------------------------------------------ medians / maxima / spectrogram correlation
extern "C" int d4w_row_median_ld(const float* x, int nrows, size_t n, size_t ld, float* med, void* stream) {
    if (!x || !med || nrows < 1 || n < 1 || ld < n) return fail(D4W_ERR_ARG, "d4w_row_median: bad argument");
    const size_t smem = (size_t)kMedCap * sizeof(float);
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_row_median, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_row_median<<<nrows, kMedThreads, smem, (cudaStream_t)stream>>>(x, n, ld, med);
    D4W_CHECK_LAUNCH("k_row_median");
    return D4W_OK;
}

extern "C" int d4w_row_median(const float* x, int nrows, size_t n, float* med, void* stream) {
    return d4w_row_median_ld(x, nrows, n, n, med, stream);
}

extern "C" int d4w_row_max(const float* x, int nrows, size_t n, float* mx, void* stream) {
    if (!x || !mx || nrows < 1 || n < 1) return fail(D4W_ERR_ARG, "d4w_row_max: bad argument");
    k_row_max<<<nrows, 256, 0, (cudaStream_t)stream>>>(x, n, mx);
    D4W_CHECK_LAUNCH("k_row_max");
    return D4W_OK;
}

// One spectrogram kernel of d4w_speccorr_multi: its rows are S[:, f0 : f0 + nf, :].
struct SpecKernel { const float* K; const float* med; float* out; int f0, nf, kw; };

// k_speccorr4 parameters for kernels ks[0 .. nk-1] sharing one staged tile; returns the dynamic shared memory it needs
static size_t speccorr4_set(const SpecKernel* ks, int nk, int nfs, SpecCorrSet& set) {
    set = SpecCorrSet{};
    set.nk = nk; set.nfs = nfs;
    int c0 = 0, fs0 = nfs, fs1 = 0;
    for (int k = 0; k < nk; ++k) {
        c0 = std::max(c0, ks[k].kw / 2);
        fs0 = std::min(fs0, ks[k].f0);
        fs1 = std::max(fs1, ks[k].f0 + ks[k].nf);
    }
    int kwp = 4, nsk = 0;
    for (int k = 0; k < nk; ++k) {
        set.K[k] = ks[k].K; set.med[k] = ks[k].med; set.out[k] = ks[k].out;
        set.f0[k] = ks[k].f0 - fs0; set.nf[k] = ks[k].nf; set.kw[k] = ks[k].kw;
        set.pad[k] = c0 - ks[k].kw / 2;
        kwp = std::max(kwp, (set.pad[k] + ks[k].kw + 3) & ~3);
        nsk += ks[k].nf;
    }
    set.fs0 = fs0; set.nst = fs1 - fs0; set.c0 = c0; set.kwp = kwp;
    return ((size_t)nsk * kwp + (size_t)set.nst * (kScTile + kwp)) * sizeof(float);
}

static int launch_speccorr4(const float* S, int nx, int nt, const SpecCorrSet& set, size_t smem, cudaStream_t st) {
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_speccorr4, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid4((nt + kScTile - 1) / kScTile, nx);
    k_speccorr4<<<grid4, kScThreads, smem, st>>>(S, nt, set);
    D4W_CHECK_LAUNCH("k_speccorr4");
    return D4W_OK;
}

// Untiled kernel for one spectrogram kernel too wide for k_speccorr4.  k_speccorr reads [nx][nf][nt]: a band of a wider
// spectrogram (nfs > nf rows) is first copied to a dense stream-ordered scratch matrix.
static int launch_speccorr_untiled(const float* S, int nx, int nfs, int nt, const SpecKernel& kk, cudaStream_t st) {
    const int tile = 256, nf = kk.nf, kw = kk.kw;
    const size_t smem = ((size_t)nf * kw + (size_t)nf * (tile + kw)) * sizeof(float);
    if (smem > 200 * 1024) return fail(D4W_ERR_UNSUPPORTED, "d4w_speccorr: kernel too large for shared memory");
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_speccorr, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    dim3 grid((nt + tile - 1) / tile, nx);
    if (nfs == nf) {
        k_speccorr<<<grid, tile, smem, st>>>(S, nf, nt, kk.K, kw, kk.med, kk.out);
        D4W_CHECK_LAUNCH("k_speccorr");
        return D4W_OK;
    }
    const size_t band = (size_t)nf * nt * sizeof(float);
    float* tmp = nullptr;
    D4W_CUDA_TRY(cudaMallocAsync((void**)&tmp, band * nx, st));
    cudaError_t e = cudaMemcpy2DAsync(tmp, band, S + (size_t)kk.f0 * nt, (size_t)nfs * nt * sizeof(float), band, nx,
                                      cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) {
        k_speccorr<<<grid, tile, smem, st>>>(tmp, nf, nt, kk.K, kw, kk.med, kk.out);
        e = cudaGetLastError();
    }
    const cudaError_t ef = cudaFreeAsync(tmp, st);
    D4W_CUDA_TRY(e);
    D4W_CUDA_TRY(ef);
    D4W_CHECK_LAUNCH("k_speccorr");
    return D4W_OK;
}

// All kernels in one k_speccorr4 pass when their tile fits; otherwise one pass per kernel, tiled or untiled.
static int speccorr_kernels(const float* S, int nx, int nfs, int nt, const SpecKernel* ks, int nk, cudaStream_t st) {
    const bool tiled = env_int("D4W_SPECCORR4", 1) != 0;
    SpecCorrSet set;
    size_t smem = speccorr4_set(ks, nk, nfs, set);
    if (tiled && smem <= 110 * 1024) return launch_speccorr4(S, nx, nt, set, smem, st);
    for (int k = 0; k < nk; ++k) {
        smem = speccorr4_set(ks + k, 1, nfs, set);
        const int rc = (tiled && smem <= 110 * 1024) ? launch_speccorr4(S, nx, nt, set, smem, st)
                                                     : launch_speccorr_untiled(S, nx, nfs, nt, ks[k], st);
        if (rc != D4W_OK) return rc;
    }
    return D4W_OK;
}

extern "C" int d4w_speccorr(const float* S, int nx, int nf, int nt, const float* K, int kw, const float* med, float* out,
                            void* stream) {
    if (!S || !K || !med || !out || nx < 1 || nf < 1 || nt < 1 || kw < 1) return fail(D4W_ERR_ARG, "d4w_speccorr: bad argument");
    if (nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_speccorr: more than 65535 rows per call");
    const SpecKernel kk{K, med, out, 0, nf, kw};
    return speccorr_kernels(S, nx, nf, nt, &kk, 1, (cudaStream_t)stream);
}

extern "C" int d4w_speccorr_multi(const float* S, int nx, int nf, int nt, int nk, const int* f0, const int* nfk,
                                  const float* const* K, const int* kw, const float* const* med, float* const* out,
                                  void* stream) {
    if (!S || !f0 || !nfk || !K || !kw || !med || !out || nx < 1 || nf < 1 || nt < 1 || nk < 1 || nk > kScMaxKernels)
        return fail(D4W_ERR_ARG, "d4w_speccorr_multi: bad argument");
    SpecKernel ks[kScMaxKernels];
    for (int k = 0; k < nk; ++k) {
        if (!K[k] || !med[k] || !out[k] || kw[k] < 1 || nfk[k] < 1 || f0[k] < 0 || f0[k] + nfk[k] > nf)
            return fail(D4W_ERR_ARG, "d4w_speccorr_multi: bad kernel");
        ks[k] = SpecKernel{K[k], med[k], out[k], f0[k], nfk[k], kw[k]};
    }
    if (nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_speccorr_multi: more than 65535 rows per call");
    return speccorr_kernels(S, nx, nf, nt, ks, nk, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------- peak picking
static void peak_level_sizes(int ns, int& nb1, int& nb2) { nb1 = (ns + kPkB - 1) / kPkB; nb2 = (nb1 + kPkB - 1) / kPkB; }

extern "C" size_t d4w_find_peaks_workspace_bytes(int nx, int ns) {
    if (nx < 1 || ns < 1) return 0;
    int nb1, nb2; peak_level_sizes(ns, nb1, nb2);
    return ((size_t)nx * (2 * (size_t)nb1 + 2 * (size_t)nb2 + 1)) * sizeof(float) + 256;
}

extern "C" int d4w_find_peaks(const float* x, int nx, int ns, double prominence, unsigned char* flags, void* ws, void* stream_v) {
    if (!x || !flags || !ws || nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_find_peaks: bad argument");
    if (nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_find_peaks: more than 65535 rows per call");
    if (!(prominence >= 0.0)) return fail(D4W_ERR_ARG, "d4w_find_peaks: prominence must be >= 0");
    cudaStream_t stream = (cudaStream_t)stream_v;
    D4W_CUDA_TRY(cudaMemsetAsync(flags, 0, (size_t)nx * ns, stream));
    if (ns < 3) return D4W_OK;
    int nb1, nb2; peak_level_sizes(ns, nb1, nb2);
    float* bmax = reinterpret_cast<float*>(ws);
    float* bmin = bmax + (size_t)nx * nb1;
    float* smax = bmin + (size_t)nx * nb1;
    float* smin = smax + (size_t)nx * nb2;
    float* rowmin = smin + (size_t)nx * nb2;
    k_peak_levels<<<nx, 256, 0, stream>>>(x, ns, bmax, bmin, smax, smin, rowmin, nb1, nb2);
    D4W_CHECK_LAUNCH("k_peak_levels");
    PeakLevels lv{bmax, bmin, smax, smin, nb1, nb2};
    dim3 grid((ns + 255) / 256, nx);
    k_peak_pick<<<grid, 256, 0, stream>>>(x, ns, lv, rowmin, prominence, flags);
    D4W_CHECK_LAUNCH("k_peak_pick");
    return D4W_OK;
}

// ---------------------------------------------------------------------------------- raw counts -> strain
extern "C" int d4w_raw2strain(const void* raw, int raw_is_int32, int nx, int ns, double scale_factor, float* out, void* stream) {
    if (!raw || !out || nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_raw2strain: bad argument");
    if (raw_is_int32) k_raw2strain<int><<<nx, 512, 0, (cudaStream_t)stream>>>(reinterpret_cast<const int*>(raw), out, ns, scale_factor);
    else k_raw2strain<float><<<nx, 512, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float*>(raw), out, ns, scale_factor);
    D4W_CHECK_LAUNCH("k_raw2strain");
    return D4W_OK;
}
