// plan_k2pos.cuh -- the bin -> position map of a d4w_fft_plan's own forward stages, for the kernels that run
// fft_forward_stages on the plan and read bins through it (k_welch in d4w_welch.cu, k_csd in d4w_csd.cu).  Host code only;
// kept out of xcorr_launch.cuh so that the translation units which include that header alone do not change.
#pragma once
#include <map>
#include <mutex>
#include <vector>
#include "xcorr_launch.cuh"

namespace d4w {

// The plan's d_k2pos inverts its pos2k, which for the prime-factor length (p->pfa, n = 2520) is the matched filter's
// Good-Thomas map, not the map of p->pl: for that length a table of p->pl's own map is built once per device and kept for
// the life of the process (one 10 KB table per device).
inline cudaError_t welch_k2pos(const d4w_fft_plan* p, const int** out) {
    if (!p->pfa) { *out = p->d_k2pos; return cudaSuccess; }
    static std::mutex mu;
    static std::map<int, int*> tables;
    std::lock_guard<std::mutex> lock(mu);
    int*& t = tables[p->device];
    if (!t) {
        const std::vector<int> p2k = make_pos2freq(p->pl);
        std::vector<int> k2pos(p2k.size());
        for (size_t i = 0; i < p2k.size(); ++i) k2pos[p2k[i]] = (int)i;
        const cudaError_t e = upload(&t, k2pos);
        if (e != cudaSuccess) { cudaFree(t); t = nullptr; return e; }
    }
    *out = t;
    return cudaSuccess;
}

}  // namespace d4w
