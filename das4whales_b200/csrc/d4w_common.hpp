// d4w_common.hpp -- error reporting, launch counting and small RAII helpers shared by the
// translation units of libd4w.so.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <string>
#include <vector>
#include "../../include/d4w.h"

namespace d4w {

std::string& last_error_ref();
std::atomic<long long>& launch_counter();

inline int fail(int code, const std::string& msg) { last_error_ref() = msg; return code; }
inline void count_launch(int n = 1) { launch_counter().fetch_add(n, std::memory_order_relaxed); }

#define D4W_CUDA_TRY(expr)                                                                          \
    do {                                                                                            \
        cudaError_t e_ = (expr);                                                                    \
        if (e_ != cudaSuccess) {                                                                    \
            (void)cudaGetLastError(); /* clear the non-sticky error so later CUDA users are not poisoned */ \
            return ::d4w::fail(D4W_ERR_CUDA, std::string(#expr) + " -> " + cudaGetErrorString(e_)); \
        }                                                                                           \
    } while (0)

#define D4W_CHECK_LAUNCH(name)                                                                      \
    do {                                                                                            \
        cudaError_t e_ = cudaGetLastError();                                                        \
        if (e_ != cudaSuccess)                                                                      \
            return ::d4w::fail(D4W_ERR_CUDA, std::string("launch ") + name + " -> " + cudaGetErrorString(e_)); \
        ::d4w::count_launch();                                                                      \
    } while (0)

template <class T>
inline cudaError_t upload(T** dptr, const std::vector<T>& h) {
    *dptr = nullptr;
    size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(T);
    cudaError_t e = cudaMalloc((void**)dptr, bytes);
    if (e != cudaSuccess) return e;
    if (!h.empty()) e = cudaMemcpy(*dptr, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
    return e;
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// Rows per launch of the row kernels, which put one row (or row pair) on each blockIdx.y: gridDim.y <= 65 535.
constexpr int kMaxGridRows = 65535;

// launch(r0, rows) for consecutive blocks of at most `block` rows covering [0, nrows), until one returns an error.  r0 is a
// size_t so that the caller's pointer offsets (r0 * row length) are computed in size_t.
template <class F>
inline int for_row_blocks(int nrows, int block, F&& launch) {
    for (int r0 = 0, rows = 0; r0 < nrows; r0 += rows) {
        rows = std::min(block, nrows - r0);
        if (const int rc = launch((size_t)r0, rows)) return rc;
    }
    return D4W_OK;
}

}  // namespace d4w
