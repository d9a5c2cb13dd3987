// d4w_imageops.cu -- host side of the improcess image operators outside the Gabor path: the Radon transform, the
// bilateral filter and the oriented gradient (C ABI in include/d4w.h; kernels in imageops_kernels.cuh).
#include <string>
#include "d4w_common.hpp"
#include "imageops_kernels.cuh"

using namespace d4w;

namespace {

__global__ void __launch_bounds__(kRadonThreads)
k_radon(RadonParams p) {
    const int bin = blockIdx.y * kRadonThreads + threadIdx.x;
    const int a = blockIdx.x;
    if (bin >= p.n) return;
    p.out[(size_t)bin * p.nangles + a] = radon_ray(p, bin, a);
}

}  // namespace

extern "C" int d4w_radon(const float* img, int h, int w, int n, int pad_r, int pad_c, const double* cs, int nangles, double* out,
                         void* stream_v) {
    if (!img || !cs || !out) return fail(D4W_ERR_ARG, "d4w_radon: null pointer");
    if (h < 1 || w < 1 || nangles < 1) return fail(D4W_ERR_ARG, "d4w_radon: h, w and nangles must be >= 1");
    if (pad_r < 0 || pad_c < 0 || n < 1 || (long long)pad_r + h > n || (long long)pad_c + w > n)
        return fail(D4W_ERR_ARG, "d4w_radon: the image must lie inside the n x n square");
    RadonParams p{img, h, w, n, pad_r, pad_c, cs, nangles, out};
    const dim3 grid((unsigned)nangles, (unsigned)((n + kRadonThreads - 1) / kRadonThreads));
    k_radon<<<grid, kRadonThreads, 0, (cudaStream_t)stream_v>>>(p);
    D4W_CHECK_LAUNCH("k_radon");
    return D4W_OK;
}

extern "C" int d4w_bilateral(const float* in, int h, int w, int is_8u, int radius, double sigma_color, double sigma_space,
                             void* ws, float* out, void* stream_v) {
    if (!in || !out || !ws) return fail(D4W_ERR_ARG, "d4w_bilateral: null pointer");
    if (in == out) return fail(D4W_ERR_ARG, "d4w_bilateral: in-place filtering is not supported");
    if (h < 1 || w < 1) return fail(D4W_ERR_ARG, "d4w_bilateral: h and w must be >= 1");
    if (radius < 1 || radius > kBilMaxRadius)
        return fail(D4W_ERR_ARG, "d4w_bilateral: radius must be in [1, " + std::to_string(kBilMaxRadius) + "]");
    if (!(sigma_color > 0.0) || !(sigma_space > 0.0)) return fail(D4W_ERR_ARG, "d4w_bilateral: sigmas must be > 0");
    const dim3 grid((unsigned)((w + kBilTX - 1) / kBilTX), (unsigned)((h + kBilTY - 1) / kBilTY));
    if (grid.y > 65535) return fail(D4W_ERR_ARG, "d4w_bilateral: image too tall");
    cudaStream_t st = (cudaStream_t)stream_v;
    unsigned* mm = static_cast<unsigned*>(ws);
    float* lut = reinterpret_cast<float*>(static_cast<char*>(ws) + 16);
    const size_t n = (size_t)h * w;
    if (!is_8u) {
        k_minmax_init<<<1, 1, 0, st>>>(mm);
        D4W_CHECK_LAUNCH("k_minmax_init");
        k_minmax<<<(unsigned)std::min<size_t>((n + 255) / 256, 2048), 256, 0, st>>>(in, n, mm);
        D4W_CHECK_LAUNCH("k_minmax");
    }
    k_bilateral_lut<<<1, 256, 0, st>>>(mm, is_8u ? 1 : 0, -0.5 / (sigma_color * sigma_color), lut);
    D4W_CHECK_LAUNCH("k_bilateral_lut");
    const size_t smem = bilateral_smem_bytes(radius, is_8u ? 1 : 0);
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_bilateral, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bilateral_smem_bytes(kBilMaxRadius, 0)));
    k_bilateral<<<grid, kBilThreads, smem, st>>>(in, h, w, radius, -0.5 / (sigma_space * sigma_space), is_8u ? 1 : 0, lut, out);
    D4W_CHECK_LAUNCH("k_bilateral");
    return D4W_OK;
}

extern "C" int d4w_grad_oriented(const float* in, int h, int w, int dft, int dfx, float* out, void* stream_v) {
    if (!in || !out) return fail(D4W_ERR_ARG, "d4w_grad_oriented: null pointer");
    if (h < 1 || w < 1) return fail(D4W_ERR_ARG, "d4w_grad_oriented: h and w must be >= 1");
    if (dft < 0 || dfx < 0 || (dft == 0 && dfx == 0))
        return fail(D4W_ERR_ARG, "d4w_grad_oriented: direction must be two shifts >= 0, not both 0");
    const int oh = dfx == 0 ? h : dft == 0 ? h - dfx : h - 2 * dfx;
    const int ow = w - dft;
    if (oh < 1 || ow < 1) return fail(D4W_ERR_ARG, "d4w_grad_oriented: the shifts leave no output");
    const size_t n = (size_t)oh * ow;
    k_grad_oriented<<<(unsigned)std::min<size_t>((n + 255) / 256, 4096), 256, 0, (cudaStream_t)stream_v>>>(in, w, dft, dfx, oh, ow, out);
    D4W_CHECK_LAUNCH("k_grad_oriented");
    return D4W_OK;
}
