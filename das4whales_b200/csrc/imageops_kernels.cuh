// imageops_kernels.cuh -- device side of the image operators of improcess that the Gabor path does not use
// (reference: src/das4whales/improcess.py under /root/reference/):
//   :347  compute_radon_transform = skimage.transform.radon(image, theta, circle=False)  -> k_radon (radon_ray)
//   :319  bilateral_filter = cv2.bilateralFilter, 8U and 32F single-channel             -> k_bilateral_lut, k_bilateral
//   :143  gradient_oriented, the three slicing branches                                  -> k_grad_oriented
// gaussian_filter and the two diagonal-edge operators are d4w_filter2d passes (image_kernels.cuh).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <cstdint>
#include "image_kernels.cuh"      // k_minmax, ord2f, reflect101

namespace d4w {

// ---------------------------------------------------------------------------------- Radon transform
// skimage pads the image into an n x n zero square and, for each angle, warps it with the inverse map
//   x = cos * col + sin * row - c (cos + sin - 1),   y = -sin * col + cos * row - c (cos - sin - 1),   c = n / 2
// (order-1 bilinear, zero outside, no clipping), then sums every column of the warped image: bin `col` is the sum over
// `row` of the bilinear sample at (y, x).  The padding is zero, so a sample contributes only when one of its four
// neighbours lies in the unpadded image: each ray is clipped analytically to those rows (with one row of margin, the
// samples themselves still test their neighbours), and only the unpadded image is read.  Coordinates and the sum are in
// double: at n ~ 17 000 a float coordinate is off by ~1e-3 pixel.
struct RadonParams {
    const float* img;            // [h][w], the unpadded image
    int h, w, n, pad_r, pad_c;   // the image sits at rows [pad_r, pad_r + h), columns [pad_c, pad_c + w) of the square
    const double* cs;            // [nangles][2] = (cos, sin)
    int nangles;
    double* out;                 // [n][nangles]
};

// narrow [lo, hi] to the rows r with e0 < k r + x0 < e1
__host__ __device__ inline void radon_clip(double k, double x0, double e0, double e1, double& lo, double& hi) {
    if (k == 0.0) {
        if (!(x0 > e0 && x0 < e1)) { lo = 1.0; hi = 0.0; }
        return;
    }
    double a = (e0 - x0) / k, b = (e1 - x0) / k;
    if (a > b) { const double t = a; a = b; b = t; }
    lo = a > lo ? a : lo;
    hi = b < hi ? b : hi;
}

__host__ __device__ inline float radon_px(const float* __restrict__ img, int h, int w, int y, int x) {
    return (y >= 0 && y < h && x >= 0 && x < w) ? img[(size_t)y * w + x] : 0.f;
}

// the ray sum of detector bin `bin` at angle `a`
__host__ __device__ inline double radon_ray(const RadonParams& p, int bin, int a) {
    const double co = p.cs[2 * a], si = p.cs[2 * a + 1];
    const double c = (double)(p.n / 2);
    // the sample of row r lies at x = si r + x0, y = co r + y0 in the coordinates of the unpadded image
    const double x0 = co * bin - c * (co + si - 1.0) - p.pad_c;
    const double y0 = -si * bin - c * (co - si - 1.0) - p.pad_r;
    double lo = 0.0, hi = (double)(p.n - 1);
    radon_clip(si, x0, -1.0, (double)p.w, lo, hi);
    radon_clip(co, y0, -1.0, (double)p.h, lo, hi);
    if (!(lo <= hi)) return 0.0;
    const int r0 = (int)floor(lo) - 1 > 0 ? (int)floor(lo) - 1 : 0;
    const int r1 = (int)ceil(hi) + 1 < p.n - 1 ? (int)ceil(hi) + 1 : p.n - 1;
    double acc = 0.0;
#pragma unroll 4
    for (int r = r0; r <= r1; ++r) {
        const double x = fma(si, (double)r, x0), y = fma(co, (double)r, y0);
        const double fx = floor(x), fy = floor(y);
        const int ix = (int)fx, iy = (int)fy;
        const float dx = (float)(x - fx), dy = (float)(y - fy);
        // skimage takes the far neighbour at ceil(); at an integer coordinate its weight is 0 either way
        const float tl = radon_px(p.img, p.h, p.w, iy, ix), tr = radon_px(p.img, p.h, p.w, iy, ix + 1);
        const float bl = radon_px(p.img, p.h, p.w, iy + 1, ix), br = radon_px(p.img, p.h, p.w, iy + 1, ix + 1);
        const float top = (1.f - dx) * tl + dx * tr, bot = (1.f - dx) * bl + dx * br;
        acc += (double)((1.f - dy) * top + dy * bot);
    }
    return acc;
}

constexpr int kRadonThreads = 128;

// ---------------------------------------------------------------------------------- bilateral filter
// cv2.bilateralFilter for one channel (OpenCV imgproc/src/bilateral_filter.dispatch.cpp, restated): taps (i, j) with
// sqrt(i^2 + j^2) <= radius, space weight (float) exp(-(i^2 + j^2) / (2 sigma_space^2)), border BORDER_REFLECT_101;
// out = sum(v w) / sum(w), w = space weight * colour weight, summed in float in tap order (i outer, j inner).
//   8U : colour weight lut[|v - v0|] with lut[i] = (float) exp(-i^2 / (2 sigma_color^2)), i < 256; the result is
//        rounded to nearest (even) and saturated to 0..255.
//   32F: scale = (float) 4096 / (max - min) of the whole image; lut[i] = (float) exp(-(i / scale)^2 / (2 sigma_color^2)),
//        i < 4098, entries after the first 0 kept 0; colour weight = lut[k] + f (lut[k + 1] - lut[k]) with
//        k + f = |v - v0| scale; an image with max - min < FLT_EPSILON gets colour weight 1 at every tap.
constexpr int kBilLut32 = 4096 + 2;
// 32 x 8 threads, eight rows each: a CTA stages the colour table (16 KB for 32F) once per 2 048 outputs; at radius 64 the
// table, the space weights and the tile take 201 KB of shared memory
constexpr int kBilTX = 32, kBilTY = 64, kBilThreads = 256;
constexpr int kBilMaxRadius = 64;

// mm: the image's min / max in the ordered-uint encoding of k_minmax (32F only)
static __global__ void __launch_bounds__(256)
k_bilateral_lut(const unsigned* __restrict__ mm, int is8u, double color_coeff, float* __restrict__ lut) {
    const int n = is8u ? 256 : kBilLut32;
    float scale = 0.f;
    if (!is8u) {
        const double lo = ord2f(mm[0]), hi = ord2f(mm[1]);
        // a range below FLT_EPSILON (a constant image) weighs every tap's colour by 1, as cv2 does
        scale = fabs(lo - hi) < 1.1920928955078125e-07 ? 0.f : (float)((double)(kBilLut32 - 2) / (hi - lo));
        if (threadIdx.x == 0) lut[n] = scale;                              // read back by k_bilateral
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (is8u) {
            lut[i] = (float)exp((double)(i * i) * color_coeff);
        } else if (scale == 0.f) {
            lut[i] = i == 0 ? 1.f : 0.f;
        } else {
            const double v = (double)((float)i / scale);
            lut[i] = (float)exp(v * v * color_coeff);
        }
    }
}

static __global__ void __launch_bounds__(kBilThreads)
k_bilateral(const float* __restrict__ in, int h, int w, int radius, double space_coeff, int is8u, const float* __restrict__ lut, float* __restrict__ out) {
    extern __shared__ __align__(16) float bsm[];
    const int d = 2 * radius + 1;
    const int tw = kBilTX + 2 * radius, th = kBilTY + 2 * radius;
    const int nlut = is8u ? 256 : kBilLut32;
    float* sW = bsm;                       // [d][d] space weights, -1 outside the circle
    float* sL = sW + d * d;                // [nlut] colour table
    float* sI = sL + nlut;                 // [th][tw] tile with halo
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * kBilTX, y0 = blockIdx.y * kBilTY;
    const float scale = is8u ? 0.f : lut[nlut];
    for (int i = tid; i < d * d; i += kBilThreads) {
        const int dy = i / d - radius, dx = i % d - radius;
        const double r = sqrt((double)dy * dy + (double)dx * dx);
        sW[i] = r > radius ? -1.f : (float)exp(r * r * space_coeff);
    }
    for (int i = tid; i < nlut; i += kBilThreads) sL[i] = lut[i];
    for (int i = tid; i < th * tw; i += kBilThreads) {
        const int ty = i / tw, tx = i - ty * tw;
        sI[i] = in[(size_t)reflect101(y0 + ty - radius, h) * w + reflect101(x0 + tx - radius, w)];
    }
    __syncthreads();
    const int cx = tid % kBilTX, cy = tid / kBilTX;
#pragma unroll 1
    for (int rr = 0; rr < kBilTY / 8; ++rr) {
        const int ly = cy + rr * 8;
        const int y = y0 + ly, x = x0 + cx;
        if (y >= h || x >= w) continue;
        const float v0 = sI[(ly + radius) * tw + cx + radius];
        float sum = 0.f, wsum = 0.f;
        for (int i = 0; i < d; ++i) {
            const float* row = sI + (ly + i) * tw + cx;
            const float* wrow = sW + i * d;
            for (int j = 0; j < d; ++j) {
                const float sw = wrow[j];
                if (sw < 0.f) continue;
                const float v = row[j];
                float cw;
                if (is8u) {
                    cw = sL[abs((int)v - (int)v0)];
                } else {
                    float alpha = fabsf(v - v0) * scale;
                    const int k = (int)floorf(alpha);
                    alpha -= (float)k;
                    cw = sL[k] + alpha * (sL[k + 1] - sL[k]);
                }
                const float wt = sw * cw;
                sum += v * wt;
                wsum += wt;
            }
        }
        float r = sum / wsum;
        if (is8u) r = fminf(fmaxf((float)__float2int_rn(r), 0.f), 255.f);
        out[(size_t)y * w + x] = r;
    }
}

__host__ inline size_t bilateral_smem_bytes(int radius, int is8u) {
    const size_t d = 2 * (size_t)radius + 1;
    return (d * d + (is8u ? 256 : kBilLut32) + (size_t)(kBilTY + 2 * radius) * (kBilTX + 2 * radius)) * sizeof(float);
}

// ---------------------------------------------------------------------------------- oriented gradient
// improcess.gradient_oriented(image, (dft, dfx)) with dft, dfx >= 0, not both 0; output [oh][ow]:
//   dfx = 0: out[i][j] = -(x[i][j] - x[i][j + dft])                                        [h][w - dft]
//   dft = 0: out[i][j] = -(x[i + dfx][j] - x[i][j])                                        [h - dfx][w]
//   else   : out[i][j] = -(x[i + dfx][j] - 0.5 x[i + 2 dfx][j + dft] - 0.5 x[i][j + dft])  [h - 2 dfx][w - dft]
static __global__ void __launch_bounds__(256)
k_grad_oriented(const float* __restrict__ in, int w, int dft, int dfx, int oh, int ow, float* __restrict__ out) {
    const size_t n = (size_t)oh * ow;
    for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < n; o += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(o / ow), j = (int)(o - (size_t)i * ow);
        float g;
        if (dfx == 0) g = -(in[(size_t)i * w + j] - in[(size_t)i * w + j + dft]);
        else if (dft == 0) g = -(in[(size_t)(i + dfx) * w + j] - in[(size_t)i * w + j]);
        else g = -((in[(size_t)(i + dfx) * w + j] - 0.5f * in[(size_t)(i + 2 * dfx) * w + j + dft]) - 0.5f * in[(size_t)i * w + j + dft]);
        out[o] = g;
    }
}

}  // namespace d4w
