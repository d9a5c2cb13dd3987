// d4w_image.cu -- host side of the image-domain ("Gabor") detector kernels, pick compaction and the instantaneous
// frequency helper (C ABI in include/d4w.h; kernels in image_kernels.cuh).
#include <cmath>
#include <cstdint>
#include "d4w_common.hpp"
#include "image_kernels.cuh"

using namespace d4w;

// grid-stride kernels: at most `per_sm` CTAs per SM of the current device
static inline unsigned grid1d(size_t n, int threads, unsigned per_sm = 16) {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) {
        (void)cudaGetLastError();
        sms = 1;
    }
    const size_t b = (n + threads - 1) / threads;
    return (unsigned)std::max<size_t>(1, std::min<size_t>(b, (size_t)sms * per_sm));
}

extern "C" int d4w_scale_pixels(const float* x, float* y, size_t n, float mul, void* dev_ws8, void* stream_v) {
    if (!x || !y || !dev_ws8 || n < 1) return fail(D4W_ERR_ARG, "d4w_scale_pixels: bad argument");
    cudaStream_t stream = (cudaStream_t)stream_v;
    unsigned* mm = reinterpret_cast<unsigned*>(dev_ws8);
    k_minmax_init<<<1, 1, 0, stream>>>(mm);
    D4W_CHECK_LAUNCH("k_minmax_init");
    k_minmax<<<grid1d(n, 256), 256, 0, stream>>>(x, n, mm);
    D4W_CHECK_LAUNCH("k_minmax");
    k_scale_pixels<<<grid1d(n, 256, 32), 256, 0, stream>>>(x, y, n, mm, mul);
    D4W_CHECK_LAUNCH("k_scale_pixels");
    return D4W_OK;
}

extern "C" int d4w_db_re_max(const float* x, float* y, size_t n, void* dev_ws8, void* stream_v) {
    if (!x || !y || !dev_ws8 || n < 1) return fail(D4W_ERR_ARG, "d4w_db_re_max: bad argument");
    cudaStream_t stream = (cudaStream_t)stream_v;
    unsigned* mm = reinterpret_cast<unsigned*>(dev_ws8);
    k_minmax_init<<<1, 1, 0, stream>>>(mm);
    D4W_CHECK_LAUNCH("k_minmax_init");
    k_minmax<<<grid1d(n, 256), 256, 0, stream>>>(x, n, mm);
    D4W_CHECK_LAUNCH("k_minmax");
    k_db_re_max<<<grid1d(n, 256, 32), 256, 0, stream>>>(x, y, n, mm);
    D4W_CHECK_LAUNCH("k_db_re_max");
    return D4W_OK;
}

extern "C" int d4w_resize_aa(const float* in, int ih, int iw, float* out, int oh, int ow, float* dev_tmp, void* stream_v) {
    if (!in || !out || !dev_tmp || ih < 1 || iw < 1 || oh < 1 || ow < 1) return fail(D4W_ERR_ARG, "d4w_resize_aa: bad argument");
    if (ih > 65535 || oh > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_resize_aa: more than 65535 rows");
    cudaStream_t stream = (cudaStream_t)stream_v;
    dim3 gh((ow + 255) / 256, ih);
    k_resize_aa_h<<<gh, 256, 0, stream>>>(in, ih, iw, dev_tmp, ow);          // [ih][iw] -> [ih][ow]
    D4W_CHECK_LAUNCH("k_resize_aa_h");
    dim3 gv((ow + 255) / 256, oh);
    k_resize_aa_v<<<gv, 256, 0, stream>>>(dev_tmp, ih, ow, out, oh);          // [ih][ow] -> [oh][ow]
    D4W_CHECK_LAUNCH("k_resize_aa_v");
    return D4W_OK;
}

extern "C" int d4w_filter2d(const float* in, int h, int w, const float* dev_K, int kh, int kw, float in_thr, float out_thr,
                            int border, float* out, void* stream_v) {
    if (!in || !dev_K || !out || h < 1 || w < 1 || kh < 1 || kw < 1) return fail(D4W_ERR_ARG, "d4w_filter2d: bad argument");
    if (in == out) return fail(D4W_ERR_ARG, "d4w_filter2d: in-place filtering is not supported");
    if (border != 0 && border != 1) return fail(D4W_ERR_ARG, "d4w_filter2d: border must be 0 (reflect-101) or 1 (zeros)");
    const int kwp = (kw + 3) & ~3;
    const size_t smem = ((size_t)kh * kwp + (size_t)(FT_TY + kh - 1) * (FT_TX + kwp)) * sizeof(float);
    if (smem > 220 * 1024) return fail(D4W_ERR_UNSUPPORTED, "d4w_filter2d: kernel too large for shared memory (about 140 x 140 taps)");
    D4W_CUDA_TRY(cudaFuncSetAttribute(k_filter2d, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    dim3 grid((w + FT_TX - 1) / FT_TX, (h + FT_TY - 1) / FT_TY);
    if (grid.y > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_filter2d: image too tall");
    k_filter2d<<<grid, FT_THREADS, smem, (cudaStream_t)stream_v>>>(in, h, w, dev_K, kh, kw, in_thr, out_thr, border, out);
    D4W_CHECK_LAUNCH("k_filter2d");
    return D4W_OK;
}

extern "C" int d4w_mask_upsample_mul(const float* trace, int nx, int ns, const float* mask, int mh, int mw, float* out,
                                     unsigned char* mask_out, void* stream_v) {
    if (!mask || (!out && !mask_out) || (out && !trace) || nx < 1 || ns < 1 || mh < 1 || mw < 1)
        return fail(D4W_ERR_ARG, "d4w_mask_upsample_mul: bad argument");
    if (nx > 65535) return fail(D4W_ERR_UNSUPPORTED, "d4w_mask_upsample_mul: more than 65535 rows per call");
    if (mh > nx || mw > ns) return fail(D4W_ERR_ARG, "d4w_mask_upsample_mul: the mask must not be larger than the trace (upsampling only)");
    dim3 grid((ns + 255) / 256, nx);
    k_mask_upsample_mul<<<grid, 256, 0, (cudaStream_t)stream_v>>>(trace, nx, ns, mask, mh, mw, out, mask_out);
    D4W_CHECK_LAUNCH("k_mask_upsample_mul");
    return D4W_OK;
}

extern "C" int d4w_inst_freq(const float* x, const float* hx, int n, double fs, float* out, void* stream_v) {
    if (!x || !hx || !out || n < 2) return fail(D4W_ERR_ARG, "d4w_inst_freq: bad argument");
    k_inst_freq<<<(n - 1 + 255) / 256, 256, 0, (cudaStream_t)stream_v>>>(x, hx, n, fs, out);
    D4W_CHECK_LAUNCH("k_inst_freq");
    return D4W_OK;
}

extern "C" int d4w_peaks_offsets(const unsigned char* flags, int nx, int ns, int* dev_counts, int* dev_offsets, void* stream_v) {
    if (!flags || !dev_counts || !dev_offsets || nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_peaks_offsets: bad argument");
    cudaStream_t stream = (cudaStream_t)stream_v;
    k_peaks_count<<<nx, 256, 0, stream>>>(flags, ns, dev_counts);
    D4W_CHECK_LAUNCH("k_peaks_count");
    k_scan_offsets<<<1, 1024, 0, stream>>>(dev_counts, nx, dev_offsets);
    D4W_CHECK_LAUNCH("k_scan_offsets");
    return D4W_OK;
}

extern "C" int d4w_peaks_fill(const unsigned char* flags, int nx, int ns, const int* dev_offsets, int* dev_idx, void* stream_v) {
    if (!flags || !dev_offsets || !dev_idx || nx < 1 || ns < 1) return fail(D4W_ERR_ARG, "d4w_peaks_fill: bad argument");
    k_peaks_fill<<<nx, 256, 0, (cudaStream_t)stream_v>>>(flags, ns, dev_offsets, dev_idx);
    D4W_CHECK_LAUNCH("k_peaks_fill");
    return D4W_OK;
}
