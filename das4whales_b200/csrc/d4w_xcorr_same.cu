// d4w_xcorr_same.cu -- the "same"-mode matched filter (C ABI in include/d4w.h): the k_xcorr* kernels instantiated with
// SAME = true, in their own translation unit (see xcorr_launch.cuh).
#include "xcorr_launch.cuh"

using namespace d4w;

extern "C" int d4w_xcorr_same(d4w_fft_plan* p, const float* x, int nx, int ns, int valid, int lag0, int ntpl, const void* dev_tabs,
                              const float* dev_rowmax, float* out, void* stream) {
    if (!p || !x || !dev_tabs || !dev_rowmax || !out) return fail(D4W_ERR_ARG, "d4w_xcorr_same: null argument");
    if (nx < 1 || nx > 65535 || ns < 1) return fail(D4W_ERR_ARG, "d4w_xcorr_same: need 1 <= nx <= 65535 rows and ns >= 1");
    if (valid < 1 || valid > p->n || ntpl < 1) return fail(D4W_ERR_ARG, "d4w_xcorr_same: bad valid / ntpl");
    // the longest (prepended) template has >= lag0 + 1 taps, so valid = nb - L + 1 <= nb - lag0
    if (lag0 < 0 || lag0 > p->n - valid) return fail(D4W_ERR_ARG, "d4w_xcorr_same: lag0 must be in [0, nb - valid]");
    return xcorr_launch<true>(p, x, nx, ns, valid, ntpl, dev_tabs, nullptr, nullptr, nullptr, dev_rowmax, lag0, out, stream);
}
