/* d4w.h -- C ABI of libd4w.so, the H100-native (sm_90a) replacement for the channel-parallel
 * DSP hot path of DAS4Whales.
 *
 * The reference has no FFI: its boundary is the Python module namespace
 * (`das4whales.dsp.*`, `das4whales.detect.*`).  Each entry point below names the reference
 * function(s) whose arithmetic it replaces (file:line under /root/reference/src/das4whales/).
 * das4whales_b200/{dsp,detect}.py keep the reference signatures and call these through cffi
 * (ABI mode; the block between D4W_CDEF_BEGIN / D4W_CDEF_END is fed to ffi.cdef verbatim).
 *
 * Conventions: plain pointers and sizes only; every `dev_` pointer is CUDA device memory on
 * the plan's device; `stream` is a cudaStream_t passed as void* (NULL = legacy default
 * stream); all calls are asynchronous on `stream` unless stated; the return value is a
 * d4w_status (0 = ok) and d4w_last_error() gives the message for the calling thread.
 * There is no CPU fallback anywhere behind this interface.
 */
#ifndef D4W_H
#define D4W_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* D4W_CDEF_BEGIN */
typedef struct d4w_fk_plan d4w_fk_plan;
typedef struct d4w_fk_mask d4w_fk_mask;

enum {
    D4W_OK = 0,
    D4W_ERR_ARG = 1,          /* bad shape / null pointer / inconsistent arguments        */
    D4W_ERR_UNSUPPORTED = 2,  /* FFT length with a prime factor > 61, matrix too large ... */
    D4W_ERR_CUDA = 3,         /* a CUDA runtime call failed (message has the cudaError)    */
    D4W_ERR_NCCL = 4
};

const char* d4w_last_error(void);
int d4w_version(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches) */
long long d4w_launch_count(void);

/* ---- f-k filter: dsp.fk_filter_filt (dsp.py:725-756), dsp.fk_filter_sparsefilt (:759-786),
 *      dsp.taper_data (:705-722) ------------------------------------------------------- */
/* Plan for an [nx channels] x [ns samples] float32 strain matrix on CUDA device `device`. */
int d4w_fk_plan_create(d4w_fk_plan** out, int nx, int ns, int device);
int d4w_fk_plan_destroy(d4w_fk_plan* plan);
/* describe the plan: info[0]=T1 (row split), [1]=T2, [2]=column tile width in samples,
 * [3]=column stages, [4]=row stages, [5]=column threads, [6]=row threads,
 * [7]=column scheme: 0 single-level cp.async, 1 single-level TMA, 2 two-level (X1 in registers, X2 fused two-stage),
 *      3 two-level as one pipelined launch per direction (intermediate kept in L2),
 *      4 chirp-z single-level (nx with a prime factor > 61, nx <= 12 800; [3] counts the stages of the M-point transform) */
int d4w_fk_plan_info(const d4w_fk_plan* plan, int* info8);
/* profiling aid (plan created with env D4W_FK_DEBUG=1): summed SM cycles per phase of the TMA column
 * kernels since the last call -- [0..2] forward: load wait, FFT, untangle+store; [4..7] inverse: store
 * drain, fill, FFT, store issue.  Synchronises the device. */
int d4w_fk_debug_phases(d4w_fk_plan* plan, unsigned long long* host8);

/* Mask descriptors.  All masks are defined exactly as the reference defines them, in the
 * fftshift-ed (k, f) layout; the library folds M_sym = (M[k,f] + M[-k,-f]) / 2 (what taking
 * `.real` at dsp.py:756 amounts to), drops wavenumber rows whose folded mask is identically
 * zero, scales by 1/(nx*ns) and stores the result in transform order.
 *
 * fan: dsp.fk_filter_design (dsp.py:85-171).  kval / fval are numpy's fftfreq steps
 * 1/(nx*step*dx) and 1/(ns*(1/fs)) computed by the caller in double. */
int d4w_fk_mask_create_fan(d4w_fk_mask** out, d4w_fk_plan* plan, double kval, double fval,
                           double cs_min, double cp_min, double cp_max, double cs_max);
/* hybrid_ninf: dsp.hybrid_ninf_filter_design (dsp.py:308-454).  host_H = the ns-long column
 * profile built at :348-349 (host pointer, copied); col_lo/col_hi = the column range of
 * :359-360,:376. */
int d4w_fk_mask_create_hybrid_ninf(d4w_fk_mask** out, d4w_fk_plan* plan, double kval, double fval,
                                   double cs_min, double cp_min, double cp_max, double cs_max,
                                   const double* host_H, int col_lo, int col_hi);
/* dense: any [nx x ns] mask in the reference's shifted layout, C-order float32 on the device
 * (design functions without a closed form here, user-made masks).  Synchronises `stream`
 * once to read back the row support. */
int d4w_fk_mask_create_dense(d4w_fk_mask** out, d4w_fk_plan* plan, const float* dev_mask_shifted,
                             void* stream);
int d4w_fk_mask_destroy(d4w_fk_mask* mask);
/* Opt-in approximate pruning: recompute the row support keeping only wavenumber rows whose folded mask exceeds eps
 * somewhere (eps = 0: the exact default).  hybrid_* masks carry Butterworth tails <= 8e-6 at every wavenumber
 * (dsp.py:372), so nothing is prunable exactly; eps = 1e-5 keeps the speed band only.  The output error is bounded by
 * eps * ||x||_2 in the l2 norm.  Must be followed by d4w_fk_mask_table_bytes / d4w_fk_mask_build.  Synchronises. */
int d4w_fk_mask_prune(d4w_fk_mask* mask, double eps, void* stream);
/* rows of the half wavenumber plane (0..nx/2) kept after support pruning */
int d4w_fk_mask_rows(const d4w_fk_mask* mask);
/* bytes of device memory the caller must provide for the transform-order table */
size_t d4w_fk_mask_table_bytes(const d4w_fk_mask* mask);
/* fill the caller's table (kept by reference until the mask is destroyed) */
int d4w_fk_mask_build(d4w_fk_mask* mask, float* dev_table, void* stream);
/* materialise the mask exactly as the reference function returns it: float64 [nx x ns],
 * shifted layout, C order, into device memory (analytic kinds only) */
int d4w_fk_mask_materialize(const d4w_fk_mask* mask, double* dev_out, void* stream);

/* bytes of workspace (pruned complex spectrum) the caller must provide for d4w_fk_apply */
size_t d4w_fk_workspace_bytes(const d4w_fk_plan* plan, const d4w_fk_mask* mask);
/* y = real(ifft2(ifftshift(fftshift(fft2(x)) * M))) with optional Tukey(alpha=0.03) taper
 * applied to x first (taper != 0; x itself is not modified).  x, y: float32 [nx x ns],
 * C order, device memory; y may alias x. */
int d4w_fk_apply(d4w_fk_plan* plan, d4w_fk_mask* mask, const float* dev_x, float* dev_y,
                 void* dev_workspace, int taper, void* stream);
/* the five passes, separately (bench / profiling): pass = 1..5 */
int d4w_fk_apply_pass(d4w_fk_plan* plan, d4w_fk_mask* mask, const float* dev_x, float* dev_y,
                      void* dev_workspace, int taper, int pass, void* stream);
/* sharded variant (one matrix over several GPUs, das4whales_b200/dist.py): `plan` gives the local
 * geometry -- passes 1/5 on a time slab [nx][plan.ns] starting at global sample t_offset with all kept
 * rows; passes 2-4 on kept rows [slot_begin, slot_begin+slot_count) over the full time axis, the
 * workspace pointing at the first local row.  The mask is the one of the full matrix. */
int d4w_fk_apply_pass_ex(d4w_fk_plan* plan, d4w_fk_mask* mask, const float* dev_x, float* dev_y,
                         void* dev_workspace, int taper, int pass, int slot_begin, int slot_count,
                         int t_offset, void* stream);

/* ---- generic shared-memory FFT plan (matched-filter blocks, STFT frames) ----------------- */
typedef struct d4w_fft_plan d4w_fft_plan;
typedef struct d4w_row_plan d4w_row_plan;
int d4w_fft_plan_create(d4w_fft_plan** out, int n, int device);
int d4w_fft_plan_destroy(d4w_fft_plan* plan);
/* host_pos2freq[p] = DFT bin stored at position p after the forward transform (n ints) */
int d4w_fft_plan_order(const d4w_fft_plan* plan, int* host_pos2freq);
/* frequency index of each entry of the multiplier tables d4w_xcorr expects (the plan's transform order, regrouped
 * so that the fused last stage reads them coalesced) */
int d4w_fft_plan_table_order(const d4w_fft_plan* plan, int* host_tab2freq);

/* ---- row statistics: np.mean / np.max(np.abs) / np.std(axis=1) used by
 *      detect.compute_cross_correlogram (detect.py:157) and dsp.snr_tr_array (dsp.py:975-976).
 *      dev_stats: double[nx][4] = {mean, absmax, population variance, 0}.  dev_segpre (optional):
 *      double[nx][ceil(ns/seglen)], prefix sums of the normalised row at segment starts. */
int d4w_row_stats(const float* dev_x, int nx, int ns, int seglen, double* dev_stats, double* dev_segpre,
                  void* stream);
/* dsp.snr_tr_array(trace, env=False) (dsp.py:976): 10*log10(x^2 / var_row) */
int d4w_snr(const float* dev_x, float* dev_out, int nx, int ns, const double* dev_stats, void* stream);

/* ---- matched filter: detect.compute_cross_correlogram / shift_xcorr (detect.py:96-166) as
 *      overlap-save FFT correlation; `plan` = fft plan of the block length nb, `valid` = nb - L + 1
 *      lags kept per block.  dev_tabs: ntpl x nb complex64 = conj(FFT_nb(template_t)) / (nb * m_t) in
 *      the plan's table order (d4w_fft_plan_table_order).  With dev_stats != NULL rows are demeaned / peak-normalised and
 *      the mean-of-padded-template term mu_t/m_t * prefix is added (dev_mu_over_m: double[ntpl]).
 *      dev_out: float32 [ntpl][nx][ns]. */
int d4w_xcorr(d4w_fft_plan* plan, const float* dev_x, int nx, int ns, int valid, int ntpl, const void* dev_tabs,
              const double* dev_mu_over_m, const double* dev_stats, const double* dev_segpre, float* dev_out,
              void* stream);
/* ---- "same"-mode matched filter: scipy.signal.correlate(x / max(x), c_t, 'same') of every row with each template
 *      (scripts/main_gabordetect.py:243-246), on the same overlap-save blocks as d4w_xcorr:
 *      out[t][row][i] = sum_n x[row][i - lag0 + n] c'_t[n] / rowmax[row], x = 0 outside [0, ns), where c'_t is template t with
 *      lag0 - floor(L_t / 2) zeros prepended (lag0 = max_t floor(L_t / 2)).  dev_tabs: ntpl x nb complex64 =
 *      conj(FFT_nb(c'_t)) / nb in d4w_fft_plan_table_order; valid = nb - max_t len(c'_t) + 1.  dev_rowmax: float[nx] from
 *      d4w_row_max (clamped at 0); rows with !(rowmax > 0) are written as zeros.  1 <= nx <= 65535.
 *      dev_out: float32 [ntpl][nx][ns]. */
int d4w_xcorr_same(d4w_fft_plan* plan, const float* dev_x, int nx, int ns, int valid, int lag0, int ntpl, const void* dev_tabs,
                   const float* dev_rowmax, float* dev_out, void* stream);

/* ---- Hilbert envelope |scipy.signal.hilbert(x, axis=1)| (detect.py:192) and
 *      dsp.snr_tr_array(trace, env=True) (dsp.py:975).  mode 0: envelope, 1: 10*log10(env^2/var).
 *      dev_out must not overlap dev_x (long rows are transformed two per complex FFT and dev_x is read again at the end).
 *      d4w_xcorr's dev_tabs are in d4w_fft_plan_table_order.
 *      Any ns up to 128 000 is accepted: a length with no T1 x T2 split (a prime factor > 61) is transformed by a chirp-z
 *      convolution of length czt_m = T1 * T2 ~ 2 ns.  d4w_row_plan_info reports the split and czt_m (0: direct transform);
 *      d4w_row_workspace_bytes sizes the workspace for nx rows of the chosen route. */
int d4w_row_plan_create(d4w_row_plan** out, int ns, int device);
int d4w_row_plan_destroy(d4w_row_plan* plan);
size_t d4w_row_workspace_bytes(const d4w_row_plan* plan, int nx);
int d4w_row_plan_info(const d4w_row_plan* plan, int* t1, int* t2, int* czt_m);
int d4w_hilbert(d4w_row_plan* plan, const float* dev_x, float* dev_out, int nx, void* dev_workspace, int mode,
                const double* dev_stats, void* stream);
/* Envelope and moment statistics of a row window (scripts/main_bathynoise.py:183-189, :257-259).  Row r is the n samples at
 * dev_x + r * ld (ld >= n), n = the row plan's length (any n up to 128 000, as d4w_hilbert).  out: double[nrows][5] =
 * {median |hilbert(x)|, mean |hilbert(x)|, mean x, mean x^2, population variance of x}; a row of variance 0 is constant and
 * gets the envelope statistics |mean x| exactly (0 for a zero channel).
 * dev_workspace: d4w_env_stats_workspace_bytes(plan, nrows, ld) bytes (the envelope of up to 65 535 rows, and a dense copy of
 * the window when ld != n).  Any nrows >= 1. */
size_t d4w_env_stats_workspace_bytes(const d4w_row_plan* plan, int nrows, size_t ld);
int d4w_env_stats(d4w_row_plan* plan, const float* dev_x, int nrows, size_t ld, double* dev_out, void* dev_workspace, void* stream);

/* ---- zero-phase IIR: dsp.bp_filt = scipy.signal.filtfilt (dsp.py:859-880) and the caller-side
 *      scipy.signal.sosfiltfilt(sos, trace, axis=1) (Example.py:55).  host_sos: double[nsec][6],
 *      host_zi: double[nsec][2] (scipy.signal.sosfilt_zi), odd extension of padlen samples,
 *      dev_tmp: float32 [nx][ns + 2*padlen]. */
int d4w_sosfiltfilt(const float* dev_x, float* dev_y, float* dev_tmp, int nx, int ns, const double* host_sos,
                    const double* host_zi, int nsec, int padlen, void* stream);

/* ---- batched STFT magnitude with librosa.stft framing (dsp.get_spectrogram dsp.py:66-68,
 *      detect.get_sliced_nspectrogram detect.py:382): centred frames, zero padding, window
 *      dev_window[n_fft]; only DFT bins bin_lo..bin_hi (inclusive) are written (the band slice of
 *      detect.py:390-392): dev_out: float32 [nx][bin_hi-bin_lo+1][1 + ns/hop]. */
int d4w_stft_mag(d4w_fft_plan* plan, const float* dev_x, float* dev_out, int nx, int ns, int hop,
                 const float* dev_window, int bin_lo, int bin_hi, void* stream);

/* Same result as d4w_stft_mag with the periodic Hann window, for a band of bins of heavily overlapping frames
 * (n_fft = hop * P): sliding DFT, every sample enters one block sum per bin instead of one FFT per frame.  Shapes covered:
 * d4w_stft_slide_supported(n_fft, hop, bin_hi - bin_lo + 1) != 0; anything else returns D4W_ERR_UNSUPPORTED.
 * Replaces the librosa.stft call of detect.get_sliced_nspectrogram inside the channel loop of
 * detect.compute_cross_correlogram_spectrocorr (/root/reference/src/das4whales/detect.py:334-408, :700-707). */
int d4w_stft_slide_supported(int nfft, int hop, int nbins);
int d4w_stft_slide(d4w_fft_plan* plan, const float* x, float* out, int nx, int ns, int hop, int bin_lo, int bin_hi,
                   void* stream);

/* ---- spectrogram-correlation detector: detect.xcorr2d / compute_cross_correlogram_spectrocorr
 *      (detect.py:579-602, :650-708).  Per-row median / maximum of a float32 matrix [nrows][n]
 *      (entries must be >= 0 for the median), and
 *      out[row][t] = max(0, sum_f sum_j S[row][f][t - kw/2 + j] K[f][j]) / (med[row] * kw). */
int d4w_row_median(const float* dev_x, int nrows, size_t n, float* dev_median, void* stream);
int d4w_row_max(const float* dev_x, int nrows, size_t n, float* dev_max, void* stream);
int d4w_speccorr(const float* dev_S, int nx, int nf, int nt, const float* dev_K, int kw, const float* dev_median,
                 float* dev_out, void* stream);
/* Median of each row of a band: row r is the n values at dev_x + r * ld (ld >= n); d4w_row_median is ld = n. */
int d4w_row_median_ld(const float* dev_x, int nrows, size_t n, size_t ld, float* dev_median, void* stream);
/* Several kernels against one band spectrogram dev_S [nx][nf][nt] (the union of their bands), S read once: for each
 * k < nk (nk <= 8), d4w_speccorr of the slice S[:, f0[k] : f0[k] + nfk[k], :] with dev_K[k] [nfk[k]][kw[k]] and
 * dev_median[k] [nx] into dev_out[k] [nx][nt], bit-equal to it.  The arrays are host arrays (of device pointers). */
int d4w_speccorr_multi(const float* dev_S, int nx, int nf, int nt, int nk, const int* f0, const int* nfk,
                       const float* const* dev_K, const int* kw, const float* const* dev_median, float* const* dev_out,
                       void* stream);

/* ---- peak picking -- detect.pick_times_env (detect.py:169-195, the find_peaks call :192) and detect.pick_times
 *      (:249-274, :271): scipy.signal.find_peaks(row, prominence=threshold) on every row of a [nx][ns] float32 matrix
 *      (flat tops -> plateau midpoint, prominence walked to the nearest strictly greater sample, compared in double).
 *      flags[nx][ns] (bytes) is cleared and set to 1 at every accepted peak; ws needs
 *      d4w_find_peaks_workspace_bytes(nx, ns) bytes. */
size_t d4w_find_peaks_workspace_bytes(int nx, int ns);
int d4w_find_peaks(const float* dev_x, int nx, int ns, double prominence, unsigned char* dev_flags, void* dev_ws, void* stream);

/* ---- loader-side fusion -- data_handle.raw2strain (data_handle.py:157-177): out = (raw - mean_row(raw)) * scale_factor,
 *      from the on-disk int32 counts (raw_is_int32 = 1) or float32 to fp32 strain; mean in double. */
int d4w_raw2strain(const void* dev_raw, int raw_is_int32, int nx, int ns, double scale_factor, float* dev_out, void* stream);
/* ---- spectral views -- dsp.get_fx (dsp.py:18-38): out[row][(f + nfft/2) % nfft] = |FFT_nfft(x[row][0:ncopy] zero-padded)[f]| * scale
 *      (scale = 2e9 / nfft), `plan` = fft plan of length nfft, ld = row stride of x in samples; and dsp.instant_freq
 *      (dsp.py:830-856): out[i] = diff(unwrap(angle(x + i hx)))[i] / (2 pi) * fs for one channel, hx = H(x) from d4w_hilbert mode 2.
 *      d4w_hilbert modes: 0 envelope, 1 envelope SNR in dB, 2 the Hilbert transform H(x) itself, 3 envelope / std_row
 *      (improcess.trace2image, improcess.py:61; needs dev_stats). */
int d4w_row_fft_mag(d4w_fft_plan* plan, const float* dev_x, int nx, size_t ld, int ncopy, double scale, float* dev_out, void* stream);
int d4w_inst_freq(const float* dev_x, const float* dev_hx, int n, double fs, float* dev_out, void* stream);

/* ---- pick compaction: flags [nx][ns] (d4w_find_peaks) -> per-row counts, exclusive offsets [nx + 1] and the ascending
 *      sample indices of every row, so that only the picks leave the GPU (detect.py:192-194, :271-272). */
int d4w_peaks_offsets(const unsigned char* dev_flags, int nx, int ns, int* dev_counts, int* dev_offsets, void* stream);
int d4w_peaks_fill(const unsigned char* dev_flags, int nx, int ns, const int* dev_offsets, int* dev_idx, void* stream);

/* ---- image-domain ("Gabor") detector -- improcess.scale_pixels / trace2image (improcess.py:23-63): y = (x - min) / (max - min) * mul
 *      (dev_ws8: 8 bytes of scratch); improcess.binning (improcess.py:395-421) = torchvision Resize, bilinear with antialiasing,
 *      float32 [ih][iw] -> [oh][ow] (dev_tmp: ih*ow floats); cv2.filter2D(img, CV_64F, K) as the script calls it
 *      (scripts/main_gabordetect.py:109,135): correlation, centre anchor, BORDER_REFLECT_101, with optional on-the-fly
 *      thresholds (NaN = none): source binarised as in > in_thr, result binarised as out > out_thr (:123-124, :136-137);
 *      border 0 = BORDER_REFLECT_101 (cv2), 1 = zeros (scipy.signal.correlate(mode='same') of detect.nxcorr2d, detect.py:573);
 *      and binning(mask, 10, 10) + apply_smooth_mask (:166-169, improcess.py:452): out = trace * (resize(mask) != 0). */
int d4w_scale_pixels(const float* dev_x, float* dev_y, size_t n, float mul, void* dev_ws8, void* stream);
/* dsp.get_spectrogram's level scaling (dsp.py:76): y = 20 log10(x / max(x)) */
int d4w_db_re_max(const float* dev_x, float* dev_y, size_t n, void* dev_ws8, void* stream);
int d4w_resize_aa(const float* dev_in, int ih, int iw, float* dev_out, int oh, int ow, float* dev_tmp, void* stream);
int d4w_filter2d(const float* dev_in, int h, int w, const float* dev_K, int kh, int kw, float in_thr, float out_thr, int border,
                 float* dev_out, void* stream);
int d4w_mask_upsample_mul(const float* dev_trace, int nx, int ns, const float* dev_mask, int mh, int mw, float* dev_out,
                          unsigned char* dev_mask_out, void* stream);
/* D4W_CDEF_END */

#ifdef __cplusplus
}
#endif
#endif /* D4W_H */
