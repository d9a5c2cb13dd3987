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
 * C order, device memory; y may alias x.  x and y must be 16-byte aligned when ns % 4 == 0
 * and 8-byte aligned when ns is even, else D4W_ERR_ARG before any launch (the same holds for
 * the pass-wise calls below and for the matrices of a mask bank). */
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

/* ---- f-k mask bank: several masks over one plan and one forward transform (scripts/main_fkcomp.py:66-95
 *      filters the same matrix with four masks, each through dsp.fk_filter_sparsefilt, :73-95) ----------- */
typedef struct d4w_fk_bank d4w_fk_bank;
/* The bank keeps the union U of the masks' kept wavenumber rows, each mask's support taken as it is now (after
 * d4w_fk_mask_prune, if any).  Every mask must be of `plan`, built (d4w_fk_mask_build) before d4w_fk_bank_build,
 * not pruned again, and must outlive the bank.  D4W_ERR_ARG: nmasks < 1, a null mask, a mask of another plan. */
int d4w_fk_bank_create(d4w_fk_bank** out, d4w_fk_plan* plan, d4w_fk_mask* const* masks, int nmasks);
int d4w_fk_bank_destroy(d4w_fk_bank* bank);
/* |U|, the rows every mask of the bank is filtered on */
int d4w_fk_bank_rows(const d4w_fk_bank* bank);
/* bytes of device memory for the bank's tables: nmasks x |U| x ns float32 */
size_t d4w_fk_bank_table_bytes(const d4w_fk_bank* bank);
/* fill the caller's table (kept by reference until the bank is destroyed): mask i's own transform-order table on the
 * slots of its kept rows and exact zeros on the other slots of U, so a pruned mask's dropped rows stay dropped */
int d4w_fk_bank_build(d4w_fk_bank* bank, float* dev_table, void* stream);
/* bytes of workspace for d4w_fk_bank_apply: two blocks of |U| kept rows (the forward transform and one mask's
 * filtered rows), plus the level-A/B intermediate of a two-level plan */
size_t d4w_fk_bank_workspace_bytes(const d4w_fk_plan* plan, const d4w_fk_bank* bank);
/* dev_ys[i] = d4w_fk_apply(plan, mask i, dev_x) for every mask, with one forward transform: P1 (optional taper, as
 * d4w_fk_apply) and P2 once, then for each mask P3 out of place into the second block, P4 and P5 into dev_ys[i].
 * dev_ys is a host array of nmasks device pointers.  One output may alias x; outputs may not overlap each other
 * (D4W_ERR_ARG), nor may the bank be applied before d4w_fk_bank_build. */
int d4w_fk_bank_apply(d4w_fk_plan* plan, d4w_fk_bank* bank, const float* dev_x, float* const* dev_ys,
                      void* dev_workspace, int taper, void* stream);
/* the passes separately (profiling): passes 1 and 2 serve every mask, passes 3..5 run mask `mask` (pass 5 writes
 * dev_ys[mask]); 1, 2, then 3, 4, 5 for each mask in turn is d4w_fk_bank_apply */
int d4w_fk_bank_apply_pass(d4w_fk_plan* plan, d4w_fk_bank* bank, const float* dev_x, float* const* dev_ys,
                           void* dev_workspace, int taper, int pass, int mask, void* stream);

/* ---- f-k power spectrum: P = |fftshift(fft2(x))|^2 over a band of the shifted plane, the filter's forward
 *      transform (P1, P2) followed by a forward-only power pass; no mask, no inverse ----------------------------- */
typedef struct d4w_fk_spectrum d4w_fk_spectrum;
/* The band is rows [k_lo, k_hi) x columns [f_lo, f_hi) of the shifted [nx x ns] plane (half-open).  Only the
 * half-plane rows k' in [0, nx/2] with +k' or -k' inside the band are transformed.  D4W_ERR_ARG: an empty band or one
 * outside the plane, a null argument.  The spectrum keeps a reference to `plan`, which must outlive it. */
int    d4w_fk_spectrum_create(d4w_fk_spectrum** out, d4w_fk_plan* plan, int k_lo, int k_hi, int f_lo, int f_hi);
int    d4w_fk_spectrum_destroy(d4w_fk_spectrum* s);
/* half-plane rows transformed */
int    d4w_fk_spectrum_rows(const d4w_fk_spectrum* s);
/* bytes of workspace for d4w_fk_spectrum_apply: the transformed rows, plus the level-A/B intermediate of a
 * two-level plan */
size_t d4w_fk_spectrum_workspace_bytes(const d4w_fk_plan* plan, const d4w_fk_spectrum* s);
/* dev_out[(k_hi - k_lo) x (f_hi - f_lo)] float32 = scale * P (accumulate = 0) or += scale * P (accumulate = 1), P the
 * band of |fftshift(fft2(x))|^2, x tapered first by Tukey(alpha=0.03) along time when taper != 0 (x itself is not
 * modified).  x: float32 [nx x ns], aligned as d4w_fk_apply requires.  D4W_ERR_ARG: a null argument, a misaligned
 * x, a spectrum made for another plan or device. */
int    d4w_fk_spectrum_apply(d4w_fk_plan* plan, d4w_fk_spectrum* s, const float* dev_x, float* dev_out,
                             void* dev_workspace, int taper, float scale, int accumulate, void* stream);

/* ---- f-k Welch spectrum: segment staging for d4w_fk_spectrum_apply -------------------------------------------- */
/* Stage nseg segments of the float32 [nx x ns] matrix dev_x, all on channels [c0, c0 + lx): segment s (0 <= s < nseg)
 * covers samples [t0 + s*step, t0 + s*step + l) and is written as a contiguous [lx x l] matrix at
 * dev_out + s * seg_stride (floats):  out[s][c][t] = (x[c0 + c][t0 + s*step + t] - m) * wx[c] * wt[t],  m the mean of
 * the row's l samples (accumulated in double) when detrend != 0, else 0.  dev_wx [lx] and dev_wt [l] are the channel and
 * time windows.  dev_x is not modified.  D4W_ERR_ARG: a null pointer, segments outside the matrix, lx > 65 535,
 * seg_stride < lx * l, dev_out / seg_stride that would leave a segment off the alignment d4w_fk_spectrum_apply needs
 * for rows of l samples (16 bytes when l % 4 == 0, 8 when l is even), or a dev_wt that is not 16-byte aligned when
 * l % 4 == 0. */
int    d4w_fk_segment_stage(const float* dev_x, int nx, int ns, int c0, int lx, int t0, int l, int step, int nseg,
                            const float* dev_wx, const float* dev_wt, int detrend, float* dev_out, size_t seg_stride,
                            void* stream);

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
 *      the mean-of-padded-template term mu_t/m_t * prefix is added (dev_mu_over_m: double[ntpl]).  Any number of rows.
 *      dev_out: float32 [ntpl][nx][ns]. */
int d4w_xcorr(d4w_fft_plan* plan, const float* dev_x, int nx, int ns, int valid, int ntpl, const void* dev_tabs,
              const double* dev_mu_over_m, const double* dev_stats, const double* dev_segpre, float* dev_out,
              void* stream);
/* ---- "same"-mode matched filter: scipy.signal.correlate(x / max(x), c_t, 'same') of every row with each template
 *      (scripts/main_gabordetect.py:243-246), on the same overlap-save blocks as d4w_xcorr:
 *      out[t][row][i] = sum_n x[row][i - lag0 + n] c'_t[n] / rowmax[row], x = 0 outside [0, ns), where c'_t is template t with
 *      lag0 - floor(L_t / 2) zeros prepended (lag0 = max_t floor(L_t / 2)).  dev_tabs: ntpl x nb complex64 =
 *      conj(FFT_nb(c'_t)) / nb in d4w_fft_plan_table_order; valid = nb - max_t len(c'_t) + 1.  dev_rowmax: float[nx] from
 *      d4w_row_max (clamped at 0); rows with !(rowmax > 0) are written as zeros.  Any nx >= 1.
 *      dev_out: float32 [ntpl][nx][ns]. */
int d4w_xcorr_same(d4w_fft_plan* plan, const float* dev_x, int nx, int ns, int valid, int lag0, int ntpl, const void* dev_tabs,
                   const float* dev_rowmax, float* dev_out, void* stream);

/* ---- Hilbert envelope |scipy.signal.hilbert(x, axis=1)| (detect.py:192) and
 *      dsp.snr_tr_array(trace, env=True) (dsp.py:975).  mode 0: envelope, 1: 10*log10(env^2/var).
 *      dev_out must not overlap dev_x (long rows are transformed two per complex FFT and dev_x is read again at the end).
 *      d4w_xcorr's dev_tabs are in d4w_fft_plan_table_order.
 *      Any ns up to 128 000 is accepted: a length with no T1 x T2 split (a prime factor > 61) is transformed by a chirp-z
 *      convolution of length czt_m = T1 * T2 ~ 2 ns.  d4w_row_plan_info reports the split and czt_m (0: direct transform);
 *      d4w_row_workspace_bytes sizes the workspace for nx rows of the chosen route.  Any number of rows: split rows go in
 *      blocks of 2 x 65 535 that reuse one block's workspace in stream order, so the bytes for min(nx, 131 070) rows
 *      suffice (a larger workspace is fine). */
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
 * dev_workspace: d4w_env_stats_workspace_bytes(plan, nrows, ld) bytes (the envelope of one block of at most 65 535 rows,
 * reused by the next in stream order, and a dense copy of the window when ld != n).  Any nrows >= 1. */
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
 *      detect.py:390-392): dev_out: float32 [nx][bin_hi-bin_lo+1][1 + ns/hop].  Any number of rows. */
int d4w_stft_mag(d4w_fft_plan* plan, const float* dev_x, float* dev_out, int nx, int ns, int hop,
                 const float* dev_window, int bin_lo, int bin_hi, void* stream);

/* Same result as d4w_stft_mag with the periodic Hann window, for a band of bins of heavily overlapping frames
 * (n_fft = hop * P): sliding DFT, every sample enters one block sum per bin instead of one FFT per frame.  Shapes covered:
 * d4w_stft_slide_supported(n_fft, hop, bin_hi - bin_lo + 1) != 0; anything else returns D4W_ERR_UNSUPPORTED.
 * Replaces the librosa.stft call of detect.get_sliced_nspectrogram inside the channel loop of
 * detect.compute_cross_correlogram_spectrocorr (/root/reference/src/das4whales/detect.py:334-408, :700-707).  Any nx >= 1. */
int d4w_stft_slide_supported(int nfft, int hop, int nbins);
int d4w_stft_slide(d4w_fft_plan* plan, const float* x, float* out, int nx, int ns, int hop, int bin_lo, int bin_hi,
                   void* stream);

/* ---- Welch power spectral density of every chunk of every row: tools.spec / tools.__spec_chunk
 *      (/root/reference/src/das4whales/tools.py:212-236), scipy.signal.welch(chunk, fs, window, nperseg, noverlap, nfft,
 *      detrend, return_onesided=True, scaling, average) per chunk.  Row r, chunk c is the `chunk` samples at
 *      dev_x + r * ns + c * chunk, c < ns / chunk (chunk = ns: the whole row).  Segment s of a chunk covers samples
 *      [s * step, s * step + nperseg), nseg = (chunk - nperseg) / step + 1 (step = nperseg - noverlap; a trailing partial
 *      segment is dropped, no padding, no centring).  detrend != 0 subtracts each segment's mean; the segment is multiplied by
 *      dev_window[nperseg] and zero-padded to nfft = the plan's length.  The periodogram |X_k|^2 * scale (scale = 1 / (fs * sum
 *      w^2) for a density, 1 / (sum w)^2 for a spectrum) is doubled at every bin but DC and, for even nfft, Nyquist (SciPy's
 *      one-sided rule), then averaged over the segments: average 0 = mean, 1 = np.median / _median_bias(nseg).
 *      dev_out: float32 [nrows][ns / chunk][nfft / 2 + 1].  Every nfft the plan accepts whose one complex frame (plus the bin
 *      sums) fits shared memory: D4W_ERR_UNSUPPORTED names the limit.  D4W_ERR_ARG: nrows < 1, chunk outside [1, ns],
 *      nperseg outside [1, chunk], step < 1, nfft < nperseg.
 *      dev_workspace: d4w_welch_workspace_bytes bytes (0 unless a median over more segments than fit shared memory, which
 *      writes every periodogram bin-major for d4w_row_median: nrows x nchunks x nbins x nseg floats). */
size_t d4w_welch_workspace_bytes(const d4w_fft_plan* plan, int nrows, int ns, int chunk, int nperseg, int step, int average);
int d4w_welch(d4w_fft_plan* plan, const float* dev_x, int nrows, int ns, int chunk, int nperseg, int step,
              const float* dev_window, int detrend, double scale, int average, float* dev_out, void* dev_workspace,
              void* stream);

/* ---- cross-spectral density and coherence of row pairs: scipy.signal.csd(x, y, fs, window, nperseg, noverlap, nfft,
 *      detrend, return_onesided=True, scaling, average) and scipy.signal.coherence(x, y, ...) for every output row at once.
 *      Output row r pairs the ns samples at dev_x + r * x_row_stride with those at dev_y + r * y_row_stride (floats); a
 *      stride of 0 broadcasts one row against every row of the other side (the neighbour pairs x[:-1], x[1:] of a
 *      contiguous matrix are dev_x, dev_x + ns with both strides ns).  Segments, detrending, window, nfft = the plan's
 *      length and scale are d4w_welch's (with chunk = ns).  Per segment P_k = conj(X_k) Y_k * scale, doubled at every bin
 *      but DC and, for even nfft, Nyquist.
 *      what 0: Pxy, dev_out float2 [nrows][nfft / 2 + 1], averaged over the segments: average 0 = mean, 1 = (np.median of
 *      Re + i np.median of Im) / _median_bias(nseg).
 *      what 1: Cxy = |Pxy|^2 / (Pxx Pyy) of the mean spectra (average must be 0), dev_out float [nrows][nfft / 2 + 1]; a
 *      row whose Pxx or Pyy is 0 gives NaN, as 0 / 0 in NumPy.
 *      Every nfft the plan accepts whose one complex frame plus the bin sums of the mean route (2 doubles per bin for Pxy, 4
 *      for Cxy; the workspace median keeps none) fits shared memory: D4W_ERR_UNSUPPORTED names the limit of the route taken.  D4W_ERR_ARG: nrows < 1, nperseg outside [1, ns], step < 1,
 *      nfft < nperseg, a row stride neither 0 nor >= ns, what = 1 with average = 1.
 *      dev_workspace: d4w_csd_workspace_bytes bytes (0 unless a median over more segments than fit shared memory, which
 *      writes every periodogram as [nrows][nbins][re, im][nseg] floats and selects each row of nseg signed values). */
size_t d4w_csd_workspace_bytes(const d4w_fft_plan* plan, int nrows, int ns, int nperseg, int step, int what, int average);
int d4w_csd(d4w_fft_plan* plan, const float* dev_x, long long x_row_stride, const float* dev_y, long long y_row_stride,
            int nrows, int ns, int nperseg, int step, const float* dev_window, int detrend, double scale, int what,
            int average, void* dev_out, void* dev_workspace, void* stream);

/* ---- spectrogram-correlation detector: detect.xcorr2d / compute_cross_correlogram_spectrocorr
 *      (detect.py:579-602, :650-708).  Per-row median / maximum of a float32 matrix [nrows][n]
 *      (entries must be >= 0 for the median), and
 *      out[row][t] = max(0, sum_f sum_j S[row][f][t - kw/2 + j] K[f][j]) / (med[row] * kw).  d4w_speccorr and
 *      d4w_speccorr_multi take any nx >= 1. */
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
 *      d4w_find_peaks_workspace_bytes(nx, ns) bytes.  Any nx >= 1: rows go in blocks of 65 535 that reuse one block's
 *      workspace in stream order, so the bytes for min(nx, 65 535) rows suffice (a larger workspace is fine). */
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
/* ---- localisation: loc.solve_lq, loc.calc_covariance_matrix, loc.calc_uncertainty_position (das4whales/loc.py:57-216) for
 *      a batch of calls, in FP64.  Call b is the observations [dev_offsets[b], dev_offsets[b + 1]) of dev_T (arrival times, s)
 *      and dev_pos ([n_obs][3], m); p = 4 unknowns (x, y, z, t0), or 3 with fix_z (z held at the first guess).
 *  d4w_loc_grid: first guess from a grid search.  Nodes (dev_gx[ix], dev_gy[iy], dev_gz[iz]), index (iz * ny + iy) * nx + ix;
 *      score = sum (T - t0* - d / c0)^2 / (n - p), t0* = mean(T - d / c0).  dev_index[b] (int64) = the node of least score
 *      (ties to the lowest index), dev_score[b] (NaN when n <= p), dev_n0[b][4] = (node, t0*); an empty call gets index -1
 *      and NaN.  fix_z needs nz = 1.  dev_workspace: d4w_loc_grid_workspace_bytes bytes.
 *  d4w_loc_solve: Nbiter Gauss-Newton steps from dev_n0[b][4] (NULL: the reference's [40000, 23000, -60, min T]) with
 *      (G^T G + 1e-5 I) dn = G^T dt and a step of 0.7 dn for the first four; then dev_n[b][4], dev_var[b] = sum dt^2 / (n - p)
 *      (NaN when n <= p), C = (G^T G)^-1 at the final n, or (G^T G + 1e-5 I)^-1 when its 2-norm condition number exceeds
 *      1 / DBL_EPSILON, and dev_unc[b][p] = sqrt(var diag C).  Optional (NULL to skip): dev_cinv[b][p][p] = C,
 *      dev_cond[b], dev_traj[b][nbiter][4] the estimate after every iteration, dev_n0_used[b][4] the first guess.  An empty
 *      call is NaN throughout.  Deterministic: no atomics, fixed reduction order. */
size_t d4w_loc_grid_workspace_bytes(int ncalls, int nx, int ny, int nz);
int d4w_loc_grid(const double* dev_T, const double* dev_pos, const long long* dev_offsets, int ncalls, double c0, int fix_z,
                 const double* dev_gx, int nx, const double* dev_gy, int ny, const double* dev_gz, int nz, void* dev_workspace,
                 long long* dev_index, double* dev_score, double* dev_n0, void* stream);
int d4w_loc_solve(const double* dev_T, const double* dev_pos, const long long* dev_offsets, int ncalls, double c0, int nbiter,
                  int fix_z, const double* dev_n0, double* dev_n, double* dev_var, double* dev_unc, double* dev_cinv,
                  double* dev_cond, double* dev_traj, double* dev_n0_used, void* stream);
/* ---- pick association by back-projection over a source grid, in FP64 (loc.associate_picks).  Picks are a CSR by channel:
 *      channel c (c < n_channels, at dev_cable_pos[c][3], m) holds the int32 samples dev_samples[dev_offsets[c] ..
 *      dev_offsets[c + 1]), n_picks = dev_offsets[n_channels]; the pipelines' (offsets, idx).  Nodes as d4w_loc_grid.
 *      T_p = s_p / fs; tau(g, c) = sqrt(dx dx + dy dy + dz dz) / c0, dx = cable_pos[c][0] - g_x (likewise y, z), left to right,
 *      every operation rounded on its own (no fused multiply-add); o = T_p - tau; bin j = floor(o r) with h = tol / 2 and
 *      r = 1 / h given by the caller.  n(g, j) counts the unassigned picks in bin j of node g; (g, j) scores n(g, j) + n(g, j + 1).
 *      Repeated: the (g, j) of highest score, ties to the lowest node, then the lowest j; stop when the score is below
 *      min_picks or after max_calls calls; else call k gets dev_node[k] = g, dev_t0[k] = (j + 1) h, the unassigned picks with
 *      bin j or j + 1 (dev_labels[p] = k, int64, CSR order; -1 for a pick of no call) and dev_count[k] = their number.
 *      *n_calls = K.  Two picks of one channel count separately; a straight cable cannot tell a source from its mirror
 *      image, and the tie rule then returns the lower node index.  Deterministic: integer counts, fixed reduction order.
 *  d4w_loc_assoc_bins: the bin range [*jlo, *jlo + *nbins) that covers every origin time of picks with T in [t_min, t_max]
 *      at channels inside host_box[0..5] = (min x, y, z, max x, y, z) from nodes inside host_box[6..11] (host memory, no
 *      device work).  D4W_ERR_UNSUPPORTED, naming the limit, when the vote's histogram (4 nodes x (nbins + 1) ints per
 *      block) does not fit shared memory: raise tol or shorten the record.  d4w_loc_associate applies it to the picks' own
 *      range (one small read-back), and reads back one record per extracted call; no per-pick data leaves the device.
 *      D4W_ERR_ARG: offsets that do not rise from 0 to n_picks, a negative sample.  dev_workspace:
 *      d4w_loc_assoc_workspace_bytes bytes. */
int d4w_loc_assoc_bins(double t_min, double t_max, const double* host_box, double c0, double r, long long* jlo, int* nbins);
size_t d4w_loc_assoc_workspace_bytes(long long n_picks, int nx, int ny, int nz);
int d4w_loc_associate(const int* dev_offsets, const int* dev_samples, int n_channels, long long n_picks, double fs,
                      const double* dev_cable_pos, double c0, const double* dev_gx, int nx, const double* dev_gy, int ny,
                      const double* dev_gz, int nz, double h, double r, int min_picks, int max_calls, void* dev_workspace,
                      long long* dev_labels, long long* dev_node, double* dev_t0, long long* dev_count, int* n_calls,
                      void* stream);

/* ---- image operators of improcess outside the Gabor path (das4whales/improcess.py:143-169, :319-367).
 *  d4w_radon: skimage.transform.radon(image, theta, circle=False) of the float32 image [h][w] placed at rows
 *      [pad_r, pad_r + h), columns [pad_c, pad_c + w) of an n x n zero square.  dev_cs: double [nangles][2] = (cos, sin) of
 *      each angle; dev_out: double [n][nangles], bin b at angle a = the sum over rows r of the bilinear sample of the square
 *      at x = cos b + sin r - c (cos + sin - 1), y = -sin b + cos r - c (cos - sin - 1), c = n / 2.  No atomics: runs are
 *      bit-identical.
 *  d4w_bilateral: cv2.bilateralFilter(img, 2 radius + 1, sigma_color, sigma_space) of one channel, with the
 *      caller's radius (1..64) and sigmas (> 0) already normalised as OpenCV does.  is_8u: the image holds the integers of an
 *      8-bit image and the result is rounded and saturated to them; otherwise 32F.  dev_workspace: D4W_BILATERAL_WS_BYTES.
 *  d4w_grad_oriented: improcess.gradient_oriented(image, (dft, dfx)) for dft, dfx >= 0, not both 0: dev_out is
 *      [h][w - dft] (dfx = 0), [h - dfx][w] (dft = 0) or [h - 2 dfx][w - dft]; an empty output is D4W_ERR_ARG. */
enum { D4W_BILATERAL_WS_BYTES = 16 + 4 * 4099 };
int d4w_radon(const float* dev_img, int h, int w, int n, int pad_r, int pad_c, const double* dev_cs, int nangles,
              double* dev_out, void* stream);
int d4w_bilateral(const float* dev_in, int h, int w, int is_8u, int radius, double sigma_color, double sigma_space,
                  void* dev_workspace, float* dev_out, void* stream);
int d4w_grad_oriented(const float* dev_in, int h, int w, int dft, int dfx, float* dev_out, void* stream);

/* ---- the tools module (das4whales/tools.py:8-157) and the legacy dsp.fk_filt (dsp.py:883-953).
 *  d4w_fan_blur: the Gaussian-blurred speed fan, float32 [nx][ns] in the reference's shifted layout: with
 *      f_j = (j - ns/2) fval, k_i = (i - nx/2) kval (numpy.fft.fftfreq's products), g = [f < k c_min and f < -k c_min],
 *      g2 the same with c_max, G = g + fliplr(g) - g2 - fliplr(g2), blurred as scipy.ndimage.gaussian_filter(G, sigma)
 *      (truncate 4, mode 'reflect', repeated for a radius beyond an axis) in float64 and normalised as
 *      (G - min) / (max - min): NaN everywhere when max == min, as NumPy's 0 / 0.  fval > 0.  The radius int(4 sigma + 0.5)
 *      must leave the shared tile within 227 KB (sigma up to about 100).  dev_workspace: d4w_fan_blur_workspace_bytes.
 *  d4w_row_moments: sum x, sum t x and sum x^2 in float64 of every time chunk of every row: row r is the n samples at
 *      dev_x + r * ld, chunk c its samples [c chunk, min((c + 1) chunk, n)), t counted from the chunk start.
 *      dev_out: double [nrows][ceil(n / chunk)][3].
 *  d4w_detrend_linear: scipy.signal.detrend(type='linear', axis=-1) of the same rows (moments of chunk = n from
 *      d4w_row_moments), written contiguously: dev_y float32 [nrows][n].  Any nrows >= 1. */
size_t d4w_fan_blur_workspace_bytes(int nx, double sigma);
int d4w_fan_blur(float* dev_out, int nx, int ns, double kval, double fval, double c_min, double c_max, double sigma,
                 void* dev_workspace, void* stream);
int d4w_row_moments(const float* dev_x, size_t ld, int nrows, int n, int chunk, double* dev_out, void* stream);
int d4w_detrend_linear(const float* dev_x, size_t ld, int nrows, int n, const double* dev_moments, float* dev_y, void* stream);

/* ---- the hybrid masks of dsp.py designed on the device, as float32 [nx][ns] in the reference's shifted layout, to hand to
 * d4w_fk_mask_create_dense.  kind 0: hybrid_filter_design (dsp.py:174-305), elementwise in float64; kind 1:
 * hybrid_gs_filter_design (:457-579); kind 2: hybrid_ninf_gs_filter_design (:582-702).  Kinds 1 and 2 are blurred as
 * scipy.ndimage.gaussian_filter(M, 20) (truncate 4, mode 'reflect') in float64, with no normalisation.  f_j = (j - ns/2) fval,
 * k_i = (i - nx/2) kval (numpy.fft.fftfreq's products); host_H = the design function's ns-long H (host pointer, read
 * before the call returns; for kinds 1 and 2 it must be 1 on one band of columns and 0 elsewhere); col_lo / col_hi = its
 * np.argmax column range (col_hi < col_lo: the reference's loop does not run; kind 0 needs col_lo <= col_hi).  D4W_ERR_ARG
 * unless the speeds are finite and > 0, fval finite and > 0, kval finite and fmin < fmax finite; nx <= 65 535.
 * cp_max is read by kind 2 only, cs_min by kind 0 only.  dev_workspace: d4w_mask_design_workspace_bytes(nx, ns). */
size_t d4w_mask_design_workspace_bytes(int nx, int ns);
int d4w_mask_design(int kind, float* dev_out, int nx, int ns, double kval, double fval, double cs_min, double cp_min,
                    double cp_max, double fmin, double fmax, int col_lo, int col_hi, const double* host_H,
                    void* dev_workspace, void* stream);
/* D4W_CDEF_END */

#ifdef __cplusplus
}
#endif
#endif /* D4W_H */
