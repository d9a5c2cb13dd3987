"""File-level detection pipelines on one GPU (BASELINE config 5: one file per GPU).

`MfDetectPipeline` is the device-side equivalent of scripts/main_mfdetect.py:42-103 of the reference:

    raw counts (int32, as stored in the HDF5 file)           data_handle.load_das_data / raw2strain   (data_handle.py:157-214)
      -> strain (demean, scale)                               d4w_raw2strain
      -> band-pass 14-30 Hz, zero phase                       dsp.bp_filt                              (main_mfdetect.py:53)
      -> f-k filter, hybrid_ninf mask                         dsp.fk_filter_sparsefilt                 (:46-47, :55)
      -> HF + LF fin-whale matched filter (one pass)          detect.compute_cross_correlogram x 2     (:72-80)
      -> detection threshold 0.5 * max correlation            (:83, :95)
      -> Hilbert envelope + prominence peak picking           detect.pick_times_env x 2                (:98-99)
      -> (channel, sample) pick lists                         detect.convert_pick_times                (:102-103)

`GaborDetectPipeline` is the same for scripts/main_gabordetect.py:58-266: the same strain, band-pass and f-k front end,
then the image-domain Gabor mask (improcess.gabor_detect, :78-169) and the script's own matched filter -- a centred
("same") correlation of each masked channel divided by its maximum with the un-padded HF / LF notes, channels whose
maximum is <= 0 skipped (detect.compute_cross_correlograms_same, :223-246) -- before the same threshold and picking (:252-266).

`SpectroDetectPipeline` is scripts/main_spectrodetect.py:39-123: the same front end, then the HF and LF
spectrogram-correlation correlograms from one sliding STFT (detect.compute_cross_correlograms_spectrocorr, :103-107) and
find_peaks with an absolute prominence on the raw correlograms (detect.pick_times, :117-118); picks are in STFT frames.

`NoiseProfilePipeline` is scripts/main_bathynoise.py:122-259: the same front end, then the per-channel noise profile
(envelope median and mean, std, SNR_1d, and the power and mean envelope of a noise window) from two envelope-statistics
passes (rows.env_stats); it yields [nx]-long float64 vectors instead of picks.

Only the raw counts go up (pinned int32, 4 bytes per sample) and only the picks come down; every intermediate matrix
stays in HBM.  `stream(files)` overlaps the H2D copy of file i+1 with the processing of file i.
"""
import numpy as np

from . import detect as _detect
from . import dsp as _dsp
from . import fk as _fk
from . import improcess as _improcess
from . import rows as _rows


class _FilePipeline:
    """Shared part of the file pipelines: strain -> band-pass -> hybrid_ninf f-k filter on the device, the
    threshold-and-pick tail, and the double-buffered upload of `stream`.  Subclasses implement process_device(raw) on top
    of _filtered and _pick (or their own picking tail)."""

    def __init__(self, nx, ns, selected_channels, dx, fs, scale_factor, device, fmin, fmax, mask_speeds, thres_frac,
                 prune_eps, bandpass):
        import scipy.signal as sp
        torch = _fk._torch()
        self.torch = torch
        self.nx, self.ns, self.fs = int(nx), int(ns), float(fs)
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.scale_factor = float(scale_factor)
        self.thres_frac = None if thres_frac is None else float(thres_frac)      # None: the subclass picks by its own rule
        self.bandpass = bool(bandpass)
        with torch.cuda.device(self.device):
            self.mask = _dsp.hybrid_ninf_filter_design((nx, ns), selected_channels, dx, fs, *mask_speeds, fmin=fmin, fmax=fmax)
            self.fk = _fk.FkFilter(self.mask, device=self.device, eps=prune_eps)
        self.sos = sp.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp", output="sos")          # dsp.bp_filt (dsp.py:878)
        self._raw = [None, None]
        self._h2d = None

    # ---- device side -------------------------------------------------------------------------------------------------
    def _filtered(self, raw):
        x = _rows.raw2strain(raw, self.scale_factor)
        if self.bandpass:
            x = _rows.sosfiltfilt(self.sos, x, padlen=3 * 17)
        return self.fk(x, out=x)

    def _maxv(self, corr):
        """max over all correlograms (0-dim device tensor; row_max clamps at 0)"""
        rmax = self.torch.stack([_rows.row_max(c) for c in corr])                # [2, nx]
        return _rows.row_max(rmax.reshape(1, -1))[0]

    def _pick(self, corr, with_snr):
        maxv = self._maxv(corr)
        thres = self.thres_frac * float(maxv.item())                             # main_mfdetect.py:95 (one scalar D2H)
        out = {"maxv": maxv, "threshold": thres}
        for name, c, thr in (("hf", corr[0], thres * 0.9), ("lf", corr[1], thres)):
            env = _rows.envelope(c)
            out["picks_" + name] = _rows.find_peaks_device(env, thr)
            del env
            if with_snr:
                out["snr_" + name] = _rows.snr(c, env=True)
        return out

    def _to_host(self, res):
        """process_device's result -> what process_file / stream yield: host pick arrays, maxv and threshold"""
        return {"picks_hf": self.picks_to_host(res["picks_hf"]), "picks_lf": self.picks_to_host(res["picks_lf"]),
                "maxv": float(res["maxv"].item()), "threshold": res["threshold"]}

    @staticmethod
    def picks_to_host(picks):
        """(offsets, idx) on the device -> array([[channel ...], [sample ...]]) like detect.convert_pick_times."""
        offsets, idx = picks
        off = offsets.cpu().numpy().astype(np.int64)
        tt = idx.cpu().numpy().astype(np.int64)
        ch = np.repeat(np.arange(len(off) - 1, dtype=np.int64), np.diff(off))
        return np.asarray((ch, tt))

    # ---- host side ---------------------------------------------------------------------------------------------------
    def _staging(self, i, like):
        torch = self.torch
        if self._raw[i] is None or self._raw[i].dtype != like.dtype:
            self._raw[i] = torch.empty((self.nx, self.ns), dtype=like.dtype, device=f"cuda:{self.device}")
        return self._raw[i]

    def process_file(self, raw_host):
        """One file: raw_host = int32 / float32 ndarray or (pinned) CPU tensor [nx, ns].  Returns host pick arrays."""
        return next(self.stream([raw_host]))

    def stream(self, files):
        """Iterate over host arrays / tensors; yields the host results of each file (_to_host: {"picks_hf", "picks_lf",
        "maxv", "threshold"} for the detectors) with the H2D copy of the next file running on a second stream under the
        processing of the current one."""
        torch = self.torch
        if self._h2d is None:
            self._h2d = torch.cuda.Stream(device=self.device)
        it = iter(files)
        cur_stream = torch.cuda.current_stream(self.device)

        def upload(i, h):
            t = h if isinstance(h, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(h))
            if t.dtype not in (torch.int32, torch.float32):
                t = t.to(torch.float32)
            dst = self._staging(i, t)
            with torch.cuda.stream(self._h2d):
                self._h2d.wait_stream(cur_stream)                 # the buffer's previous consumer has finished
                dst.copy_(t, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._h2d)
            return dst, ev

        nxt = next(it, None)
        if nxt is None:
            return
        pending = upload(0, nxt)
        i = 0
        while pending is not None:
            dst, ev = pending
            nxt = next(it, None)
            # enqueue the next file's copy first: it waits (on the copy stream) for the kernels already queued -- the
            # previous user of that staging buffer -- and then runs under this file's processing
            pending = upload((i + 1) % 2, nxt) if nxt is not None else None
            cur_stream.wait_event(ev)
            yield self._to_host(self.process_device(dst))
            i += 1


class MfDetectPipeline(_FilePipeline):
    def __init__(self, nx, ns, selected_channels, dx, fs, scale_factor, device=None, fmin=14., fmax=30.,
                 mask_speeds=(1350., 1450., 3300, 3450), hf=(17.8, 28.8, 0.68), lf=(14.7, 21.8, 0.78), thres_frac=0.5,
                 prune_eps=0.0, bandpass=True):
        super().__init__(nx, ns, selected_channels, dx, fs, scale_factor, device, fmin, fmax, mask_speeds, thres_frac,
                         prune_eps, bandpass)
        time = np.arange(ns) / fs
        self.templates = [_detect.gen_template_fincall(time, fs, *hf), _detect.gen_template_fincall(time, fs, *lf)]

    def process_device(self, raw, with_snr=False):
        """raw: int32 (or float32) CUDA tensor [nx, ns] of interrogator counts.  Returns a dict of DEVICE results:
        picks_hf / picks_lf = (offsets int32 [nx + 1], idx int32 [n]) , maxv (0-dim tensor), optionally snr_hf / snr_lf."""
        torch = self.torch
        with torch.cuda.device(self.device):
            y = self._filtered(raw)
            corr = _rows.cross_correlogram_chunked(y, self.templates, normalize=True)
            del y
            return self._pick(corr, with_snr)


class GaborDetectPipeline(_FilePipeline):
    """scripts/main_gabordetect.py:58-266 on the device; the script's values are the defaults.  Same interface as
    MfDetectPipeline (process_device / process_file / stream)."""

    def __init__(self, nx, ns, selected_channels, dx, fs, scale_factor, device=None, fmin=14., fmax=30.,
                 mask_speeds=(1350., 1450., 3300, 3450), hf=(17.8, 28.8, 0.68), lf=(14.7, 21.8, 0.78), thres_frac=0.5,
                 c0=1500., bin_factor=10, threshold=9100., threshold2=150., prune_eps=0.0, bandpass=True):
        super().__init__(nx, ns, selected_channels, dx, fs, scale_factor, device, fmin, fmax, mask_speeds, thres_frac,
                         prune_eps, bandpass)
        self.dx, self.selected_channels = float(dx), list(selected_channels)
        self.c0, self.bin_factor = float(c0), int(bin_factor)
        self.threshold, self.threshold2 = float(threshold), float(threshold2)
        notes = []
        for fmin_, fmax_, dur in (hf, lf):                                    # main_gabordetect.py:223-227
            c = _detect.gen_hyperbolic_chirp(fmin_, fmax_, dur, fs)
            notes.append(np.hanning(len(c)) * c)
        self.templates = notes

    def process_device(self, raw, with_snr=False, with_intermediates=False):
        """raw: int32 (or float32) CUDA tensor [nx, ns] of interrogator counts.  Returns a dict of DEVICE results:
        picks_hf / picks_lf = (offsets int32 [nx + 1], idx int32 [n]), maxv (0-dim tensor), optionally snr_hf / snr_lf and,
        with_intermediates, the masked trace ("masked") and the HF / LF correlograms ("corr")."""
        torch = self.torch
        with torch.cuda.device(self.device):
            y = self._filtered(raw)
            masked = _improcess.gabor_detect(y, self.fs, self.dx, self.selected_channels, c0=self.c0,
                                             bin_factor=self.bin_factor, threshold=self.threshold, threshold2=self.threshold2)
            del y
            corr = _rows.cross_correlogram_same(masked, self.templates)
            out = self._pick(corr, with_snr)
            if with_intermediates:
                out["masked"], out["corr"] = masked, corr
            return out


KERNEL_HF = {"f0": 27., "f1": 17., "dur": 0.8, "bdwidth": 4.}          # scripts/main_spectrodetect.py:103
KERNEL_LF = {"f0": 20., "f1": 14., "dur": 1.2, "bdwidth": 4.}          # :104


class SpectroDetectPipeline(_FilePipeline):
    """scripts/main_spectrodetect.py:39-123 on the device; the script's values are the defaults (flims = the band-pass band
    fmin .. fmax, :102).  Same interface as MfDetectPipeline (process_device / process_file / stream).  Picks are STFT frame
    indices; `spectro_fs` (frames per second, :123) converts them to seconds, `nt` is the number of frames per channel."""

    def __init__(self, nx, ns, selected_channels, dx, fs, scale_factor, device=None, fmin=14., fmax=30.,
                 mask_speeds=(1350., 1450., 3300, 3450), kernel_hf=None, kernel_lf=None, win_size=0.8, overlap_pct=0.95,
                 threshold=14., prune_eps=0.0, bandpass=True):
        super().__init__(nx, ns, selected_channels, dx, fs, scale_factor, device, fmin, fmax, mask_speeds, None,
                         prune_eps, bandpass)
        self.kernels = [dict(KERNEL_HF if kernel_hf is None else kernel_hf), dict(KERNEL_LF if kernel_lf is None else kernel_lf)]
        self.flims = (float(fmin), float(fmax))
        self.win_size, self.overlap_pct = float(win_size), float(overlap_pct)
        self.threshold = float(threshold)
        self.nperseg, self.nhop, self.bands, self.union, self.per_kernel = _detect.spectrocorr_layout(
            self.fs, self.flims, self.kernels, self.win_size, self.overlap_pct, self.ns)
        self.nt = 1 + self.ns // self.nhop
        self.spectro_fs = self.nt / ((self.ns - 1) / self.fs)                # nt / time[-1], time = arange(ns) / fs

    def process_device(self, raw, with_snr=False, with_intermediates=False):
        """raw: int32 (or float32) CUDA tensor [nx, ns] of interrogator counts.  Returns a dict of DEVICE results:
        picks_hf / picks_lf = (offsets int32 [nx + 1], idx int32 [n]) in frames, maxv (0-dim tensor), threshold, optionally
        snr_hf / snr_lf (snr_tr_array(env=True) of each correlogram, :113-114) and, with_intermediates, the HF / LF
        correlograms ("corr", [nx, nt] each)."""
        torch = self.torch
        with torch.cuda.device(self.device):
            y = self._filtered(raw)
            corr = _detect._spectrocorr_device(y, self.nperseg, self.nhop, self.union, self.per_kernel)
            del y
            out = {"maxv": self._maxv(corr), "threshold": self.threshold}             # :108
            for name, c in zip(("hf", "lf"), corr):
                out["picks_" + name] = _rows.find_peaks_device(c, self.threshold)    # pick_times, :117-118
                if with_snr:
                    out["snr_" + name] = _rows.snr(c, env=True)
            if with_intermediates:
                out["corr"] = corr
            return out


class NoiseProfilePipeline(_FilePipeline):
    """scripts/main_bathynoise.py:122-259 on the device; the script's values are the defaults.  The same front end as the
    detectors, then the per-channel noise profile of dsp.cable_noise_profile: two rows.env_stats passes (the whole rows and
    the noise window tnoise, int(t * fs) samples), so only [nx]-long vectors leave the GPU.  process_file / stream yield
    dicts of float64 ndarrays keyed by dsp.NOISE_PROFILE_KEYS."""

    def __init__(self, nx, ns, selected_channels, dx, fs, scale_factor, device=None, fmin=14., fmax=30.,
                 mask_speeds=(1350., 1450., 3300, 3450), tnoise=(19., 26.), p_ref=1e-11, prune_eps=0.0, bandpass=True):
        self.i0, self.i1 = _dsp.noise_window(ns, fs, tnoise)
        self.p_ref = float(p_ref)
        super().__init__(nx, ns, selected_channels, dx, fs, scale_factor, device, fmin, fmax, mask_speeds, None,
                         prune_eps, bandpass)

    def process_device(self, raw, with_image=False):
        """raw: int32 (or float32) CUDA tensor [nx, ns] of interrogator counts.  Returns a dict of float64 CUDA tensors [nx]
        keyed by dsp.NOISE_PROFILE_KEYS and, with_image, "image" = |hilbert(trf_fk)| / std(trf_fk) (float32 [nx, ns], the
        t-x plot of :139)."""
        torch = self.torch
        with torch.cuda.device(self.device):
            y = self._filtered(raw)
            full = _rows.env_stats(y)
            win = _rows.env_stats(y, self.i0, self.i1 - self.i0)
            out = _dsp.noise_profile_from_stats(full, win, self.p_ref)
            if with_image:
                out["image"] = _rows.envelope_over_std(y)
            return out

    def _to_host(self, res):
        return {k: v.cpu().numpy() for k, v in res.items()}


def process_file(raw, metadata, selected_channels, **kw):
    """Convenience wrapper: raw [nx, ns] counts + the reference's metadata dict (data_handle.get_acquisition_parameters:
    fs, dx, scale_factor) -> picks of the HF and LF fin-whale notes."""
    nx, ns = raw.shape
    pipe = MfDetectPipeline(nx, ns, selected_channels, metadata["dx"], metadata["fs"], metadata["scale_factor"], **kw)
    return pipe.process_file(raw)


def process_file_gabor(raw, metadata, selected_channels, **kw):
    """Convenience wrapper of GaborDetectPipeline: raw [nx, ns] counts + the reference's metadata dict (fs, dx,
    scale_factor) -> picks of the HF and LF fin-whale notes of scripts/main_gabordetect.py."""
    nx, ns = raw.shape
    pipe = GaborDetectPipeline(nx, ns, selected_channels, metadata["dx"], metadata["fs"], metadata["scale_factor"], **kw)
    return pipe.process_file(raw)


def process_file_spectro(raw, metadata, selected_channels, **kw):
    """Convenience wrapper of SpectroDetectPipeline: raw [nx, ns] counts + the reference's metadata dict (fs, dx,
    scale_factor) -> frame-index picks of the HF and LF notes of scripts/main_spectrodetect.py."""
    nx, ns = raw.shape
    pipe = SpectroDetectPipeline(nx, ns, selected_channels, metadata["dx"], metadata["fs"], metadata["scale_factor"], **kw)
    return pipe.process_file(raw)


def process_file_noise(raw, metadata, selected_channels, **kw):
    """Convenience wrapper of NoiseProfilePipeline: raw [nx, ns] counts + the reference's metadata dict (fs, dx,
    scale_factor) -> the per-channel noise profile of scripts/main_bathynoise.py (float64 ndarrays)."""
    nx, ns = raw.shape
    pipe = NoiseProfilePipeline(nx, ns, selected_channels, metadata["dx"], metadata["fs"], metadata["scale_factor"], **kw)
    return pipe.process_file(raw)
