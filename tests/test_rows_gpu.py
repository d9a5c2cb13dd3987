"""GPU parity tests for the per-channel operators (matched filter, envelope / SNR, zero-phase
IIR, STFT) against the golden vectors of the unmodified reference and the float64 oracle.
Contract tolerance: max-norm relative error <= 1e-4 (fp32 kernels)."""
import numpy as np
import pytest

from conftest import rel_err
from oracle import dsp_oracle as O, detect_oracle as D

pytestmark = pytest.mark.gpu
FS = 200.0
TOL = 1e-4


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available()
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def test_cross_correlogram_golden(dw, golden):
    g = golden("matched_filter")
    x = g["x"]
    for tag in ("hf", "lf"):
        out = dw.detect.compute_cross_correlogram(x, g["tpl_" + tag])
        assert out.shape == x.shape and out.dtype == np.float64
        e = rel_err(out, g["corr_" + tag])
        assert e[0] <= 2e-5, (tag, e)
    both = dw.detect.compute_cross_correlograms(x, [g["tpl_hf"], g["tpl_lf"]])
    assert rel_err(both[0], g["corr_hf"])[0] <= 2e-5 and rel_err(both[1], g["corr_lf"])[0] <= 2e-5
    a = np.array([1., 2, 3, 4, 5]); b = np.array([2., 1, 0, -1, 2])
    assert rel_err(dw.detect.shift_xcorr(a, b), g["sx"])[0] <= 1e-5
    assert rel_err(dw.detect.shift_nxcorr(a, b), g["snx"])[0] <= 1e-5


@pytest.mark.parametrize("nx,ns", [(7, 1500), (33, 12000), (5, 120000)])
def test_cross_correlogram_vs_oracle(dw, nx, ns):
    rng = np.random.default_rng(ns)
    x = (rng.standard_normal((nx, ns)) + 0.3).astype(np.float32)     # non-zero mean exercises the mu term
    time = np.arange(ns) / FS
    hf = D.gen_template_fincall(time, FS, 17.8, 28.8, 0.68)
    lf = D.gen_template_fincall(time, FS, 14.7, 21.8, 0.78)
    assert rel_err(dw.detect.gen_template_fincall(time, FS, 17.8, 28.8, 0.68), hf)[0] == 0
    outs = dw.detect.compute_cross_correlograms(x, [hf, lf])
    for o, t in zip(outs, (hf, lf)):
        ref = D.compute_cross_correlogram(x.astype(np.float64), t)
        e = rel_err(o, ref)
        assert e[0] <= 2e-5 and e[1] <= 2e-5, e


def test_envelope_and_picks_golden(dw, golden):
    g = golden("matched_filter")
    for tag in ("hf", "lf"):
        env = dw.detect.envelope(g["corr_" + tag])
        assert rel_err(env, g["env_" + tag])[0] <= 2e-5
        picks = dw.detect.convert_pick_times(dw.detect.pick_times_env(g["corr_" + tag], 0.05))
        ref = g["picks_" + tag]
        # fp32 envelope: allow a pick to move only if it sat exactly at the prominence threshold
        assert picks.shape[1] >= 1 and abs(picks.shape[1] - ref.shape[1]) <= 1
        if picks.shape == ref.shape:
            assert np.array_equal(picks, ref)


def test_snr_golden_and_kat(dw, golden):
    s = golden("snr")
    out = dw.dsp.snr_tr_array(s["kat_in"])                       # reference KAT tests/test_dsp.py:136-141
    assert np.allclose(out[0], [-3.01029996, 3.01029996, 6.53212514, 9.03089987, 10.96910013], atol=1e-5)
    for env in (0, 1):
        out = dw.dsp.snr_tr_array(s["x"], env=bool(env))
        ref = s[f"snr_env{env}"]
        # dB values: compare in the linear domain (10**(dB/10)), relative to the row peak
        lin, lref = 10 ** (out / 10), 10 ** (ref / 10)
        assert rel_err(lin, lref)[0] <= TOL, env


HILBERT_ROUTES = [{}, {"D4W_ROW_FUSED": "0"}, {"D4W_HILBERT_PAIR": "0"}, {"D4W_ROW_FUSED": "0", "D4W_HILBERT_PAIR": "0"}]


@pytest.mark.parametrize("env", HILBERT_ROUTES)
def test_envelope_routes_agree(dw, monkeypatch, env):
    """Every route of the split-row Hilbert transform (two real rows per complex transform or one per row; middle pass
    k_row_mid_fused, the default here, or k_row_mid) gives the oracle's envelope and SNR, an odd row count included."""
    from das4whales_b200 import _lib, rows
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setattr(rows, "_row_plans", {})                  # plans read the options when they are created
    nx, ns = 5, 120000
    x = np.random.default_rng(11).standard_normal((nx, ns)).astype(np.float32)
    L = _lib.lib()
    try:
        env_ = dw.detect.envelope(x)
        snr = dw.dsp.snr_tr_array(x, env=True)
        (plan,) = rows._row_plans.values()
        ws = L.d4w_row_workspace_bytes(plan.ptr, nx)
    finally:
        for p in rows._row_plans.values():
            L.d4w_row_plan_destroy(p.ptr)
    pair = env.get("D4W_HILBERT_PAIR", "1") != "0"
    assert ws == ((nx + 1) // 2 if pair else nx) * ns * 8
    assert rel_err(env_, D.envelope(x.astype(np.float64)))[0] <= 2e-5
    ref = O.snr_tr_array(x.astype(np.float64), env=True)
    assert rel_err(10 ** (snr / 10), 10 ** (ref / 10))[0] <= TOL


@pytest.mark.parametrize("ns", [600, 12000, 36000, 120000])
def test_envelope_vs_oracle_lengths(dw, ns):
    rng = np.random.default_rng(ns)
    x = rng.standard_normal((3, ns)).astype(np.float32)
    env = dw.detect.envelope(x)
    assert rel_err(env, D.envelope(x.astype(np.float64)))[0] <= 2e-5
    snr = dw.dsp.snr_tr_array(x, env=True)
    ref = O.snr_tr_array(x.astype(np.float64), env=True)
    assert rel_err(10 ** (snr / 10), 10 ** (ref / 10))[0] <= TOL


def test_iir_golden(dw, golden):
    g = golden("iir")
    x = g["bp_x"]
    y = dw.dsp.bp_filt(x, FS, 14, 30)
    e = rel_err(y, g["bp_y"])
    assert e[0] <= TOL, e
    sos = dw.dsp.butterworth_filter([5, [10, 30], "bp"], FS)
    assert rel_err(sos, g["sos_bp5"])[0] <= 1e-14
    assert rel_err(dw.dsp.sosfiltfilt(sos, x), g["sos_bp5_y"])[0] <= TOL
    assert rel_err(dw.dsp.sosfiltfilt(g["sos_hp2"], x), g["sos_hp2_y"])[0] <= TOL
    with pytest.raises(ValueError):      # SciPy: input must be longer than padlen
        dw.dsp.bp_filt(np.zeros((2, 40)), FS, 14, 30)


@pytest.mark.parametrize("nx,ns", [(70, 12000), (33, 5003), (5, 60000)])
def test_bp_filt_vs_oracle(dw, nx, ns):
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((nx, ns)) + np.linspace(0, 2, ns)[None, :]).astype(np.float32)   # trend stresses the edges
    y = dw.dsp.bp_filt(x, FS, 14, 30)
    ref = O.bp_filt(x.astype(np.float64), FS, 14, 30)
    e = rel_err(y, ref)
    assert e[0] <= TOL and e[1] <= TOL, e


@pytest.mark.parametrize("nfft,ov", [(128, 0.8), (256, 0.95), (256, 0.9), (160, 0.95)])
def test_get_spectrogram_vs_oracle(dw, nfft, ov):
    rng = np.random.default_rng(nfft)
    y = rng.standard_normal(12000).astype(np.float32)
    p, tt, ff = dw.dsp.get_spectrogram(y, FS, nfft=nfft, overlap_pct=ov)
    pr, ttr, ffr = O.get_spectrogram(y.astype(np.float64), FS, nfft=nfft, overlap_pct=ov)
    assert p.shape == pr.shape and np.allclose(tt, ttr) and np.allclose(ff, ffr)
    assert rel_err(10 ** (p / 20), 10 ** (pr / 20))[0] <= 2e-5


def test_stft_batched(dw):
    import torch
    from das4whales_b200 import rows
    rng = np.random.default_rng(3)
    x = rng.standard_normal((9, 6000)).astype(np.float32)
    mag = rows.stft_mag(torch.from_numpy(x).cuda(), 160, 8).cpu().numpy()
    for i in (0, 4, 8):
        ref = np.abs(O.stft_librosa(x[i].astype(np.float64), 160, 8))
        assert mag[i].shape == ref.shape
        assert rel_err(mag[i], ref)[0] <= 2e-5


def test_spectrocorr_pieces_golden(dw, golden):
    g = golden("spectrocorr")
    _, _, ker = dw.detect.buildkernel(27., 16., 4., 0.9, g["ff"], g["tt"], FS, 12., 36.)
    assert rel_err(ker, g["ker"])[0] <= 1e-14
    out = dw.detect.xcorr2d(g["S"], g["ker"])
    assert rel_err(out, g["xc2d"])[0] <= 2e-5


@pytest.mark.parametrize("kern", [{'f0': 27., 'f1': 17., 'dur': 0.8, 'bdwidth': 4.}, {'f0': 20., 'f1': 14., 'dur': 1.2, 'bdwidth': 4.}])
def test_spectrocorr_detector_vs_oracle(dw, kern):
    """scripts/main_spectrodetect.py:100-107 parameters on a small synthetic matrix."""
    rng = np.random.default_rng(11)
    x = rng.standard_normal((6, 9000)).astype(np.float32)
    flims = [14., 30.]
    out = dw.detect.compute_cross_correlogram_spectrocorr(x, FS, flims, kern, 0.8, 0.95)
    ref = D.compute_cross_correlogram_spectrocorr(x.astype(np.float64), FS, flims, kern, 0.8, 0.95)
    assert out.shape == ref.shape
    e = rel_err(out, ref)
    assert e[0] <= TOL and e[1] <= TOL, e
    # the single-trace helper keeps the reference's return order (spectrogram, ff, tt)
    p, ff, tt = dw.detect.get_sliced_nspectrogram(x[0], FS, 2., 32., 160, 8)
    pr, ffr, ttr = D.get_sliced_nspectrogram(x[0].astype(np.float64), FS, 2., 32., 160, 8)
    assert p.shape == pr.shape and np.allclose(ff, ffr) and np.allclose(tt, ttr)
    assert rel_err(p, pr)[0] <= 2e-5


def test_row_median_exact(dw):
    import torch
    from das4whales_b200 import rows
    rng = np.random.default_rng(5)
    for n in (7, 1000, 4097, 150001):
        a = np.abs(rng.standard_normal((3, n))).astype(np.float32)
        a[1, : n // 3] = 0.25                     # many ties
        med = rows.row_median(torch.from_numpy(a).cuda()).cpu().numpy()
        assert np.array_equal(med, np.median(a, axis=1).astype(np.float32)), n


@pytest.mark.parametrize("n", [16385, 200000, 300001, 465031, 700001])
def test_row_median_bracketed_select(dw, n):
    """Rows longer than the shared buffer: sample bracket + one collection pass (k_row_median), incl. the cases that must
    fall back to the radix select over the whole row (ties overflowing the bracket, constant rows)."""
    import torch
    from das4whales_b200 import rows
    rng = np.random.default_rng(n)
    a = np.stack([
        np.abs(rng.standard_normal(n) + 1j * rng.standard_normal(n)),      # Rayleigh, like |STFT| of noise
        rng.standard_cauchy(n) ** 2,                                       # heavy tail
        np.floor(rng.random(n) * 5),                                       # five distinct values: the bracket overflows
        np.where(rng.random(n) < 0.6, 0.0, rng.random(n)),                 # median inside a block of zeros
        np.full(n, 2.5),
        np.sort(rng.random(n)),                                            # monotone: systematic sample = exact quantiles
    ]).astype(np.float32)
    med = rows.row_median(torch.from_numpy(a).cuda()).cpu().numpy()
    assert np.array_equal(med, np.median(a, axis=1).astype(np.float32))


@pytest.mark.parametrize("nfft,hop,b0,b1,ns", [(160, 8, 2, 32, 9000), (160, 8, 0, 30, 9001), (160, 8, 50, 80, 12345),
                                               (160, 8, 12, 24, 120000), (160, 8, 30, 30, 2000), (160, 8, 14, 20, 7),
                                               (128, 8, 3, 18, 4000), (128, 8, 27, 64, 6001), (256, 16, 20, 27, 5000)])
def test_stft_sliding_dft_band(dw, nfft, hop, b0, b1, ns):
    """d4w_stft_slide (sliding DFT over a band of bins) vs the fp64 restatement of librosa.stft and vs the per-frame FFT
    kernel; row 1 carries a strong out-of-band tone (the rectangular-window recursion sees its leakage, the Hann
    combination has to cancel it)."""
    import os
    import torch
    from das4whales_b200 import rows, _lib
    assert _lib.lib().d4w_stft_slide_supported(nfft, hop, b1 - b0 + 1) == 1
    rng = np.random.default_rng(ns)
    x = rng.standard_normal((4, ns)).astype(np.float32)
    x[1] += (50 * np.sin(2 * np.pi * 0.7 * np.arange(ns) / FS)).astype(np.float32)
    x[2] += 1000.0                                                          # DC offset
    xd = torch.from_numpy(x).cuda()
    got = rows.stft_mag(xd, nfft, hop, b0, b1).cpu().numpy()
    os.environ["D4W_STFT_SLIDE"] = "0"
    try:
        fft_path = rows.stft_mag(xd, nfft, hop, b0, b1).cpu().numpy()
    finally:
        del os.environ["D4W_STFT_SLIDE"]
    assert got.shape == fft_path.shape == (4, b1 - b0 + 1, 1 + ns // hop)
    for i in range(4):
        full = np.abs(O.stft_librosa(x[i].astype(np.float64), nfft, hop))
        ref = full[b0:b1 + 1]
        scale = max(ref.max(), 1e-30) if i != 2 else full.max()           # the DC row is judged against its full spectrum
        assert np.abs(got[i] - ref).max() / scale <= 2e-5, (i, np.abs(got[i] - ref).max() / scale)
        assert np.abs(fft_path[i] - ref).max() / scale <= 2e-5


def test_stft_sliding_dft_not_used_outside_its_shapes(dw):
    from das4whales_b200 import _lib
    L = _lib.lib()
    assert L.d4w_stft_slide_supported(160, 8, 81) == 0        # whole spectrum: the per-frame FFT is cheaper
    assert L.d4w_stft_slide_supported(160, 40, 13) == 0       # 75 % overlap
    assert L.d4w_stft_slide_supported(100, 5, 13) == 0


def test_sosfiltfilt_chunked_equals_sequential(dw):
    """Time-chunked recursion (warm-up from the slowest pole) vs the plain sequential kernel."""
    import os
    import subprocess
    import sys
    import torch
    from das4whales_b200 import rows
    rng = np.random.default_rng(8)
    x = torch.from_numpy((rng.standard_normal((40, 30000)) + 5.0).astype(np.float32)).cuda()    # DC offset stresses the start-up
    for spec in ([8, [14, 30], "bp"], [2, 5, "hp"], [5, [10, 30], "bp"]):
        sos = dw.dsp.butterworth_filter(spec, FS)
        y = rows.sosfiltfilt(sos, x).cpu().numpy()
        import scipy.signal as sps
        ref = sps.sosfiltfilt(sos, x.cpu().numpy().astype(np.float64), axis=1)
        assert rel_err(y, ref)[0] <= 2e-5, spec


def _scipy_picks(x32, thr):
    import scipy.signal as sps
    return [sps.find_peaks(np.asarray(r, dtype=np.float64), prominence=thr)[0] for r in x32]


def test_find_peaks_golden_ties_and_plateaus(dw, golden):
    """Device find_peaks(prominence) == the reference's picks, index for index, on rows built to have exact ties,
    flat tops, a constant row, a monotone row and a long plateau (values are exactly representable in float32)."""
    g = golden("picks")
    x = g["x"]
    for thr in (0.0, 0.4, 2.0):
        got = dw.detect.pick_times(x, thr)
        ref = _scipy_picks(x.astype(np.float32), thr)
        assert len(got) == x.shape[0]
        for a, b in zip(got, ref):
            assert a.dtype == np.int64 and np.array_equal(a, b)
        if thr != 2.0:     # multiples of 1/3: a prominence of exactly 2.0 is rounding-marginal in float64 and in float32
            assert np.array_equal(dw.detect.convert_pick_times(got), g[f"picks_thr{thr}"])


@pytest.mark.parametrize("ns", [2, 3, 64, 65, 4097, 120000])
def test_find_peaks_vs_scipy_random(dw, ns):
    """Bit-exact index parity with scipy.signal.find_peaks on the same float32 rows: white noise (many shallow peaks),
    a smooth envelope-like row (few, wide peaks -> long prominence walks over blocks and superblocks), quantised rows."""
    import torch
    rng = np.random.default_rng(ns)
    rows = [rng.standard_normal(ns), np.abs(np.sin(np.arange(ns) * 0.003)) * (1 + 0.1 * rng.standard_normal(ns)),
            np.round(rng.standard_normal(ns) * 2) / 2, np.full(ns, 1.5), np.arange(ns, dtype=np.float64),
            np.concatenate([np.zeros(ns // 2), np.ones(ns - ns // 2)])]
    x = np.stack(rows).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    for thr in (0.0, 0.3, 1.0, 5.0):
        got = dw.rows.find_peaks(xd, thr)
        ref = _scipy_picks(x, thr)
        for r, (a, b) in enumerate(zip(got, ref)):
            assert np.array_equal(a, b), (ns, thr, r, len(a), len(b))


def test_pick_times_env_pipeline_vs_oracle(dw, golden):
    """Envelope (fp32 on the device) + device picking against the float64 reference picks: identical away from
    threshold-marginal peaks; at least 99 % of the reference picks must be reproduced exactly."""
    g = golden("matched_filter")
    for tag in ("hf", "lf"):
        got = dw.detect.convert_pick_times(dw.detect.pick_times_env(g["corr_" + tag], 0.05))
        ref = g["picks_" + tag]
        gs, rs = set(map(tuple, got.T.tolist())), set(map(tuple, ref.T.tolist()))
        assert len(gs & rs) >= 0.99 * len(rs) and len(gs) <= 1.01 * len(rs) + 1


def test_raw2strain_golden(dw, golden):
    import torch
    r = golden("raw2strain")
    meta = {"scale_factor": float(r["scale_factor"])}
    out = dw.data_handle.raw2strain(r["raw"], meta)                       # int32 ndarray -> float64 ndarray
    assert out.dtype == np.float64 and rel_err(out, r["strain"])[0] <= 1e-6
    outd = dw.data_handle.raw2strain(torch.from_numpy(r["raw"]).cuda(), meta)
    assert outd.dtype == torch.float32 and rel_err(outd.cpu().numpy(), r["strain"])[0] <= 1e-6
    f = r["raw"].astype(np.float64)
    ret = dw.data_handle.raw2strain(f, meta)
    assert ret is f and rel_err(f, r["strain"])[0] <= 1e-6                # in place for float arrays, like the reference
