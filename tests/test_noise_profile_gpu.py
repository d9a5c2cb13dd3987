"""GPU tests of the cable noise profile: rows.env_stats (d4w_env_stats: row statistics, d4w_hilbert's envelope, row
statistics and median of the envelope, composed on a workspace) on every Hilbert route it sits on -- whole rows in one CTA,
chirp-z rows in one CTA, split rows two per transform -- and dsp.cable_noise_profile and pipeline.NoiseProfilePipeline,
all against the float64 restatement of scripts/main_bathynoise.py:183-259 (oracle/noise_oracle.py).

Tolerances: the envelope is computed in fp32, so every linear quantity (envelope median and mean, mean, std) is held to
1e-4 relative per channel and 1e-5 in max-norm over channels; a perturbed row's median moves by at most the largest
perturbation of its envelope, so the envelope's error bounds the median's.  The dB quantities are held to 1e-3 dB."""
import numpy as np
import pytest
import scipy.signal as sps

from oracle import noise_oracle as N

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available()
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _strain(nx, ns, seed, zero_row=None):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((nx, ns)) * np.linspace(0.5, 2.0, nx)[:, None]
    t = np.arange(ns) / FS
    for i in range(0, nx, 3):                                   # a 25 -> 16 Hz sweep in every third channel
        t0 = (i * 0.37) % max(0.1, t[-1] - 1.0)
        m = (t >= t0) & (t < t0 + 1.0)
        x[i, m] += 4 * sps.chirp(t[m] - t0, f0=25, f1=16, t1=1.0, method="hyperbolic") * np.hanning(m.sum())
    if zero_row is not None:
        x[zero_row] = 0.0
    return (x * 1e-9).astype(np.float32)


def _check_linear(got, ref, what):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    den = np.abs(ref)
    per = np.where(den > 0, err / np.where(den > 0, den, 1.0), err)
    assert np.all(per <= 1e-4), (what, float(per.max()))
    assert err.max() <= 1e-5 * max(den.max(), 1e-300), (what, float(err.max() / den.max()))


def _check_record(rec, x64):
    ref = N.env_stats(x64)
    assert rec.shape == ref.shape == (x64.shape[0], 5)
    for j, name in enumerate(("median_env", "mean_env")):
        _check_linear(rec[:, j], ref[:, j], name)
    _check_linear(np.sqrt(rec[:, 4]), np.sqrt(ref[:, 4]), "std")
    _check_linear(np.sqrt(rec[:, 3]), np.sqrt(ref[:, 3]), "rms")
    # the mean of a zero-mean row is a difference of large sums: hold it to the row's scale
    scale = np.sqrt(ref[:, 3])
    assert np.all(np.abs(rec[:, 2] - ref[:, 2]) <= 1e-6 * np.where(scale > 0, scale, 1.0))


def _route(dw, n):
    """the Hilbert route d4w_hilbert takes for rows of n samples"""
    t1, _, m = dw.rows.row_plan(n, 0).info()
    return ("whole" if t1 == 1 else "split") + ("_czt" if m else "")


# (nx, ns, t0, n, route): whole rows and windows read in place at an offset, odd and even n, windows ending at ns
CASES = [
    (6, 1400, 0, None, "whole"),
    (6, 12000, 0, None, "whole"),
    (5, 16384, 0, None, "whole"),
    (6, 12000, 3800, 1400, "whole"),                  # the script's noise window of a 60 s record
    (6, 12000, 12000 - 1401, 1401, "whole_czt"),     # odd chirp-z window ending at ns
    (6, 1401, 0, None, "whole_czt"),
    (6, 4099, 0, None, "whole_czt"),
    (4, 9000, 117, 4099, "whole_czt"),
    (6, 12000, 975, 11025, "whole"),                  # odd direct window ending at ns
    (3, 16385, 0, None, "split_czt"),
    (2, 120000, 0, None, "split"),
    (3, 40000, 3000, 17000, "split"),                 # strided long window
    (3, 20000, 20000 - 16385, 16385, "split_czt"),    # strided long window ending at ns
]


@pytest.mark.parametrize("nx,ns,t0,n,route", CASES)
def test_env_stats_matches_oracle(dw, nx, ns, t0, n, route):
    import torch
    nn = ns - t0 if n is None else n
    assert _route(dw, nn) == route
    x = _strain(nx, ns, ns + t0, zero_row=1)
    rec = dw.rows.env_stats(torch.from_numpy(x).cuda(), t0, n)
    assert rec.dtype == torch.float64 and rec.is_cuda and tuple(rec.shape) == (nx, 5)
    rec = rec.cpu().numpy()
    assert np.all(rec[1] == 0.0)                                                   # the zero channel
    _check_record(rec, x[:, t0:t0 + nn].astype(np.float64))


def test_window_in_place_equals_the_copied_window(dw):
    """a window read in place at ld = ns gives bit for bit what the same samples give as a dense matrix"""
    import torch
    x = torch.from_numpy(_strain(5, 20000, 3)).cuda()
    for t0, n in ((2000, 16384), (3616, 16384), (100, 1401), (19999 - 16385, 16385)):
        a = dw.rows.env_stats(x, t0, n)
        b = dw.rows.env_stats(x[:, t0:t0 + n].contiguous())
        assert torch.equal(a, b), (t0, n)


def test_record_is_the_public_calls_bit_for_bit(dw):
    """the record is what rows.row_stats, rows.envelope, rows.row_stats of the envelope and rows.row_median give, bit for bit"""
    import torch
    for n in (1401, 16384, 20000):
        x = torch.from_numpy(_strain(8, n, n)).cuda()
        rec = dw.rows.env_stats(x)
        env = dw.rows.envelope(x)
        st, _ = dw.rows.row_stats(x)
        ste, _ = dw.rows.row_stats(env)
        mean, var = st[:, 0], st[:, 2]
        want = torch.stack([dw.rows.row_median(env).double(), ste[:, 0], mean, var + mean * mean, var], dim=1)
        assert torch.equal(rec, want), n


def test_more_than_65535_long_rows_through_the_abi(dw):
    """d4w_env_stats splits a call into passes of at most 65 535 rows.  For rows this long rows.env_stats never hands it that
    many (its 8 GB workspace cap is fewer rows), so the C entry point is called directly"""
    import torch
    from das4whales_b200 import _lib
    nx, n = 65537, 16385
    assert _route(dw, n) == "split_czt"
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn((nx, n), device="cuda", generator=g)
    x[65535] = 0.0                                                 # a zero channel as the first row of the second pass
    plan = dw.rows.row_plan(n, 0)
    L = _lib.lib()
    wsb = int(L.d4w_env_stats_workspace_bytes(plan.ptr, nx, n))
    assert wsb == int(L.d4w_env_stats_workspace_bytes(plan.ptr, 65535, n)) > 0
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    out = torch.empty((nx, 5), dtype=torch.float64, device="cuda")
    _lib.check(L.d4w_env_stats(plan.ptr, _lib.ptr(x, "float*"), nx, n, _lib.ptr(out, "double*"), _lib.ptr(ws),
                               _lib.stream_ptr()), "env_stats")
    rows_ = [0, 1, 65533, 65534, 65535, 65536]
    rec = out[rows_].cpu().numpy()
    assert np.all(rec[4] == 0.0)
    _check_record(rec, x[rows_].double().cpu().numpy())


def test_env_stats_of_no_rows(dw):
    import torch
    for ns in (1400, 16385):
        out = dw.rows.env_stats(torch.zeros((0, ns), dtype=torch.float32, device="cuda"))
        assert tuple(out.shape) == (0, 5) and out.dtype == torch.float64


def test_more_than_65535_rows(dw):
    import torch
    nx, ns = 70000, 64
    rng = np.random.default_rng(4)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    rec = dw.rows.env_stats(torch.from_numpy(x).cuda()).cpu().numpy()
    rows_ = [0, 1, 65534, 65535, 65536, nx - 1]
    _check_record(rec[rows_], x[rows_].astype(np.float64))
    part = dw.rows.env_stats(torch.from_numpy(x[65530:65540]).cuda()).cpu().numpy()
    assert np.array_equal(rec[65530:65540], part)


def test_env_stats_rejects_bad_windows(dw):
    import torch
    x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
    for t0, n in ((-1, 10), (0, 0), (95, 6), (100, 1)):
        with pytest.raises(ValueError):
            dw.rows.env_stats(x, t0, n)


def _check_profile(prof, ref, keys):
    for k in keys:
        g, r = np.asarray(prof[k], dtype=np.float64), np.asarray(ref[k], dtype=np.float64)
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(g), fin) and np.array_equal(np.isnan(g), np.isnan(r)), k
        assert np.array_equal(g[np.isinf(r)], r[np.isinf(r)]), k
        if k in ("SNR_1d", "noise_power_db"):
            assert np.all(np.abs(g[fin] - r[fin]) <= 1e-3), (k, float(np.abs(g[fin] - r[fin]).max()))
        elif k == "noise_power":
            _check_linear(np.sqrt(g), np.sqrt(r), k)
        elif k == "std_med_diff":                      # a difference: bounded by its terms' errors
            assert np.all(np.abs(g - r) <= 1e-4 * (np.asarray(ref["std"]) + np.asarray(ref["med"]))), k
        else:
            _check_linear(g, r, k)


@pytest.mark.parametrize("ns,tnoise", [(12000, (19., 26.)), (6001, (20., 30.005))])
def test_cable_noise_profile_ndarray_and_tensor(dw, ns, tnoise):
    import torch
    x = _strain(9, ns, 7, zero_row=4)
    ref = N.cable_noise_profile(x.astype(np.float64), FS, tnoise)
    prof = dw.dsp.cable_noise_profile(x, FS, tnoise)
    assert tuple(prof) == dw.dsp.NOISE_PROFILE_KEYS
    for k, v in prof.items():
        assert isinstance(v, np.ndarray) and v.dtype == np.float64 and v.shape == (9,), k
    assert np.isnan(prof["SNR_1d"][4]) and prof["noise_power_db"][4] == -np.inf
    _check_profile(prof, ref, dw.dsp.NOISE_PROFILE_KEYS)
    pt = dw.dsp.cable_noise_profile(torch.from_numpy(x).cuda(), FS, tnoise)
    for k, v in pt.items():
        assert isinstance(v, torch.Tensor) and v.is_cuda and v.dtype == torch.float64, k
        # the same records; torch's and NumPy's log10 may differ in the last bit
        np.testing.assert_allclose(v.cpu().numpy(), prof[k], rtol=1e-14, atol=0, equal_nan=True, err_msg=k)
    with pytest.raises(ValueError):
        dw.dsp.cable_noise_profile(x, FS, (ns / FS, ns / FS + 1))


# ---------------------------------------------------------------------------------------------------- file pipeline
def _oracle_chain(raw, scale, sel):
    from oracle import data_oracle as DH, dsp_oracle as O
    nx, ns = raw.shape
    x = DH.raw2strain(raw, {"scale_factor": scale})
    x = O.bp_filt(x, FS, 14., 30.)
    m = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, 1350., 1450., 3300, 3450, 14., 30.)
    return O.fk_filter_filt(x, m)


def test_noise_pipeline_matches_oracle_chain(dw):
    """raw2strain -> bp_filt -> hybrid_ninf f-k -> profile against the float64 script chain.  The f-k filter's contract is
    a max-norm error e <= 1e-4 max|y|.  Every linear quantity is a mean, median or rms of the row or of its envelope; the
    envelope's perturbation |H e| has an rms <= sqrt(2) |e|_inf, so those are held to 2e-4 max|y| (absolute) and the
    noise power (quadratic) to 5e-4 max|y|^2; its dB value to 4.35 x that relative change."""
    import torch
    from das4whales_b200 import pipeline
    from oracle.make_golden import synth
    nx, ns, sel = 200, 6000, [0, 200, 1]
    x = synth(nx, ns, seed=21, ncalls=3)
    counts = np.round(x * 5.0e4).astype(np.int32) + 1234
    scale = 4.0838e-11 * 1550.0 / 2.0419
    y = _oracle_chain(counts, scale, sel)
    ref = N.cable_noise_profile(y, FS)
    ymax = float(np.abs(y).max())
    pipe = pipeline.NoiseProfilePipeline(nx, ns, sel, DX, FS, scale)
    assert (pipe.i0, pipe.i1) == (3800, 5200)
    dev = pipe.process_device(torch.from_numpy(counts).cuda(), with_image=True)
    assert set(dev) == set(dw.dsp.NOISE_PROFILE_KEYS) | {"image"}
    for k in ("med", "mean", "std", "std_med_diff", "noise_mean"):
        g = dev[k].cpu().numpy()
        assert dev[k].dtype == torch.float64 and g.shape == (nx,)
        assert np.abs(g - ref[k]).max() <= 2e-4 * ymax, (k, float(np.abs(g - ref[k]).max() / ymax))
    p = dev["noise_power"].cpu().numpy()
    dp = np.abs(p - ref["noise_power"])
    assert dp.max() <= 5e-4 * ymax ** 2
    assert np.all(np.abs(dev["noise_power_db"].cpu().numpy() - ref["noise_power_db"]) <= 4.35 * dp / ref["noise_power"] + 1e-9)
    snr = dev["SNR_1d"].cpu().numpy()
    rel = (np.abs(dev["std"].cpu().numpy() - ref["std"]) / ref["std"] + np.abs(dev["med"].cpu().numpy() - ref["med"]) / ref["med"])
    assert np.all(np.abs(snr - ref["SNR_1d"]) <= 8.7 * rel + 1e-9)
    img = dev["image"].cpu().numpy().astype(np.float64)
    img_ref = N.image(y)
    assert img.shape == (nx, ns)
    assert np.abs(img - img_ref).max() <= 2e-4 * ymax / ref["std"].min() * 1.5
    res = pipe.process_file(counts)
    assert set(res) == set(dw.dsp.NOISE_PROFILE_KEYS)
    for k in dw.dsp.NOISE_PROFILE_KEYS:
        assert isinstance(res[k], np.ndarray) and res[k].dtype == np.float64
        assert np.array_equal(res[k], dev[k].cpu().numpy()), k
    outs = list(pipe.stream([counts, counts.astype(np.float32), counts]))
    assert len(outs) == 3
    for o in outs:
        assert set(o) == set(dw.dsp.NOISE_PROFILE_KEYS)
        for k in dw.dsp.NOISE_PROFILE_KEYS:
            assert np.array_equal(o[k], res[k]), k
    one = pipeline.process_file_noise(counts, {"dx": DX, "fs": FS, "scale_factor": scale}, sel)
    for k in dw.dsp.NOISE_PROFILE_KEYS:
        assert np.array_equal(one[k], res[k]), k
    with pytest.raises(ValueError):
        pipeline.NoiseProfilePipeline(nx, ns, sel, DX, FS, scale, tnoise=(29., 31.))
