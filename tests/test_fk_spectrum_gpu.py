"""GPU: the f-k power spectrum (dsp.fk_spectrum, fk.FkSpectrum) against float64 |fftshift(fft2(x))|^2.

Every shape of tests/test_fk_routes_host.ROUTES (each column scheme and row route the planner picks from the shape
alone) and two chirp-z channel counts, whole plane and a band, plain and tapered; then the semantics of the public
function on a small shape: inclusive band edges, negative-frequency bands, the taper leaving the input untouched,
block averaging, output types, the support size, and every ValueError.  The 10 000 x 120 000 case compares the default
band with a float64 spectrum computed slab by slab on the same GPU, when enough device memory is free."""
import os

import numpy as np
import pytest
import scipy.signal as sps

from test_fk_routes_host import FIELDS, ROUTES

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
MAX_TOL, L2_TOL = 2e-5, 1e-5
CZT_SHAPES = [(4897, 1200), (7346, 1200)]


@pytest.fixture(scope="module")
def fk():
    """The routes shapes pick by themselves: no D4W_* variable, and no plan cached under another environment."""
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from das4whales_b200 import _lib, fk
    _lib.lib()
    with pytest.MonkeyPatch.context() as mp:
        for k in [k for k in os.environ if k.startswith("D4W_")]:
            mp.delenv(k)
        fk.free_plans()
        yield fk
        fk.free_plans()
    torch.cuda.empty_cache()


def _power64(x, tapering=False):
    """|fftshift(fft2(x))|^2 in float64 on the device."""
    import torch
    x64 = x.to(torch.float64)
    if tapering:
        x64 = x64 * torch.from_numpy(sps.windows.tukey(x.shape[1], alpha=0.03)).to(x.device)[None, :]
    return torch.fft.fftshift(torch.fft.fft2(x64)).abs() ** 2


def _errs(p, ref):
    import torch
    p = torch.as_tensor(p, device=ref.device).to(torch.float64)
    d = p - ref
    return float(d.abs().max() / ref.abs().max()), float(torch.linalg.vector_norm(d) / torch.linalg.vector_norm(ref))


def _check(p, ref, what):
    emax, el2 = _errs(p, ref)
    print(f"{what}: max-norm {emax:.2e}, l2 {el2:.2e}")
    assert emax <= MAX_TOL and el2 <= L2_TOL, (what, emax, el2)


def _rows_touching(nx, k_lo, k_hi):
    return sum(1 for k in range(nx // 2 + 1)
               if k_lo <= (k + nx // 2) % nx < k_hi or k_lo <= (nx - k + nx // 2) % nx < k_hi)


@pytest.mark.parametrize("nx,ns", sorted(ROUTES) + CZT_SHAPES)
def test_route_vs_float64(fk, nx, ns):
    import torch
    import das4whales_b200 as dw
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    if (nx, ns) in ROUTES:
        want = dict(zip(FIELDS, ROUTES[(nx, ns)]))
        assert (plan.col_scheme, plan.tile, plan.col_threads, plan.t1) == \
            (want["scheme"], 2 * want["nc"], want["col_threads"], want["t1"]), (nx, ns)
    else:
        assert plan.col_scheme == 4, (nx, ns)
    x = torch.randn(nx, ns, device="cuda", generator=torch.Generator(device="cuda").manual_seed(nx * 5 + ns))
    ref = _power64(x)
    whole = fk.FkSpectrum((nx, ns), (0, nx), (0, ns))
    assert whole.rows == nx // 2 + 1
    p = whole(x)
    assert torch.equal(p, whole(x)), "two runs differ"
    _check(p, ref, f"{nx} x {ns} scheme {plan.col_scheme} T1 {plan.t1}, whole plane")
    del p, whole
    # default band of dsp.fk_spectrum (f >= 0) restricted to |k| <= a third of the wavenumber range
    knum = np.fft.fftshift(np.fft.fftfreq(nx, DX))
    kmax = float(np.max(np.abs(knum))) / 3
    p, f, k = dw.dsp.fk_spectrum(x, [0, nx, 1], DX, FS, k_range=(-kmax, kmax))
    freq = np.fft.fftshift(np.fft.fftfreq(ns, 1 / FS))
    fi, ki = np.flatnonzero(freq >= 0), np.flatnonzero(np.abs(knum) <= kmax)
    assert np.array_equal(f, freq[fi]) and np.array_equal(k, knum[ki])
    _check(p, ref[ki[0]:ki[-1] + 1, fi[0]:fi[-1] + 1], f"{nx} x {ns}, f >= 0 and |k| <= {kmax:.4f}")
    del ref
    p = dw.dsp.fk_spectrum(x, [0, nx, 1], DX, FS, k_range=(-kmax, kmax), tapering=True)[0]
    _check(p, _power64(x, tapering=True)[ki[0]:ki[-1] + 1, fi[0]:fi[-1] + 1], f"{nx} x {ns}, band, tapered")
    fk.free_plans()
    torch.cuda.empty_cache()


NX, NS = 120, 1000          # even nx and ns: the Nyquist row and column exist


@pytest.fixture(scope="module")
def small(fk):
    rng = np.random.default_rng(11)
    return rng.standard_normal((NX, NS)).astype(np.float32)


def _np_power(x, tapering=False):
    x64 = x.astype(np.float64) * (sps.windows.tukey(x.shape[1], 0.03)[None, :] if tapering else 1.0)
    return np.abs(np.fft.fftshift(np.fft.fft2(x64))) ** 2


def _np_check(p, ref, what):
    d = p - ref
    emax, el2 = np.max(np.abs(d)) / np.max(ref), np.linalg.norm(d) / np.linalg.norm(ref)
    assert emax <= MAX_TOL and el2 <= L2_TOL, (what, emax, el2)


def test_band_edges_on_grid_values_are_inclusive(small):
    import das4whales_b200 as dw
    freq = np.fft.fftshift(np.fft.fftfreq(NS, 1 / FS))
    knum = np.fft.fftshift(np.fft.fftfreq(NX, DX))
    ref = _np_power(small)
    for (f0, f1), (k0, k1) in (((510, 600), (30, 81)), ((0, NS - 1), (0, NX - 1)), ((700, 702), (60, 62))):
        p, f, k = dw.dsp.fk_spectrum(small, [0, NX, 1], DX, FS, f_range=(freq[f0], freq[f1]), k_range=(knum[k0], knum[k1]))
        assert np.array_equal(f, freq[f0:f1 + 1]) and np.array_equal(k, knum[k0:k1 + 1])
        assert p.shape == (k1 + 1 - k0, f1 + 1 - f0)
        _np_check(p, ref[k0:k1 + 1, f0:f1 + 1], (f0, f1, k0, k1))


def test_default_and_negative_frequency_bands(small):
    import das4whales_b200 as dw
    freq = np.fft.fftshift(np.fft.fftfreq(NS, 1 / FS))
    ref = _np_power(small)
    p, f, k = dw.dsp.fk_spectrum(small, [0, NX, 1], DX, FS)
    assert f[0] == 0.0 and np.array_equal(f, freq[NS // 2:]) and len(k) == NX          # Nyquist (-fs/2) left out
    _np_check(p, ref[:, NS // 2:], "default")
    p, f, k = dw.dsp.fk_spectrum(small, [0, NX, 1], DX, FS, f_range=(-FS / 2, -10.0))
    sel = np.flatnonzero((freq >= -FS / 2) & (freq <= -10.0))
    assert f[0] == -FS / 2 and np.array_equal(f, freq[sel])
    _np_check(p, ref[:, sel[0]:sel[-1] + 1], "negative frequencies with the Nyquist column")


def test_tapering_leaves_the_input_untouched(small):
    import torch
    import das4whales_b200 as dw
    x = small.copy()
    p = dw.dsp.fk_spectrum(x, [0, NX, 1], DX, FS, f_range=(-np.inf, np.inf), tapering=True)[0]
    assert np.array_equal(x, small)
    _np_check(p, _np_power(small, tapering=True), "tapered ndarray")
    xt = torch.from_numpy(small).cuda()
    keep = xt.clone()
    pt = dw.dsp.fk_spectrum(xt, [0, NX, 1], DX, FS, f_range=(-np.inf, np.inf), tapering=True)[0]
    assert torch.equal(xt, keep)
    _np_check(pt.cpu().numpy().astype(np.float64), _np_power(small, tapering=True), "tapered tensor")


@pytest.mark.parametrize("tapering", [False, True])
def test_nperseg_is_the_mean_of_whole_blocks(small, tapering):
    import torch
    import das4whales_b200 as dw
    L = 300                                              # three blocks; the last 100 samples are not used
    ref = np.mean([_np_power(small[:, b * L:(b + 1) * L], tapering) for b in range(NS // L)], axis=0)
    p, f, k = dw.dsp.fk_spectrum(small, [0, NX, 1], DX, FS, f_range=(-np.inf, np.inf), nperseg=L, tapering=tapering)
    assert p.shape == (NX, L) and np.array_equal(f, np.fft.fftshift(np.fft.fftfreq(L, 1 / FS)))
    _np_check(p, ref, "nperseg")
    pt = dw.dsp.fk_spectrum(torch.from_numpy(small).cuda(), [0, NX, 1], DX, FS, f_range=(-np.inf, np.inf), nperseg=L,
                            tapering=tapering)[0]
    _np_check(pt.cpu().numpy().astype(np.float64), ref, "nperseg tensor")
    p1 = dw.dsp.fk_spectrum(small, [0, NX, 1], DX, FS, nperseg=NS)[0]       # one block: the plain spectrum
    _np_check(p1, _np_power(small)[:, NS // 2:], "nperseg = ns")


def test_output_types(small):
    import torch
    import das4whales_b200 as dw
    p, f, k = dw.dsp.fk_spectrum(small, [0, NX, 1], DX, FS)
    assert isinstance(p, np.ndarray) and p.dtype == np.float64
    assert f.dtype == np.float64 and k.dtype == np.float64
    pt, ft, kt = dw.dsp.fk_spectrum(torch.from_numpy(small).cuda(), [0, NX, 1], DX, FS)
    assert isinstance(pt, torch.Tensor) and pt.is_cuda and pt.dtype == torch.float32
    assert np.array_equal(ft, f) and np.array_equal(kt, k)
    assert np.array_equal(pt.cpu().numpy().astype(np.float64), p)


@pytest.mark.parametrize("k_idx", [(0, NX), (NX // 2, NX // 2 + 1), (NX // 2 + 1, NX), (1, NX // 2), (0, 1), (10, 17),
                                   (100, 101)])
def test_rows_are_the_half_plane_rows_touching_the_band(fk, small, k_idx):
    import torch
    spec = fk.FkSpectrum((NX, NS), k_idx, (0, NS))
    assert spec.rows == _rows_touching(NX, *k_idx)
    p = spec(torch.from_numpy(small).cuda())
    _np_check(p.cpu().numpy().astype(np.float64), _np_power(small)[k_idx[0]:k_idx[1]], k_idx)


def test_value_errors(fk, small):
    import torch
    import das4whales_b200 as dw
    sel = [0, NX, 1]
    with pytest.raises(ValueError, match="selects no"):
        dw.dsp.fk_spectrum(small, sel, DX, FS, f_range=(150., 200.))
    with pytest.raises(ValueError, match="selects no"):
        dw.dsp.fk_spectrum(small, sel, DX, FS, k_range=(1.0, 2.0))
    for n in (0, -5, NS + 1):
        with pytest.raises(ValueError, match="nperseg"):
            dw.dsp.fk_spectrum(small, sel, DX, FS, nperseg=n)
    for bad in (small[0], small[None], small.astype(np.complex64)):
        with pytest.raises(ValueError, match="real 2-D"):
            dw.dsp.fk_spectrum(bad, sel, DX, FS)
    with pytest.raises(ValueError, match="real 2-D"):
        dw.dsp.fk_spectrum(torch.from_numpy(small.astype(np.complex64)).cuda(), sel, DX, FS)
    with pytest.raises(ValueError, match="supported_shape"):           # 67 samples: a prime factor above 61
        dw.dsp.fk_spectrum(np.zeros((40, 134)), [0, 40, 1], DX, FS)
    with pytest.raises(ValueError, match="supported_shape"):
        dw.dsp.fk_spectrum(small, sel, DX, FS, nperseg=67)
    for k_idx, f_idx in (((0, 0), (0, NS)), ((0, NX + 1), (0, NS)), ((0, NX), (5, 5)), ((-1, 3), (0, NS))):
        with pytest.raises(ValueError):
            fk.FkSpectrum((NX, NS), k_idx, f_idx)


# ---- full size -------------------------------------------------------------------------------------------------------
FX, FNS = 10000, 120000


def test_fullsize_default_band_vs_float64(fk):
    """10 000 x 120 000, f >= 0, every wavenumber, against a float64 spectrum computed on the GPU slab by slab (rfft over
    time per row slab, then the channel FFT per column slab), with the spectrum's plan released first."""
    import torch
    import das4whales_b200 as dw
    from das4whales_b200 import synth
    real, half = FX * FNS * 4, FX * (FNS // 2 + 1) * 16
    need = real + FX * (FNS // 2) * 4 + half + 8 * 1024 * FX * 16
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 1e9:.1f} GB of free device memory; {free / 1e9:.1f} GB are free")
    x = synth.synth_strain(FX, FNS, seed=99)
    p, f, k = dw.dsp.fk_spectrum(x, [0, FX, 1], DX, FS)
    assert p.shape == (FX, FNS // 2) and f[0] == 0.0
    fk.free_plans()
    torch.cuda.empty_cache()
    s = torch.empty((FX, FNS // 2 + 1), dtype=torch.complex128, device=x.device)
    for r0 in range(0, FX, 256):
        s[r0:r0 + 256] = torch.fft.rfft(x[r0:r0 + 256].to(torch.float64), dim=1)
    del x
    for c0 in range(0, FNS // 2, 1024):
        s[:, c0:c0 + 1024] = torch.fft.fft(s[:, c0:c0 + 1024], dim=0)
    dmax = rmax = dss = rss = 0.0
    for r0 in range(0, FX, 256):
        rows = torch.arange(r0, min(r0 + 256, FX), device=s.device)
        ref = s[(rows - FX // 2) % FX, :FNS // 2].abs() ** 2        # shifted row r holds k = r - nx/2
        d = p[r0:r0 + 256].to(torch.float64) - ref
        dmax, rmax = max(dmax, float(d.abs().max())), max(rmax, float(ref.max()))
        dss, rss = dss + float((d * d).sum()), rss + float((ref * ref).sum())
    emax, el2 = dmax / rmax, (dss / rss) ** 0.5
    print(f"full size {FX} x {FNS}, default band: max-norm {emax:.2e}, l2 {el2:.2e}")
    assert emax <= MAX_TOL and el2 <= L2_TOL, (emax, el2)
    del s, p
    torch.cuda.empty_cache()
