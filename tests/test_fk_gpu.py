"""GPU parity tests for the f-k filter (through das4whales_b200.dsp -> cffi -> C ABI -> CUDA)
against the float64 oracle and the committed golden vectors of the unmodified reference.
Tolerance (BASELINE.json north_star): max-norm relative error <= 1e-4 for fp32; the kernels
are expected ~1e-6, so the asserts use 2e-5 to catch regressions early."""
import numpy as np
import pytest

from conftest import rel_err
from oracle import dsp_oracle as O

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
TOL = 2e-5          # << the 1e-4 contract


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()      # must load the in-tree libd4w.so or fail loudly
    return dw


def test_golden_fixtures_dense_masks(dw, golden):
    """The reference's own outputs (tests/golden/fk_apply.npz) with the reference's dense masks."""
    g, gm = golden("fk_apply"), golden("masks")
    for tag in ("fan_even", "fan_odd", "fan_p19", "ninf_even", "hyb_even"):
        x, yref = g[tag + "_x"], g[tag + "_y"]
        m = gm[str(g[tag + "_mask"])]
        taper = bool(g[tag + "_taper"])
        xin = x.copy()
        y = dw.dsp.fk_filter_filt(xin, m, tapering=taper)
        assert y.dtype == np.float64 and y.shape == x.shape
        e = rel_err(y, yref)
        assert e[0] <= TOL and e[1] <= TOL, (tag, e)
        if taper:   # reference side effect: the caller's array is tapered in place (dsp.py:721,745)
            assert rel_err(xin, O.taper_data(x.copy()))[0] <= 1e-15
        else:
            assert np.array_equal(xin, x)
        if tag.startswith("fan"):
            ys = dw.dsp.fk_filter_sparsefilt(x.copy(), np.asfortranarray(m), tapering=taper)
            assert rel_err(ys, yref)[0] <= TOL


SHAPES = [(64, 400, 1), (63, 405, 1), (100, 1200, 1), (551, 1200, 2), (96, 18000, 1), (1024, 4096, 1),
          (3000, 6000, 1)]


@pytest.mark.parametrize("nx,ns,step", SHAPES)
def test_fan_mask_analytic_vs_oracle(dw, nx, ns, step):
    rng = np.random.default_rng(nx + ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    sel = [0, nx * step, step]
    mask = dw.dsp.fk_filter_design((nx, ns), sel, DX, FS)
    y = dw.dsp.fk_filter_filt(x, mask)
    mref = O.fk_filter_design((nx, ns), sel, DX, FS)
    ref = O.fk_filter_filt(x.astype(np.float64), mref)
    e = rel_err(y, ref)
    assert e[0] <= TOL and e[1] <= TOL, e
    if nx * ns <= 2_000_000:
        md = np.asarray(mask)
        assert md.flags["F_CONTIGUOUS"] and md.dtype == np.float64
        assert np.max(np.abs(md - mref)) <= 1e-12


@pytest.mark.parametrize("nx,ns", [(64, 400), (100, 1200), (551, 2400), (2000, 12000)])
def test_hybrid_ninf_vs_oracle(dw, nx, ns):
    rng = np.random.default_rng(7)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    sel = [0, nx, 1]
    args = (1350., 1450., 3300, 3450, 14., 30.)
    mask = dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *args)
    y = dw.dsp.fk_filter_sparsefilt(x.copy(), mask, tapering=True)   # tapering mutates its input like the reference
    mref = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *args)
    ref = O.fk_filter_filt(x.astype(np.float64), mref, tapering=True)
    e = rel_err(y, ref)
    assert e[0] <= TOL and e[1] <= TOL, e
    if nx * ns <= 2_000_000:
        assert np.max(np.abs(mask.todense() - mref)) <= 1e-12


T1_SPLITS = [(24000, 3), (36000, 4), (50000, 5), (60000, 6), (80000, 8), (100000, 10), (120000, 12), (150000, 15),
             (160000, 16), (200000, 20), (250000, 25)]


@pytest.mark.parametrize("ns,t1", T1_SPLITS)
def test_every_time_split_vs_oracle(dw, ns, t1):
    """Each length picks its own time split ns = T1 x T2 (T2 <= 10 240), so every k_row_split<T1> instantiation the
    planner can choose runs on the device (the config-2 length 120 000 is T1 = 12)."""
    import torch
    from das4whales_b200 import fk
    nx = 48
    assert fk.get_plan(nx, ns, torch.cuda.current_device()).t1 == t1
    x = np.random.default_rng(ns).standard_normal((nx, ns)).astype(np.float32)
    sel = [0, nx, 1]
    y = dw.dsp.fk_filter_filt(x, dw.dsp.fk_filter_design((nx, ns), sel, DX, FS))
    ref = O.fk_filter_filt(x.astype(np.float64), O.fk_filter_design((nx, ns), sel, DX, FS))
    e = rel_err(y, ref)
    assert e[0] <= TOL and e[1] <= TOL, e


@pytest.mark.parametrize("nx,scheme", [(48, 0), (200, 2)])
def test_config2_length_hybrid_tapered_vs_oracle(dw, nx, scheme):
    """ns = 120 000 (T1 = 12) with the tapered hybrid_ninf mask; at 200 channels the column transform is two-level,
    25 x 8 with the shared-memory level B."""
    import torch
    from das4whales_b200 import fk
    ns = 120000
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    assert (plan.t1, plan.col_scheme) == (12, scheme)
    x = np.random.default_rng(nx).standard_normal((nx, ns)).astype(np.float32)
    sel, args = [0, nx, 1], (1350., 1450., 3300, 3450, 14., 30.)
    y = dw.dsp.fk_filter_filt(x.copy(), dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *args), tapering=True)
    ref = O.fk_filter_filt(x.astype(np.float64), O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *args), tapering=True)
    e = rel_err(y, ref)
    assert e[0] <= TOL and e[1] <= TOL, e
    y = dw.dsp.fk_filter_filt(x, dw.dsp.fk_filter_design((nx, ns), sel, DX, FS))
    e = rel_err(y, O.fk_filter_filt(x.astype(np.float64), O.fk_filter_design((nx, ns), sel, DX, FS)))
    assert e[0] <= TOL and e[1] <= TOL, e


def test_edge_cases(dw):
    # odd time length breaks the reference's hybrid design the same way (dsp.py:349 broadcast)
    with pytest.raises(ValueError):
        dw.dsp.hybrid_ninf_filter_design((10, 11), [0, 10, 1], DX, FS)
    # FFT length with a large prime factor: explicit error, no silent fallback
    m = dw.dsp.fk_filter_design((8, 2 * 401), [0, 8, 1], DX, FS)
    with pytest.raises(ValueError):
        dw.dsp.fk_filter_filt(np.zeros((8, 802)), m)
    # shape mismatch raises like NumPy broadcasting does
    m = dw.dsp.fk_filter_design((10, 10), [0, 10, 1], DX, FS)
    with pytest.raises(ValueError):
        dw.dsp.fk_filter_filt(np.zeros((12, 10)), m)
    # all-zero mask -> all-zero output; tiny shapes from the reference's own tests (10 x 10)
    y = dw.dsp.fk_filter_filt(np.ones((10, 10)), np.zeros((10, 10)))
    assert y.shape == (10, 10) and np.all(y == 0)
    # identity mask -> identity
    x = np.random.default_rng(1).standard_normal((10, 10))
    y = dw.dsp.fk_filter_filt(x, np.ones((10, 10)))
    assert rel_err(y, x)[0] <= TOL


def test_tensor_in_tensor_out(dw):
    import torch
    nx, ns = 128, 2000
    x = torch.randn(nx, ns, device="cuda", dtype=torch.float32)
    mask = dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS)
    y = dw.dsp.fk_filter_filt(x, mask)
    assert isinstance(y, torch.Tensor) and y.is_cuda and y.dtype == torch.float32
    ref = O.fk_filter_filt(x.cpu().numpy().astype(np.float64), O.fk_filter_design((nx, ns), [0, nx, 1], DX, FS))
    assert rel_err(y.cpu().numpy(), ref)[0] <= TOL


def test_full_size_properties(dw):
    """BASELINE config 2 (10 000 x 120 000 fp32): the float64 oracle does not fit in host RAM, so
    check size-independent properties: plane waves are eigenfunctions with eigenvalue
    M_sym[k0, f0]; linearity; circular shift covariance."""
    import torch
    from das4whales_b200 import synth
    from das4whales_b200.fk import FkFilter
    nx, ns = 10000, 120000
    free = torch.cuda.mem_get_info()[0]
    if free < 40 << 30:
        pytest.skip("needs ~40 GB of device memory")
    mask = dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS, 1400, 1450, 3400, 3500)
    flt = FkFilter(mask)
    assert 0 < flt.rows_kept < nx // 2 + 1
    kval, fval = 1.0 / (nx * DX), FS / ns

    def mval(k0, f0):
        k, f = k0 * kval, f0 * fval
        if abs(k) < 0.005:
            return 0.0
        v = abs(f / k)
        m = 1.0
        if 1400 <= v <= 1450:
            m = np.sin(0.5 * np.pi * (v - 1400) / 50)
        if 3400 <= v <= 3500:
            m = 1 - np.sin(0.5 * np.pi * (v - 3400) / 100)
        if v >= 3500 or v < 1400:
            m = 0.0
        return m

    # pass band, both transition ramps, stop band (k0, f0 in DFT bins)
    for k0, f0 in ((400, 24000), (400, 16748), (400, 40549), (2000, 12000), (50, 3000)):
        x = synth.plane_wave(nx, ns, k0, f0)
        y = flt(x)
        want = mval(k0, f0)
        err = float((y - want * x).abs().max())
        assert err <= 1e-4, (k0, f0, want, err)
        del x, y
    a = synth.synth_strain(nx, ns, seed=1)
    b = synth.synth_strain(nx, ns, seed=2, amp=0.0)
    ya, yb = flt(a), flt(b)
    scale = float(ya.abs().max())
    a.mul_(0.5).add_(b, alpha=-2.0)                # a <- 0.5 a - 2 b
    yc = flt(a)
    lin = float((yc - (0.5 * ya - 2.0 * yb)).abs().max()) / scale
    assert lin <= 2e-5, lin
    del ya, yc, a
    sh = torch.roll(b, shifts=(37, 1001), dims=(0, 1))
    ysh = flt(sh)
    cov = float((ysh - torch.roll(yb, shifts=(37, 1001), dims=(0, 1))).abs().max()) / scale
    assert cov <= 2e-5, cov


def test_dense_design_masks_and_legacy_fk_filt(dw, golden):
    """hybrid / gs designs go through the dense-mask GPU path; legacy dsp.fk_filt reuses it."""
    g = golden("masks")
    rng = np.random.default_rng(2)
    x = rng.standard_normal((40, 240)).astype(np.float32)
    sel = [0, 40, 1]
    for mask in (dw.dsp.hybrid_filter_design((40, 240), sel, DX, FS), dw.dsp.hybrid_gs_filter_design((40, 240), sel, DX, FS),
                 dw.dsp.hybrid_ninf_gs_filter_design((40, 240), sel, DX, FS)):
        y = dw.dsp.fk_filter_sparsefilt(x, mask)
        ref = O.fk_filter_filt(x.astype(np.float64), mask.todense())
        assert rel_err(y, ref)[0] <= TOL
    y = dw.dsp.fk_filt(g["legacy_x"], 1, FS, 1, DX, 1450., 3400.)
    assert rel_err(y, g["legacy_y"])[0] <= TOL


# channel counts with no factor 16, 20 or 25 whose dual column fits one tile: 3^8, 3 x 7^4, 3^6 x 11, 3^3 x 7^3, 5 x 7^4
@pytest.mark.parametrize("nx,ns", [(6561, 1200), (7203, 1200), (8019, 1200), (9261, 1200), (12005, 1200)])
def test_tma_column_kernels_many_tiles_repeatable(dw, nx, ns):
    """Persistent TMA column kernels (one dual column per tile, several tiles per CTA): result must
    match the oracle and be bit-identical between runs (guards the generic/async proxy ordering)."""
    import torch
    from das4whales_b200 import fk
    assert fk.get_plan(nx, ns, torch.cuda.current_device()).col_scheme == 1
    rng = np.random.default_rng(nx)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    sel = [0, nx, 1]
    mask = dw.dsp.fk_filter_design((nx, ns), sel, DX, FS)
    xd = torch.from_numpy(x).cuda()
    y1 = dw.dsp.fk_filter_filt(xd, mask).cpu().numpy()
    y2 = dw.dsp.fk_filter_filt(xd, mask).cpu().numpy()
    assert np.array_equal(y1, y2)
    ref = O.fk_filter_filt(x.astype(np.float64), O.fk_filter_design((nx, ns), sel, DX, FS))
    assert rel_err(y1, ref)[0] <= TOL


COLUMN_SCHEMES = [{"D4W_COL_TWO_LEVEL": "0"},                                   # single-level persistent TMA kernels
                  {"D4W_COL_TWO_LEVEL": "0", "D4W_COL_TMA": "0"},               # single-level cp.async dual kernels
                  {"D4W_COL_PIPE": "0"},                                        # two-level, separate A / B launches
                  {"D4W_COL_PIPE": "0", "D4W_COL_CHUNK_PAIRS": "64"},           # ... in time chunks
                  {"D4W_COL_PIPE": "0", "D4W_COLB_FUSED": "0"},                 # shared-memory engine level B
                  {"D4W_COLB_RA": "16"},                                        # pipelined, 16 x 25 level B
                  {"D4W_PIPE_CQ": "40", "D4W_PIPE_LAG": "3"},                   # pipelined, narrower chunks / deeper ring
                  {"D4W_PIPE_HINTS": "0"},
                  {"D4W_ROW_FUSED": "1"}]                                       # opt-in fused middle row pass (P3)


@pytest.mark.parametrize("env", COLUMN_SCHEMES)
def test_column_schemes_agree(dw, monkeypatch, env):
    """Every column-transform scheme (the default is the pipelined two-level one) gives the oracle's answer, is
    repeatable bit for bit, and the ragged last chunk (ns/2 = 1100 pairs, chunks of 160) is handled."""
    import torch
    from das4whales_b200 import fk
    nx, ns = 10000, 2200
    rng = np.random.default_rng(5)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    sel = [0, nx, 1]
    ref = O.fk_filter_filt(x.astype(np.float64), O.fk_filter_design((nx, ns), sel, DX, FS), tapering=True)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    fk.free_plans()
    try:
        mask = dw.dsp.fk_filter_design((nx, ns), sel, DX, FS)
        xd = torch.from_numpy(x).cuda()
        y1 = dw.dsp.fk_filter_filt(xd.clone(), mask, tapering=True).cpu().numpy()
        y2 = dw.dsp.fk_filter_filt(xd.clone(), mask, tapering=True).cpu().numpy()
    finally:
        fk.free_plans()
    assert np.array_equal(y1, y2)
    assert rel_err(y1, ref)[0] <= TOL
