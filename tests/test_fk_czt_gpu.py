"""GPU: the f-k filter at channel counts with a prime factor above 61, which the planner sends through the chirp-z column
transform (plan_info[7] == 4), against the float64 NumPy filter.  Script-style channel selections produce such counts
most of the time (4897 = 59 x 83, 3061 prime, 6122 = 2 x 3061, 7346 = 2 x 3673)."""
import os

import numpy as np
import pytest

from conftest import rel_err
from oracle import dsp_oracle as O

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
HYB = (1350., 1450., 3300, 3450, 14., 30.)
MAX_NORM, L2 = 1e-4, 1e-5
CZT_MAX_NX = 12800
WORKERS = os.cpu_count() or 1


def _largest_prime(n):
    p, big = 2, 1
    while p * p <= n:
        while n % p == 0:
            big, n = p, n // p
        p += 1
    return max(big, n)


def _awkward(n):
    return _largest_prime(n) > 61


LARGEST_AWKWARD = max(n for n in range(CZT_MAX_NX - 500, CZT_MAX_NX + 1) if _awkward(n))
NEXT_AWKWARD = min(n for n in range(CZT_MAX_NX + 1, CZT_MAX_NX + 500) if _awkward(n))


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _scheme(nx, ns):
    import torch
    from das4whales_b200 import fk
    return fk.get_plan(nx, ns, torch.cuda.current_device()).col_scheme


def _check(y, ref, what):
    e = rel_err(y, ref)
    print(f"czt parity {what}: max-norm {e[0]:.2e} l2 {e[1]:.2e}")
    assert e[0] <= MAX_NORM and e[1] <= L2, (what, e)
    return e


@pytest.mark.parametrize("ns", [1200, 12000])
@pytest.mark.parametrize("nx", [3061, 4897, 6122, 7346, LARGEST_AWKWARD])
def test_czt_masks_vs_float64(dw, nx, ns):
    """Fan, tapered hybrid_ninf and dense masks; ndarray in / out and CUDA tensor in / out; float64 NumPy reference."""
    import torch
    assert _awkward(nx) and _scheme(nx, ns) == 4
    rng = np.random.default_rng(nx + ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    x64 = x.astype(np.float64)
    xd = torch.from_numpy(x).cuda()
    step = 4                                   # script-style selection [start, stop, step] // dx
    sel = [0, nx * step, step]

    mref = O.fk_filter_design((nx, ns), sel, DX, FS)
    ref = O.fk_filter_filt(x64, mref, workers=WORKERS)
    _check(dw.dsp.fk_filter_filt(x.copy(), dw.dsp.fk_filter_design((nx, ns), sel, DX, FS)), ref, f"{nx}x{ns} fan ndarray")
    y = dw.dsp.fk_filter_filt(xd.clone(), dw.dsp.fk_filter_design((nx, ns), sel, DX, FS))
    assert isinstance(y, torch.Tensor) and y.is_cuda
    _check(y.cpu().numpy(), ref, f"{nx}x{ns} fan tensor")
    # dense: the same fan as a plain ndarray (host) and as a float32 CUDA tensor
    _check(dw.dsp.fk_filter_filt(x.copy(), np.asarray(mref)), ref, f"{nx}x{ns} dense ndarray")
    y = dw.dsp.fk_filter_filt(xd.clone(), torch.from_numpy(np.ascontiguousarray(mref)).cuda())
    _check(y.cpu().numpy(), ref, f"{nx}x{ns} dense tensor")
    del mref, ref

    mh = O.hybrid_ninf_filter_design((nx, ns), [0, nx, 1], DX, FS, *HYB)
    ref = O.fk_filter_filt(x64.copy(), mh, tapering=True, workers=WORKERS)
    del mh
    mask = dw.dsp.hybrid_ninf_filter_design((nx, ns), [0, nx, 1], DX, FS, *HYB)
    _check(dw.dsp.fk_filter_filt(x.copy(), mask, tapering=True), ref, f"{nx}x{ns} hybrid_ninf tapered ndarray")
    y = dw.dsp.fk_filter_sparsefilt(xd.clone(), mask, tapering=True)
    _check(y.cpu().numpy(), ref, f"{nx}x{ns} hybrid_ninf tapered tensor")


@pytest.mark.parametrize("nx,ns", [(4897, 1200), (6122, 1215)])
def test_czt_eps_pruning(dw, nx, ns):
    """Opt-in eps pruning on a chirp-z plan: kept-row count and output against the pruned float64 filter, and the l2
    bound ||y_eps - y||_2 <= eps ||x||_2 against the exact filter."""
    import torch
    from das4whales_b200 import fk
    rng = np.random.default_rng(nx)
    m = rng.standard_normal((nx, ns)) * 10.0 ** rng.uniform(-9, 0, (nx, 1))
    m[rng.random(nx) < 0.2] = 0.0
    m = m.astype(np.float32).astype(np.float64)
    x = rng.standard_normal((nx, ns)).astype(np.float32).astype(np.float64)
    xd = torch.from_numpy(x.astype(np.float32)).cuda()
    exact = O.fk_filter_filt(x, m)
    for eps in (1e-7, 1e-4):
        flt = fk.FkFilter(m, eps=eps)
        assert flt.plan.col_scheme == 4
        y = flt(xd).cpu().numpy().astype(np.float64)
        ref, kept = O.fk_filter_filt_pruned(x, m, eps)
        assert flt.rows_kept == kept < np.count_nonzero(O.fold_rowmax(m))
        _check(y, ref, f"{nx}x{ns} eps={eps}")
        assert np.linalg.norm(y - exact) <= eps * np.linalg.norm(x) + 1e-6 * np.linalg.norm(exact)


def test_czt_ooi_scale_hybrid_whole_matrix(dw):
    """7346 x 12 000 (an OOI-scale selection) with the tapered hybrid_ninf mask, every sample of y against float64."""
    import torch
    from oracle import torch_oracle as TO
    nx, ns = 7346, 12000
    assert _scheme(nx, ns) == 4
    gen = torch.Generator(device="cuda").manual_seed(7346)
    x = torch.randn((nx, ns), device="cuda", generator=gen)
    y = dw.dsp.fk_filter_filt(x.clone(), dw.dsp.hybrid_ninf_filter_design((nx, ns), [0, nx, 1], DX, FS, *HYB), tapering=True)
    cols = TO.hybrid_ninf_columns((nx, ns), [0, nx, 1], DX, FS, *HYB, device="cuda")
    e = TO.fk_filter_errors(x, y, cols, tapering=True)
    print(f"czt parity {nx}x{ns} hybrid_ninf tapered whole matrix (float64): max-norm {e.max_norm:.2e} l2 {e.l2:.2e}")
    assert e.max_norm <= MAX_NORM and e.l2 <= L2, e


def test_czt_plan_scheme_and_smooth_shapes_unchanged(dw):
    """Chirp-z plans report scheme 4; the channel counts the rest of the suite uses keep their mixed-radix schemes."""
    for nx in (3061, 4897, 6122, 7346, LARGEST_AWKWARD):
        assert _scheme(nx, 12000) == 4
    for nx in (11020, 5510, 8000, 10000):
        assert _scheme(nx, 12000) <= 3


def test_czt_capacity_boundary(dw):
    import torch
    from das4whales_b200 import fk
    dev = torch.cuda.current_device()
    assert fk.get_plan(LARGEST_AWKWARD, 1200, dev).col_scheme == 4
    with pytest.raises(ValueError, match="12800"):
        fk.get_plan(NEXT_AWKWARD, 1200, dev)
    with pytest.raises(ValueError):
        dw.dsp.fk_filter_filt(np.zeros((NEXT_AWKWARD, 1200), np.float32), dw.dsp.fk_filter_design((NEXT_AWKWARD, 1200), [0, NEXT_AWKWARD, 1], DX, FS))
    rng = np.random.default_rng(12)
    for nx in rng.integers(2, 28001, 24):
        nx2, ns2 = dw.dsp.supported_shape(int(nx), 1200)
        assert nx2 <= nx and (nx2 == nx or nx > CZT_MAX_NX)
        fk.get_plan(nx2, ns2, dev)
    fk.free_plans()


def test_czt_legacy_fk_filt(dw):
    """The legacy one-call dsp.fk_filt at an awkward channel count."""
    nx, ns = 4897, 1200
    x = np.random.default_rng(3).standard_normal((nx, ns))
    args = (1, FS, 1, DX, 1400., 3500.)
    _check(dw.dsp.fk_filt(x, *args), O.fk_filt(x, *args), f"{nx}x{ns} legacy fk_filt")


@pytest.mark.parametrize("world,nsub", [(2, 1), (2, 3)])
def test_czt_sharded_local_group(dw, world, nsub):
    """dist.ShardedFkFilter on time slabs of a chirp-z plan, ranks stepped in one process, against the single-GPU filter."""
    import torch
    from das4whales_b200 import dist as d4wdist
    from das4whales_b200.fk import FkFilter
    nx, ns = 6122, 9600
    gen = torch.Generator(device="cuda").manual_seed(nx)
    x = torch.randn((nx, ns), device="cuda", generator=gen)
    mask = dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS)
    ref = FkFilter(mask)(x, tapering=True)
    be = d4wdist.CudaBackend(mask, nx, ns, world, nsub=nsub)
    assert be.slab.col_scheme == 4
    filters = [d4wdist.ShardedFkFilter(nx, ns, be, rank=r, world=world) for r in range(world)]
    cpr = nx // world
    ys = d4wdist.run_local_group(filters, [x[r * cpr:(r + 1) * cpr].contiguous() for r in range(world)], tapering=True)
    e = rel_err(torch.cat(ys, dim=0).cpu().numpy(), ref.cpu().numpy())
    assert e[0] <= 5e-6 and e[1] <= 5e-6, e
