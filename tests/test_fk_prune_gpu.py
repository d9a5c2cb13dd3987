"""GPU: the f-k filter's opt-in support pruning (`eps`) against the exact pruning rule restated in float64 NumPy
(oracle/dsp_oracle.fk_filter_filt_pruned): wavenumber row k of the folded mask M_sym is kept iff
max_f float32(|M_sym[k, f]|) > float32(eps).  The number of kept rows must be the oracle's exactly, the output must match
the pruned float64 filter, and the output must stay within eps ||x||_2 of the exact (unpruned) filter."""
import numpy as np
import pytest

from conftest import rel_err
from oracle import dsp_oracle as O

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
TOL = 2e-5
HYB = (1350., 1450., 3300, 3450, 14., 30.)


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _scattered_mask(rng, nx, ns):
    """Signed, non-symmetric dense mask whose rows span nine decades (10**U(-9, 0)) and a fifth of them empty, so that
    eps leaves holes anywhere in the kept-row set; float32-representable, as the device keeps dense masks in float32."""
    m = rng.standard_normal((nx, ns)) * 10.0 ** rng.uniform(-9, 0, (nx, 1))
    m[rng.random(nx) < 0.2] = 0.0
    return m.astype(np.float32).astype(np.float64)


def _check(flt_rows, y, x, m, eps):
    ref, kept = O.fk_filter_filt_pruned(x, m, eps)
    assert flt_rows == kept, (flt_rows, kept)
    e = rel_err(y, ref)
    assert e[0] <= TOL and e[1] <= TOL, e
    exact = O.fk_filter_filt(x, m)
    assert np.linalg.norm(y - exact) <= eps * np.linalg.norm(x) + 1e-6 * np.linalg.norm(exact)
    return kept


# each shape picks a different column scheme by default (fk._Plan.col_scheme: 0 single-level cp.async, 1 single-level
# TMA, 2 two-level, 3 pipelined two-level)
PRUNE_SHAPES = [(63, 406, 0),       # ns % 4 != 0
                (551, 1200, 0),     # dual cp.async kernels, 8 columns per tile
                (6561, 1200, 1),    # 2 columns per tile, no 16/20/25 factor for a two-level split
                (1000, 2400, 2),    # 25 x 40, shared-memory level B
                (10000, 2200, 3)]   # 25 x 400, fused 20 x 20 level B


@pytest.mark.parametrize("nx,ns,scheme", PRUNE_SHAPES)
def test_dense_scattered_support_pruned(dw, nx, ns, scheme):
    import torch
    from das4whales_b200 import fk
    assert fk.get_plan(nx, ns, torch.cuda.current_device()).col_scheme == scheme
    rng = np.random.default_rng(nx + ns)
    m = _scattered_mask(rng, nx, ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32).astype(np.float64)
    rowmax = O.fold_rowmax(m)
    xd = torch.from_numpy(x.astype(np.float32)).cuda()
    for eps in (1e-7, 1e-4):
        flt = fk.FkFilter(m, eps=eps)
        kept = _check(flt.rows_kept, flt(xd).cpu().numpy().astype(np.float64), x, m, eps)
        keep = np.nonzero(rowmax > np.float32(eps))[0]
        assert 0 < kept < np.count_nonzero(rowmax) and keep[-1] + 1 > kept       # holes inside the kept set


COLUMN_SCHEMES = [{"D4W_COL_TWO_LEVEL": "0"},
                  {"D4W_COL_TWO_LEVEL": "0", "D4W_COL_TMA": "0"},
                  {"D4W_COL_PIPE": "0"},
                  {"D4W_COL_PIPE": "0", "D4W_COL_CHUNK_PAIRS": "64"},
                  {"D4W_COL_PIPE": "0", "D4W_COLB_FUSED": "0"},
                  {"D4W_COLB_RA": "16"},
                  {"D4W_PIPE_CQ": "40", "D4W_PIPE_LAG": "3"},
                  {"D4W_PIPE_HINTS": "0"},
                  {"D4W_ROW_FUSED": "1"}]


@pytest.mark.parametrize("env", COLUMN_SCHEMES)
def test_dense_scattered_support_pruned_column_schemes(dw, monkeypatch, env):
    """The same scattered support at 10 000 x 2 200 through every column-transform scheme (the per-plane entry and
    need tables of the two-level kernels, the chunk ring of the pipelined one)."""
    import torch
    from das4whales_b200 import fk
    nx, ns, eps = 10000, 2200, 1e-5
    rng = np.random.default_rng(3)
    m = _scattered_mask(rng, nx, ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32).astype(np.float64)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    fk.free_plans()
    try:
        flt = fk.FkFilter(m, eps=eps)
        rows, y = flt.rows_kept, flt(torch.from_numpy(x.astype(np.float32)).cuda()).cpu().numpy().astype(np.float64)
        del flt
    finally:
        fk.free_plans()
    _check(rows, y, x, m, eps)


def test_eps_boundary_is_exact(dw):
    """eps equal to a row's maximum drops the row; the next float32 below it keeps the row.  Dense masks are folded in
    double from their float32 values on the device exactly as the oracle folds them, so the boundary is bit-exact."""
    import torch
    from das4whales_b200 import fk
    nx, ns = 551, 1200
    rng = np.random.default_rng(17)
    m = _scattered_mask(rng, nx, ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32).astype(np.float64)
    xd = torch.from_numpy(x.astype(np.float32)).cuda()
    rowmax = O.fold_rowmax(m)
    order = np.argsort(rowmax)
    for k in (int(order[-(nx // 6)]), int(order[-3])):
        kept = []
        for eps in (float(rowmax[k]), float(np.nextafter(rowmax[k], np.float32(0)))):
            flt = fk.FkFilter(m, eps=eps)
            kept.append(_check(flt.rows_kept, flt(xd).cpu().numpy().astype(np.float64), x, m, eps))
        assert kept[1] - kept[0] == np.count_nonzero(rowmax == rowmax[k]) >= 1


def test_every_way_eps_arrives(dw):
    """FkFilter(ndarray, eps=...), FkMask.from_dense with prune_eps, a CUDA tensor mask, and an analytic hybrid_ninf
    FkMask at eps = 1e-7, 1e-5, 1e-3.  The device evaluates analytic masks in another order than the oracle, so for them
    eps is moved halfway between the two distinct row maxima around it: no row maximum lies within rounding of eps."""
    import torch
    from das4whales_b200 import fk
    nx, ns = 1000, 2400
    rng = np.random.default_rng(23)
    m = _scattered_mask(rng, nx, ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32).astype(np.float64)
    xd = torch.from_numpy(x.astype(np.float32)).cuda()
    eps = 1e-5
    flt = fk.FkFilter(m, eps=eps)
    _check(flt.rows_kept, flt(xd).cpu().numpy().astype(np.float64), x, m, eps)
    fm = fk.FkMask.from_dense(m)
    fm.prune_eps = eps
    y = dw.dsp.fk_filter_filt(x.astype(np.float32), fm)
    _check(fk.FkFilter(fm).rows_kept, y, x, m, eps)
    flt = fk.FkFilter(torch.from_numpy(m.astype(np.float32)).cuda(), eps=eps)
    _check(flt.rows_kept, flt(xd).cpu().numpy().astype(np.float64), x, m, eps)

    sel = [0, nx, 1]
    mh = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB)
    vals = np.unique(O.fold_rowmax(mh))
    for nominal in (1e-7, 1e-5, 1e-3):
        i = int(np.searchsorted(vals, nominal))
        lo, hi = (float(vals[i - 1]) if i else 0.0), float(vals[i])
        assert hi - lo > 1e-4 * hi, (nominal, lo, hi)
        eps = 0.5 * (lo + hi)
        flt = fk.FkFilter(dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB), eps=eps)
        _check(flt.rows_kept, flt(xd).cpu().numpy().astype(np.float64), x, mh, eps)


def test_eps_keyed_device_mask_cache(dw):
    """A pruned table built for eps must not be handed to a later exact filter on the same mask object."""
    import torch
    from das4whales_b200 import fk
    nx, ns = 1000, 2400
    sel = [0, nx, 1]
    x = np.random.default_rng(29).standard_normal((nx, ns)).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    mask = dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB)
    mh = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB)
    pruned = fk.FkFilter(mask, eps=1e-3)         # 1e-3 lies 4 % above the nearest row maximum at this shape
    y_eps = pruned(xd).cpu().numpy()
    exact = fk.FkFilter(mask)
    y = exact(xd).cpu().numpy()
    _check(pruned.rows_kept, y_eps.astype(np.float64), x.astype(np.float64), mh, 1e-3)
    assert pruned.rows_kept < exact.rows_kept == np.count_nonzero(O.fold_rowmax(mh) > 0)
    e = rel_err(y, O.fk_filter_filt(x.astype(np.float64), mh))
    assert e[0] <= TOL and e[1] <= TOL, e
    assert fk.FkFilter(mask, eps=1e-3).rows_kept == pruned.rows_kept
