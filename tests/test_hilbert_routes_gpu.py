"""GPU parity of the Hilbert family on every direct route the row planner can pick: whole rows in one CTA (k_hilbert_row),
including transforms built from generic prime stages (7..61, fft_smem.cuh stage_generic, whose device code no CPU test
runs), and split rows two per transform (k_hsplit_fwd2<T1> -> middle pass -> k_hsplit_inv2<T1>) for every split radix
of row_plan.hpp's with_t1, under either middle pass.  Envelope, H(x), envelope / std, envelope SNR and instant_freq
against float64 scipy.signal.hilbert.  The chirp-z routes are in test_hilbert_czt_gpu.py; test_hilbert_routes_host.py
checks on the CPU that these tables are what the planner picks and that they cover every radix."""
import numpy as np
import pytest
import scipy.signal as sps

from conftest import rel_err
from oracle import dsp_oracle as O
from test_hilbert_czt_gpu import FS, TOL, _chirp_rows
from test_rows_gpu import HILBERT_ROUTES

pytestmark = pytest.mark.gpu

# (n, T1, T2) as the planner splits n on an H100 (227 KB of shared memory per block).  Whole rows (T1 = 1) whose
# transform runs generic prime stages, then at least one split per radix; T2 factorisations in the comments.
DIRECT_ROUTES = [
    (12005, 1, 12005),      # 5 * 7^4
    (16337, 1, 16337),      # 17 * 31^2
    (12103, 1, 12103),      # 7^2 * 13 * 19
    (13000, 1, 13000),      # 2^3 * 5^3 * 13
    (18000, 2, 9000),
    (16492, 2, 8246),       # 2 * 7 * 19 * 31
    (17457, 3, 5819),       # 11 * 23^2
    (20608, 4, 5152),       # 2^5 * 7 * 23
    (16445, 5, 3289),       # 11 * 13 * 23
    (45000, 5, 9000),
    (31878, 6, 5313),       # 3 * 7 * 11 * 23
    (60000, 6, 10000),
    (41624, 8, 5203),       # 11^2 * 43
    (75000, 8, 9375),
    (53690, 10, 5369),      # 7 * 13 * 59
    (100000, 10, 10000),
    (62604, 12, 5217),      # 3 * 37 * 47
    (53235, 15, 3549),      # 3 * 7 * 13^2
    (84224, 16, 5264),      # 2^4 * 7 * 47
    (128000, 16, 8000),
    (102500, 20, 5125),     # 5^3 * 41
    (125000, 20, 6250),
    (55225, 25, 2209),      # 47^2
]
# 1, 2 or 3 rows in turn: an odd count leaves the last pair of a split route half empty
CASES = [(i % 3 + 1, n, t1, t2) for i, (n, t1, t2) in enumerate(DIRECT_ROUTES)]


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available()
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


@pytest.fixture
def fresh_plans(monkeypatch):
    """Plans read D4W_ROW_FUSED when they are created: start from an empty cache, free what was made."""
    from das4whales_b200 import _lib, rows
    monkeypatch.setattr(rows, "_row_plans", {})
    yield rows
    for p in rows._row_plans.values():
        _lib.lib().d4w_row_plan_destroy(p.ptr)


@pytest.mark.parametrize("env", HILBERT_ROUTES, ids=["fused", "row_mid"])
@pytest.mark.parametrize("nx,n,t1,t2", CASES)
def test_hilbert_family_direct_routes(dw, fresh_plans, monkeypatch, env, nx, n, t1, t2):
    import torch
    from das4whales_b200 import _lib
    rows = fresh_plans
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    plan = rows.row_plan(n, 0)
    assert plan.info() == (t1, t2, 0), (n, plan.info())
    x = _chirp_rows(nx, n, seed=n)
    x64 = x.astype(np.float64)
    a = sps.hilbert(x64, axis=1)
    e = rel_err(dw.detect.envelope(x), np.abs(a))[0]
    assert e <= 2e-5, (n, nx, e)
    xd = torch.from_numpy(x).cuda()
    e = rel_err(rows.hilbert_imag(xd).cpu().numpy(), a.imag)[0]
    assert e <= 2e-5, (n, nx, e)
    eos = rows.envelope_over_std(xd).cpu().numpy()
    assert rel_err(eos, np.abs(a) / x64.std(axis=1, keepdims=True))[0] <= 2e-5, (n, nx)
    snr = dw.dsp.snr_tr_array(x, env=True)
    ref = O.snr_tr_array(x64, env=True)
    assert rel_err(10 ** (snr / 10), 10 ** (ref / 10))[0] <= TOL, (n, nx)
    fi = dw.dsp.instant_freq(x[0], FS)
    fref = O.instant_freq(x64[0], FS)
    assert fi.shape == fref.shape == (n - 1,)
    assert np.max(np.abs(fi - fref)) <= 2e-4 * FS, n
    assert np.max(np.abs(fi[50:-50] - fref[50:-50])) <= 2e-5 * FS, n
    ws = _lib.lib().d4w_row_workspace_bytes(plan.ptr, nx)
    assert ws == (16 if t1 == 1 else (nx + 1) // 2 * n * 8), (n, ws)
