"""BASELINE-size parity (configs[1] and configs[2]: 10 000 channels x 120 000 samples) -- DIRECT comparison of the CUDA f-k
filter with the float64 answer for the whole matrix, computed on the same GPU by oracle/torch_oracle.fk_filter_errors:
the literal fft2 -> x ifftshift(M) -> ifft2 of the reference in float64, slab by slab, with the mask generated column slab
by column slab (pinned against the NumPy oracle on the CPU by test_oracle_golden.py).  The filter's plan and buffers are
released before the oracle runs, so by the shapes a comparison needs about 31 GB of device memory (36 GB with a dense
mask), and each test checks the free memory it needs first (the card may be shared).
Contract (SURVEY 8d): max-norm error <= 1e-4 and l2 error <= 1e-5 relative to the float64 result.

Config 3 adds the HF + LF fin-whale matched filter and the envelope on the filtered matrix; those are checked on 64 full
120 000-sample rows against the float64 NumPy/SciPy oracle (rows are independent in these operators)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
NX, NS = 10000, 120000
FAN = (1400.0, 1450.0, 3400.0, 3500.0)
HYB = (1350., 1450., 3300, 3450, 14., 30.)           # the masks the reference scripts use (main_mfdetect.py:46-47)
REAL = NX * NS * 4                                    # one float32 [NX, NS] matrix
ROWS_PER_SLAB, COLS_PER_SLAB = 256, 1024
# the oracle's complex128 spectrum, plus its largest slab temporaries (about four complex128 slabs)
ORACLE = NX * NS * 16 + 64 * max(ROWS_PER_SLAB * NS, COLS_PER_SLAB * NX)


def _require(torch, need, what):
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"{what} needs {need / 1e9:.1f} GB of free device memory; {free / 1e9:.1f} GB are free")


@pytest.fixture(scope="module")
def env():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _require(torch, 2 * REAL, f"the {NX} x {NS} float32 input")
    import das4whales_b200 as dw
    from das4whales_b200 import _lib, fk, synth
    _lib.lib()
    x = synth.synth_strain(NX, NS, seed=1234)
    yield dw, torch, x
    del x
    fk.free_plans()
    torch.cuda.empty_cache()


def _filter_vs_float64(torch, x, make_mask, mask_cols, tapering=False, eps=0.0, what=""):
    """Run FkFilter(make_mask(), eps) on x, release the filter, then compare its output with the streaming float64
    oracle.  Returns (errors, rows kept)."""
    from das4whales_b200 import fk
    from oracle import torch_oracle as TO
    flt = fk.FkFilter(make_mask(), eps=eps)
    rows = flt.rows_kept
    _require(torch, REAL + max(flt.dm.workspace_bytes, ORACLE), what)
    y = flt(x, tapering=tapering)
    torch.cuda.synchronize()
    del flt
    fk.free_plans()                     # the plan's workspace and the mask table are gone before the oracle starts
    torch.cuda.empty_cache()
    e = TO.fk_filter_errors(x, y, mask_cols, tapering=tapering, rows_per_slab=ROWS_PER_SLAB, cols_per_slab=COLS_PER_SLAB)
    del y
    torch.cuda.empty_cache()
    return e, rows


def test_config2_fan_mask_direct(env):
    dw, torch, x = env
    from oracle import torch_oracle as TO
    sel = [0, NX, 1]
    e, rows = _filter_vs_float64(torch, x, lambda: dw.dsp.fk_filter_design((NX, NS), sel, DX, FS, *FAN),
                                 TO.fan_columns((NX, NS), sel, DX, FS, *FAN, device=x.device), what="config 2 fan mask")
    print(f"config 2 fan mask ({rows} rows kept): max-norm {e.max_norm:.2e}, l2 {e.l2:.2e}")
    assert e.max_norm <= 1e-4 and e.l2 <= 1e-5, e


def test_config2_hybrid_ninf_mask_direct(env):
    dw, torch, x = env
    from oracle import torch_oracle as TO
    sel = [0, NX, 1]
    e, rows = _filter_vs_float64(torch, x, lambda: dw.dsp.hybrid_ninf_filter_design((NX, NS), sel, DX, FS, *HYB),
                                 TO.hybrid_ninf_columns((NX, NS), sel, DX, FS, *HYB, device=x.device), tapering=True,
                                 what="config 2 hybrid_ninf mask")
    print(f"config 2 hybrid_ninf mask (tapered, {rows} rows kept): max-norm {e.max_norm:.2e}, l2 {e.l2:.2e}")
    assert e.max_norm <= 1e-4 and e.l2 <= 1e-5, e


def test_config2_hybrid_ninf_eps_pruned_error_bound(env):
    """Opt-in support pruning by threshold (`eps`): rows of the folded mask that never exceed eps are dropped.  Against
    the exact float64 answer the error stays inside the 1e-4 max-norm contract for the documented eps = 1e-5, and the
    l2 error inside the pruning bound eps ||x||_2 (plus fp32 rounding, 1e-6 ||y||_2)."""
    dw, torch, x = env
    from oracle import torch_oracle as TO
    sel, eps = [0, NX, 1], 1e-5
    e, rows = _filter_vs_float64(torch, x, lambda: dw.dsp.hybrid_ninf_filter_design((NX, NS), sel, DX, FS, *HYB),
                                 TO.hybrid_ninf_columns((NX, NS), sel, DX, FS, *HYB, device=x.device), eps=eps,
                                 what="config 2 hybrid_ninf mask, eps = 1e-5")
    x_l2 = float(torch.linalg.vector_norm(x, dtype=torch.float64))
    bound = eps * x_l2 + 1e-6 * e.ref_l2
    print(f"config 2 hybrid_ninf eps=1e-5 ({rows} rows kept): max-norm {e.max_norm:.2e}, l2 {e.l2:.2e} "
          f"(bound eps*||x||/||y|| + 1e-6 = {bound / e.ref_l2:.2e})")
    assert rows < 0.3 * (NX // 2 + 1)
    assert e.max_norm <= 1e-4, e
    assert e.l2 * e.ref_l2 <= bound, (e, bound)


def test_config2_dense_mask_direct(env):
    """The fan mask handed over as a dense float32 CUDA tensor (d4w_fk_mask_create_dense's support scan and table
    build at full size), against the float64 filter with exactly those float32 mask values."""
    dw, torch, x = env
    from oracle import torch_oracle as TO
    sel = [0, NX, 1]
    _require(torch, REAL, "the dense float32 mask")
    dense = torch.empty((NX, NS), dtype=torch.float32, device=x.device)
    fan = TO.fan_columns((NX, NS), sel, DX, FS, *FAN, device=x.device)
    for c0 in range(0, NS, 4096):
        dense[:, c0:c0 + 4096] = fan(torch.arange(c0, min(NS, c0 + 4096), device=x.device)).to(torch.float32)
    e, rows = _filter_vs_float64(torch, x, lambda: dense, TO.dense_columns(dense), what="config 2 dense fan mask")
    del dense
    print(f"config 2 dense float32 fan mask ({rows} rows kept): max-norm {e.max_norm:.2e}, l2 {e.l2:.2e}")
    assert e.max_norm <= 1e-4 and e.l2 <= 1e-5, e


def test_config3_matched_filter_and_envelope_on_full_rows(env):
    dw, torch, x = env
    from oracle import detect_oracle as D
    from das4whales_b200.fk import FkFilter
    mask = dw.dsp.fk_filter_design((NX, NS), [0, NX, 1], DX, FS, *FAN)
    flt = FkFilter(mask)
    # y, two correlograms and one envelope, the filter's workspace, and room for the matched filter's chunks
    _require(torch, 4 * REAL + flt.dm.workspace_bytes + (2 << 30), "config 3")
    y = flt(x)
    del flt
    tgrid = np.arange(NS) / FS
    tpls = [dw.detect.gen_template_fincall(tgrid, FS, 17.8, 28.8, 0.68), dw.detect.gen_template_fincall(tgrid, FS, 14.7, 21.8, 0.78)]
    corr = dw.detect.compute_cross_correlograms(y, tpls)
    env_hf = dw.detect.envelope(corr[0])
    rows = np.random.default_rng(7).choice(NX, size=64, replace=False)
    rows.sort()
    ridx = torch.from_numpy(rows).to(y.device)
    yr = y[ridx].cpu().numpy().astype(np.float64)
    for t, c in zip(tpls, corr):
        ref = D.compute_cross_correlogram(yr, t)
        got = c[ridx].cpu().numpy().astype(np.float64)
        emax = np.max(np.abs(got - ref)) / np.max(np.abs(ref))
        el2 = np.linalg.norm(got - ref) / np.linalg.norm(ref)
        print(f"config 3 matched filter on 64 rows: max-norm {emax:.2e}, l2 {el2:.2e}")
        assert emax <= 1e-4 and el2 <= 1e-5, (emax, el2)
    # envelope of the GPU correlogram rows vs scipy.signal.hilbert on the same rows
    cr = corr[0][ridx].cpu().numpy().astype(np.float64)
    eref = D.envelope(cr)
    egot = env_hf[ridx].cpu().numpy().astype(np.float64)
    assert np.max(np.abs(egot - eref)) / np.max(eref) <= 1e-4
    # picks on those rows: indices equal to SciPy's on the same (GPU) envelope rows
    thr = 0.5 * float(eref.max())
    picks = dw.detect.pick_times_env(corr[0][ridx].contiguous(), thr)
    import scipy.signal as sps
    for i in range(len(rows)):
        ref_idx = sps.find_peaks(egot[i].astype(np.float32), prominence=thr)[0]
        assert np.array_equal(picks[i], ref_idx)
