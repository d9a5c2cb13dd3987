"""GPU tests of the f-k mask bank (d4w_fk_bank_*, fk.FkFilterBank, dsp.fk_filter_filts) and of
pipeline.FkCompPipeline.

Every output of a bank is pinned with torch.equal to the single-mask filter FkFilter(mask_i) on the same input: the
arithmetic on every kept row is the same, and rows outside a mask's support are exact zeros in both paths (at most the
sign of a zero differs, which torch.equal ignores).  The shapes cover every column scheme the planner reaches by default.
The pipeline is pinned element for element to the chain of today's calls and, at a small shape, to
scripts/main_fkcomp.py:56-122 restated on the float64 oracles."""
import numpy as np
import pytest

from conftest import rel_err
from oracle import dsp_oracle as O

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
SPEEDS = (1350., 1450., 3300., 3450.)          # scripts/main_fkcomp.py:59-62
TOL = 1e-4


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _rows_mask(rng, nx, ns, rows):
    """Signed dense mask that is zero outside the shifted rows `rows` (float32-representable)."""
    m = rng.standard_normal((nx, ns))
    keep = np.zeros(nx, dtype=bool)
    keep[rows] = True
    m[~keep] = 0.0
    return m.astype(np.float32).astype(np.float64)


def _legacy_fk_filt_mask(shape, sel):
    return O.fk_filt_mask(shape, 1, FS, sel[2], DX, 1350., 3450.)


def _masks(dw, rng, nx, ns, kinds):
    sel = [0, nx, 1]
    c = dict(cs_min=SPEEDS[0], cp_min=SPEEDS[1], cp_max=SPEEDS[2], cs_max=SPEEDS[3], fmin=14., fmax=30.)
    inf = dict(cs_min=SPEEDS[0], cp_min=SPEEDS[1], fmin=14., fmax=30.)
    make = {
        "fan": lambda: dw.dsp.fk_filter_design((nx, ns), sel, DX, FS, *SPEEDS),
        "hybrid_ninf": lambda: dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, **c),
        "hybrid": lambda: dw.dsp.hybrid_filter_design((nx, ns), sel, DX, FS, **inf),
        "hybrid_gs": lambda: dw.dsp.hybrid_gs_filter_design((nx, ns), sel, DX, FS, **inf),
        "hybrid_ninf_gs": lambda: dw.dsp.hybrid_ninf_gs_filter_design((nx, ns), sel, DX, FS, **c),
        "fk_filt": lambda: _legacy_fk_filt_mask((nx, ns), sel),
        "random_rows": lambda: _rows_mask(rng, nx, ns, rng.random(nx) < 0.3),
        "low_rows": lambda: _rows_mask(rng, nx, ns, np.arange(nx // 2 - 3, nx // 2 + 4)),   # |k| <= 3
    }
    out = []
    for k in kinds:
        if k.endswith("@pruned"):                     # eps-pruned hybrid_ninf: its Butterworth tails are dropped
            m = make[k.split("@")[0]]()
            m.prune_eps = 1e-5
            out.append(m)
        else:
            out.append(make[k]())
    return out


# (nx, ns, default column scheme, masks): 0 single-level cp.async, 1 single-level TMA, 2 two-level, 3 pipelined
# two-level, 4 chirp-z
BANK_CASES = [
    (63, 406, 0, ["fan", "random_rows", "low_rows", "fk_filt"]),
    (551, 1200, 0, ["fan", "hybrid_ninf", "hybrid", "hybrid_gs", "hybrid_ninf_gs", "fk_filt", "random_rows"]),
    (6561, 1200, 1, ["hybrid_ninf@pruned", "hybrid_ninf", "fan", "random_rows"]),
    (1000, 2400, 2, ["fan", "hybrid_ninf", "hybrid_ninf@pruned", "low_rows", "random_rows"]),
    (10000, 2200, 3, ["hybrid_ninf@pruned", "fan", "hybrid", "random_rows"]),
    (4897, 1200, 4, ["fan", "hybrid_ninf@pruned", "hybrid", "low_rows"]),
    (11020, 12000, 2, ["hybrid_ninf", "hybrid_ninf@pruned", "fan", "hybrid"]),
]


@pytest.mark.parametrize("nx,ns,scheme,kinds", BANK_CASES)
def test_bank_outputs_equal_single_mask_filters(dw, nx, ns, scheme, kinds):
    import torch
    from das4whales_b200 import fk
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    assert plan.col_scheme == scheme
    info = dw._lib.ffi.new("int[8]")
    dw._lib.check(dw._lib.lib().d4w_fk_plan_info(plan.ptr, info), "plan info")
    assert info[7] == scheme
    rng = np.random.default_rng(nx * 7 + ns)
    masks = _masks(dw, rng, nx, ns, kinds)
    x = torch.from_numpy(rng.standard_normal((nx, ns)).astype(np.float32)).cuda()
    bank = fk.FkFilterBank(masks)
    singles = [fk.FkFilter(m) for m in masks]
    rows = [f.rows_kept for f in singles]
    assert bank.rows_kept >= max(rows)
    if "@pruned" in "".join(kinds) or "low_rows" in kinds:
        assert any(r < bank.rows_kept for r in rows), "the union must be larger than some mask's support"
    for tapering in (False, True):
        ys = bank(x, tapering=tapering)
        for k, y, f in zip(kinds, ys, singles):
            assert torch.equal(y, f(x, tapering=tapering)), (nx, ns, k, tapering)
    del ys, bank, singles
    torch.cuda.empty_cache()


def test_one_mask_bank_equals_apply(dw):
    import torch
    from das4whales_b200 import fk
    nx, ns = 1000, 2400
    rng = np.random.default_rng(3)
    m = _masks(dw, rng, nx, ns, ["hybrid_ninf"])[0]
    x = torch.from_numpy(rng.standard_normal((nx, ns)).astype(np.float32)).cuda()
    bank = fk.FkFilterBank([m])
    assert bank.rows_kept == fk.FkFilter(m).rows_kept
    for tapering in (False, True):
        assert torch.equal(bank(x, tapering=tapering)[0], fk.FkFilter(m)(x, tapering=tapering))


def test_disjoint_supports(dw):
    """Two masks on disjoint wavenumber rows: each output keeps only its own rows, and the other mask's rows of U are
    exact zeros in its table."""
    import torch
    from das4whales_b200 import fk
    nx, ns = 551, 1200
    rng = np.random.default_rng(5)
    a = _rows_mask(rng, nx, ns, np.arange(nx // 2 - 10, nx // 2 + 11))        # |k| <= 10
    far = (np.abs(np.arange(nx) - nx // 2) > 40) & (np.abs(np.arange(nx) - nx // 2) < 90)
    b = _rows_mask(rng, nx, ns, far)                                           # 40 < |k| < 90
    x = torch.from_numpy(rng.standard_normal((nx, ns)).astype(np.float32)).cuda()
    bank = fk.FkFilterBank([a, b])
    fa, fb = fk.FkFilter(a), fk.FkFilter(b)
    assert bank.rows_kept == fa.rows_kept + fb.rows_kept
    ya, yb = bank(x)
    assert torch.equal(ya, fa(x)) and torch.equal(yb, fb(x))
    x64 = x.cpu().numpy().astype(np.float64)
    for y, m in ((ya, a), (yb, b)):
        e = rel_err(y.cpu().numpy(), O.fk_filter_filt(x64, m))
        assert e[0] <= TOL and e[1] <= 1e-5, e


def test_errors_and_aliasing(dw):
    import torch
    from das4whales_b200 import fk, _lib
    L, ffi = _lib.lib(), _lib.ffi
    nx, ns = 63, 406
    rng = np.random.default_rng(8)
    m1, m2 = _masks(dw, rng, nx, ns, ["fan", "random_rows"])
    x = torch.from_numpy(rng.standard_normal((nx, ns)).astype(np.float32)).cuda()
    with pytest.raises(ValueError):
        fk.FkFilterBank([])
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    out = ffi.new("d4w_fk_bank**")
    assert L.d4w_fk_bank_create(out, plan.ptr, ffi.new("d4w_fk_mask*[]", 1), 0) == 1            # nmasks < 1
    other = fk.get_plan(64, ns, torch.cuda.current_device())
    dm_other = fk.device_mask_for(_rows_mask(rng, 64, ns, np.arange(30, 34)), other)
    dm1 = fk.device_mask_for(m1, plan)
    assert L.d4w_fk_bank_create(out, plan.ptr, ffi.new("d4w_fk_mask*[]", [dm1.ptr, dm_other.ptr]), 2) == 1
    assert "another plan" in ffi.string(L.d4w_last_error()).decode()
    with pytest.raises(ValueError):
        fk.FkFilterBank([m1, np.zeros((64, ns))], shape=(nx, ns))                               # mask of another shape
    # a bank used before d4w_fk_bank_build
    assert L.d4w_fk_bank_create(out, plan.ptr, ffi.new("d4w_fk_mask*[]", [dm1.ptr]), 1) == 0
    raw = out[0]
    try:
        ws = torch.empty(int(L.d4w_fk_bank_workspace_bytes(plan.ptr, raw)), dtype=torch.uint8, device="cuda")
        y = torch.empty_like(x)
        rc = L.d4w_fk_bank_apply(plan.ptr, raw, _lib.ptr(x, "float*"), ffi.new("float*[]", [_lib.ptr(y, "float*")]),
                                 _lib.ptr(ws), 0, _lib.stream_ptr())
        assert rc == 1 and "d4w_fk_bank_build" in ffi.string(L.d4w_last_error()).decode()
    finally:
        L.d4w_fk_bank_destroy(raw)
    bank = fk.FkFilterBank([m1, m2])
    y = torch.empty_like(x)
    with pytest.raises(ValueError, match="overlap"):
        bank(x, outs=[y, y])
    flat = torch.empty(2 * nx * ns + 7, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError, match="overlap"):                                            # partial overlap
        bank(x, outs=[flat[:nx * ns].view(nx, ns), flat[7:7 + nx * ns].view(nx, ns)])
    ref = [fk.FkFilter(m1)(x), fk.FkFilter(m2)(x)]
    for i in range(2):                                  # one output may alias x, which is last read in P1
        xa = x.clone()
        outs = [torch.empty_like(x), torch.empty_like(x)]
        outs[i] = xa
        ys = bank(xa, outs=outs)
        assert ys[i] is xa
        assert torch.equal(ys[0], ref[0]) and torch.equal(ys[1], ref[1])


def test_fk_filter_filts_parity(dw):
    import torch
    nx, ns = 551, 1200
    rng = np.random.default_rng(11)
    kinds = ["fan", "hybrid_ninf", "hybrid_gs", "random_rows"]
    masks = _masks(dw, rng, nx, ns, kinds)
    x = rng.standard_normal((nx, ns))
    for tapering in (False, True):
        xh = x.copy()
        ys = dw.dsp.fk_filter_filts(xh, masks, tapering=tapering)
        assert len(ys) == len(masks) and all(y.dtype == np.float64 for y in ys)
        for k, y, m in zip(kinds, ys, masks):
            e = rel_err(y, O.fk_filter_filt(x.copy(), np.asarray(m), tapering=tapering))
            assert e[0] <= TOL and e[1] <= 1e-5, (k, tapering, e)
            assert np.array_equal(y, dw.dsp.fk_filter_filt(x.copy(), m, tapering=tapering)), k
        once = x.copy()                                  # the caller's array is tapered once, as fk_filter_filt does
        dw.dsp.fk_filter_filt(once, masks[0], tapering=tapering)
        assert np.array_equal(xh, once)
        assert np.array_equal(xh, x) != tapering
    xd = torch.from_numpy(x.astype(np.float32)).cuda()
    yd = dw.dsp.fk_filter_filts(xd, masks)
    for k, y, m in zip(kinds, yd, masks):
        assert y.dtype == torch.float32 and y.is_cuda
        assert torch.equal(y, dw.dsp.fk_filter_filt(xd, m)), k
        e = rel_err(y.cpu().numpy(), O.fk_filter_filt(xd.cpu().numpy().astype(np.float64), np.asarray(m)))
        assert e[0] <= TOL and e[1] <= 1e-5, (k, e)


def _counts(nx, ns, seed):
    from oracle.make_golden import synth
    x = synth(nx, ns, seed=seed, ncalls=3)
    return np.round(x * 5.0e4).astype(np.int32) + 1234


SCALE = 4.0838e-11 * 1550.0 / 2.0419
NAMES = ("nf_cos", "nf_gs", "inf_cos", "inf_gs")


def test_fkcomp_pipeline_equals_todays_calls(dw):
    """process_device = raw2strain, bp_filt, four fk_filter_sparsefilt and four snr_tr_array(env=True), element for
    element; argmax = np.argmax of the same float32 inf_cos output."""
    import torch
    from das4whales_b200 import pipeline, rows
    nx, ns, sel = 400, 6000, [0, 400, 1]
    counts = _counts(nx, ns, 21)
    pipe = pipeline.FkCompPipeline(nx, ns, sel, DX, FS, SCALE)
    assert not hasattr(pipe, "fk")                       # no unused hybrid_ninf FkFilter
    raw = torch.from_numpy(counts).cuda()
    dev = pipe.process_device(raw, with_traces=True)
    x = dw.dsp.bp_filt(rows.raw2strain(raw, SCALE), FS, 14., 30.)
    for name in NAMES:
        y = dw.dsp.fk_filter_sparsefilt(x, pipe.masks[name])
        assert torch.equal(dev["traces"][name], y), name
        assert torch.equal(dev["snr"][name], dw.dsp.snr_tr_array(y, env=True)), name
    inf = dev["traces"]["inf_cos"].cpu().numpy()
    xi, tj = np.unravel_index(np.argmax(inf, axis=None), inf.shape)
    assert dev["argmax"] == (int(xi), int(tj))
    assert torch.equal(dev["section"].cpu(), torch.from_numpy(inf[:, tj]))
    host = pipe.process_file(counts)
    assert host["argmax"] == dev["argmax"]
    for name in NAMES:
        assert host["snr"][name].dtype == np.float64
        assert np.array_equal(host["snr"][name], dev["snr"][name].cpu().numpy().astype(np.float64))
    outs = list(pipe.stream([counts, counts.astype(np.float32)]))
    assert len(outs) == 2 and all(o["argmax"] == host["argmax"] for o in outs)
    assert all(np.array_equal(o["section"], host["section"]) for o in outs)


def test_fkcomp_pipeline_matches_oracle_script(dw):
    """scripts/main_fkcomp.py:56-122 restated on the float64 oracles."""
    import torch
    from das4whales_b200 import pipeline
    from oracle import data_oracle as DH
    nx, ns, sel = 200, 6000, [0, 200, 1]
    counts = _counts(nx, ns, 9)
    tr = O.bp_filt(DH.raw2strain(counts, {"scale_factor": SCALE}), FS, 14., 30.)        # :66
    shape = (nx, ns)
    ref_masks = [O.hybrid_ninf_filter_design(shape, sel, DX, FS, *SPEEDS, 14., 30.),    # :73
                 O.hybrid_ninf_gs_filter_design(shape, sel, DX, FS, *SPEEDS, 14., 30.),  # :79
                 O.hybrid_filter_design(shape, sel, DX, FS, SPEEDS[0], SPEEDS[1], 14., 30.),   # :86
                 O.hybrid_gs_filter_design(shape, sel, DX, FS, SPEEDS[0], SPEEDS[1], 14., 30.)]  # :92
    refs = {n: O.fk_filter_filt(tr, np.asarray(m)) for n, m in zip(NAMES, ref_masks)}
    dev = pipeline.FkCompPipeline(nx, ns, sel, DX, FS, SCALE).process_device(torch.from_numpy(counts).cuda(),
                                                                            with_traces=True)
    for name in NAMES:
        y = dev["traces"][name].cpu().numpy().astype(np.float64)
        assert rel_err(y, refs[name])[0] <= TOL, name
        snr = dev["snr"][name].cpu().numpy()
        assert rel_err(10 ** (snr / 10), 10 ** (O.snr_tr_array(y, env=True) / 10))[0] <= TOL, name
    ref = refs["inf_cos"]
    xi, tj = dev["argmax"]                               # :104; a float32 near-tie may pick another sample of the peak
    assert ref[xi, tj] >= ref.max() - TOL * np.abs(ref).max()
    assert rel_err(dev["section"].cpu().numpy(), ref[:, tj])[0] <= TOL                # :106
    one = pipeline.process_file_fkcomp(counts, {"dx": DX, "fs": FS, "scale_factor": SCALE}, sel)
    assert one["argmax"] == dev["argmax"]
