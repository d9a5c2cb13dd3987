"""GPU: one case per f-k filter route the planner picks from the shape alone (no D4W_* variable set), each checked
against the float64 filter.  tests/test_fk_routes_host.py pins the same shapes to their routes on the CPU and checks
that these routes are all the ones shapes reach (chirp-z columns are tested in test_fk_czt_gpu.py).

Every case asserts the plan (column scheme, tile, column block size, time split) against the host table, then filters
with three masks and compares with the literal float64 fft2 -> x mask -> ifft2 computed on the device:
  * the speed fan (fk_filter_design);
  * the tapered hybrid_ninf mask every reference script uses (even ns only, as in the reference);
  * a scattered dense mask pruned with eps, so that the kept wavenumber rows have holes, which exercises the slot and
    per-plane tables of every column scheme.
It also checks that two runs agree bit for bit and that a two-mask FkFilterBank equals the two single filters.

The alignment cases pin d4w_fk_apply's refusal of a matrix that does not start on the boundary its column kernels
need, and FkFilter's aligned copy of such a view."""
import os

import pytest
import scipy.signal as sps

from test_fk_routes_host import FIELDS, ROUTES

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
TOL = 2e-5
HYB = (1350., 1450., 3300, 3450, 14., 30.)
EPS = 1e-5
D4W_ERR_ARG = 1

# one shape per route of test_fk_routes_host.REACHABLE but chirp-z; nx * ns <= 30 M except the pipelined time split
GPU_ROUTES = [(13122, 1200), (15625, 1210), (20000, 1210),          # scalar k_col_*<512>
              (5510, 1200), (5510, 1210),                           # dual, 4 columns per tile, radix 19 / 29
              (64, 400), (63, 405),                                 # dual, 8 columns per tile
              (6561, 1200), (7203, 1200),                           # TMA <512>
              (6859, 1200), (8303, 1200),                           # TMA <256>
              (1024, 4096), (11020, 1200), (6000, 1200),            # two-level X1 = 16 / 20 / 25, shared-memory level B
              (20000, 1200), (25000, 1200),                         # ... 4 / 2 pairs per level-B tile, one column per tile
              (4096, 1200), (5120, 1200), (6400, 1200),             # fused (16, 16) after X1 = 16 / 20 / 25
              (8000, 1200), (12500, 1200), (15625, 1200),           # fused (20, 16), (20, 25), (25, 25)
              (10000, 2480), (10000, 16400)]                        # pipelined: ragged last chunk; time split T1 = 2


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


def _errs(y, ref):
    import torch
    d = y.to(torch.float64) - ref
    return float(d.abs().max() / ref.abs().max()), float(torch.linalg.vector_norm(d) / torch.linalg.vector_norm(ref))


def _filt64(x, mu, tapering=False):
    """real(ifft2(fft2(x) * mu)) in float64, mu the mask in the un-shifted layout (dsp.py:725-756)."""
    import torch
    x64 = x.to(torch.float64)
    if tapering:
        x64 = x64 * torch.from_numpy(sps.windows.tukey(x.shape[1], alpha=0.03)).to(x.device)[None, :]
    s = torch.fft.fft2(x64)
    del x64
    s *= mu
    return torch.fft.ifft2(s).real


def _scattered(nx, ns, seed):
    """Signed, non-symmetric float32 dense mask (shifted layout) whose rows span nine decades, a fifth of them empty."""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    scale = 10.0 ** torch.empty(nx, 1, device="cuda", dtype=torch.float64).uniform_(-9, 0, generator=g)
    m = torch.randn(nx, ns, device="cuda", dtype=torch.float64, generator=g) * scale
    m[torch.rand(nx, device="cuda", generator=g) < 0.2] = 0.0
    return m.to(torch.float32)


def _pruned_fold(m32, eps):
    """(M_sym with the rows eps prunes zeroed, kept rows, rows with any non-zero): oracle/dsp_oracle.fold_mask and
    fk_filter_filt_pruned restated on the device."""
    import torch
    mu = torch.fft.ifftshift(m32.to(torch.float64))
    msym = 0.5 * (mu + torch.roll(torch.flip(mu, (0, 1)), (1, 1), (0, 1)))
    del mu
    nx = msym.shape[0]
    rowmax = msym[: nx // 2 + 1].abs().to(torch.float32).amax(dim=1)
    keep = rowmax > torch.tensor(eps, dtype=torch.float32, device=rowmax.device)
    drop = torch.nonzero(~keep).flatten()
    msym[drop] = 0.0
    msym[(nx - drop) % nx] = 0.0
    kept = torch.nonzero(keep).flatten()
    return msym, int(kept.numel()), int(torch.count_nonzero(rowmax)), int(kept[-1]) + 1


@pytest.mark.parametrize("nx,ns", GPU_ROUTES)
def test_route_vs_float64(fk, nx, ns):
    import torch
    from oracle import torch_oracle as TO
    import das4whales_b200 as dw
    want = dict(zip(FIELDS, ROUTES[(nx, ns)]))
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    assert (plan.col_scheme, plan.tile, plan.col_threads, plan.t1) == \
        (want["scheme"], 2 * want["nc"], want["col_threads"], want["t1"]), (nx, ns)
    sel = [0, nx, 1]
    x = torch.randn(nx, ns, device="cuda", generator=torch.Generator(device="cuda").manual_seed(nx * 7 + ns))
    report = []

    fan = dw.dsp.fk_filter_design((nx, ns), sel, DX, FS)
    flt = fk.FkFilter(fan)
    y = flt(x)
    assert torch.equal(y, flt(x)), "fan: two runs differ"
    mu = torch.fft.ifftshift(TO.fk_filter_design((nx, ns), sel, DX, FS, device="cuda"))
    report.append(("fan", _errs(y, _filt64(x, mu))))
    del mu, y

    if ns % 2 == 0:
        hyb = dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB)
        y = fk.FkFilter(hyb)(x, tapering=True)
        mu = torch.fft.ifftshift(TO.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB, device="cuda"))
        report.append(("hybrid_ninf tapered", _errs(y, _filt64(x, mu, tapering=True))))
        del mu, y

    m32 = _scattered(nx, ns, nx + ns)
    pflt = fk.FkFilter(m32, eps=EPS)
    y = pflt(x)
    assert torch.equal(y, pflt(x)), "pruned dense: two runs differ"
    msym, kept, nonzero, last = _pruned_fold(m32, EPS)
    assert pflt.rows_kept == kept, (pflt.rows_kept, kept)
    assert 0 < kept < nonzero and last > kept, (kept, nonzero, last)           # holes inside the kept set
    report.append((f"dense pruned ({kept} rows)", _errs(y, _filt64(x, msym))))
    del msym, y, pflt

    dense = fk.FkFilter(m32)
    bank = fk.FkFilterBank([fan, m32])
    ys = bank(x, tapering=True)
    assert torch.equal(ys[0], flt(x, tapering=True)) and torch.equal(ys[1], dense(x, tapering=True)), "bank"
    del ys, bank, dense, flt

    for what, (emax, el2) in report:
        print(f"route {nx} x {ns} scheme {plan.col_scheme}, {what}: max-norm {emax:.2e}, l2 {el2:.2e}")
        assert emax <= TOL and el2 <= TOL, (what, emax, el2)
    fk.free_plans()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("nx,ns", [(6000, 1200), (6561, 1200), (5510, 1210)])
def test_misaligned_pointer_refused_before_any_launch(fk, nx, ns):
    """d4w_fk_apply and d4w_fk_bank_apply refuse an x or y that does not start on the 16-byte (ns % 4 == 0) or 8-byte
    (ns even) boundary, and launch nothing."""
    import torch
    from das4whales_b200 import _lib
    import das4whales_b200 as dw
    L = _lib.lib()
    flt = fk.FkFilter(dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS))
    bank = fk.FkFilterBank([dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS)])
    buf = torch.zeros(nx * ns + 4, device="cuda")
    good, bad = buf[:nx * ns], buf[1:1 + nx * ns]
    out = torch.empty(nx, ns, device="cuda")
    stream = _lib.stream_ptr()
    torch.cuda.synchronize()
    n0 = L.d4w_launch_count()
    for xp, yp in ((bad, out), (good, buf[1:1 + nx * ns])):
        rc = L.d4w_fk_apply(flt.plan.ptr, flt.dm.ptr, _lib.ptr(xp, "float*"), _lib.ptr(yp, "float*"), _lib.ptr(flt._ws()), 0,
                            stream)
        assert rc == D4W_ERR_ARG and "aligned" in _lib.ffi.string(L.d4w_last_error()).decode()
        ys = _lib.ffi.new("float*[]", [_lib.ptr(yp, "float*")])
        rc = L.d4w_fk_bank_apply(bank.plan.ptr, bank.ptr, _lib.ptr(xp, "float*"), ys, _lib.ptr(bank._ws()), 0, stream)
        assert rc == D4W_ERR_ARG
    assert L.d4w_launch_count() == n0
    if ns % 4:                    # 8 bytes is enough when ns % 4 == 2
        rc = L.d4w_fk_apply(flt.plan.ptr, flt.dm.ptr, _lib.ptr(buf[2:2 + nx * ns], "float*"), _lib.ptr(out, "float*"),
                            _lib.ptr(flt._ws()), 0, stream)
        assert rc == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("nx,ns", [(6000, 1200), (6561, 1200), (5510, 1210)])
def test_misaligned_views_filter_like_aligned(fk, nx, ns):
    """A contiguous view that starts one float into its allocation (buf[1:].view(nx, ns)), as input, as output and in a
    bank, gives the aligned result bit for bit (two-level, TMA, and dual at ns % 4 == 2)."""
    import torch
    import das4whales_b200 as dw
    sel = [0, nx, 1]
    x = torch.randn(nx, ns, device="cuda", generator=torch.Generator(device="cuda").manual_seed(nx))
    fan = dw.dsp.fk_filter_design((nx, ns), sel, DX, FS)
    hyb = dw.dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *HYB)
    flt = fk.FkFilter(fan)
    want = flt(x, tapering=True)
    xv = torch.empty(nx * ns + 1, device="cuda")[1:].view(nx, ns)
    xv.copy_(x)
    assert xv.is_contiguous() and xv.data_ptr() % 8
    assert torch.equal(flt(xv, tapering=True), want)
    assert torch.equal(xv, x)                                               # the input is left as it was
    ov = torch.empty(nx * ns + 1, device="cuda")[1:].view(nx, ns)
    assert flt(x, out=ov, tapering=True) is ov and torch.equal(ov, want)
    assert torch.equal(dw.dsp.fk_filter_filt(xv, fan), flt(x))
    bank = fk.FkFilterBank([fan, hyb])
    ref = bank(x)
    o2 = torch.empty(nx * ns + 2, device="cuda")[2:].view(nx, ns)
    outs = bank(xv, outs=[ov, o2])
    assert outs[0] is ov and outs[1] is o2
    assert torch.equal(ov, ref[0]) and torch.equal(o2, ref[1])
