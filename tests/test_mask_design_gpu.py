"""GPU: the hybrid, hybrid_gs and hybrid_ninf_gs masks designed on the device (d4w_mask_design) against the host design that
`todense()` returns -- the float32 plane, the kept rows, the filter, the float64 oracle, FkCompPipeline and the numbers
tools.disp_comprate reads."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu

DX, FS = 2.0419046878814697, 200.0
TOL = 2e-5                              # the f-k tests' tolerance against the float64 oracle
OOI = dict(cs_min=1350., cp_min=1450., cp_max=3300., cs_max=3450., fmin=14., fmax=30.)     # FkCompPipeline's defaults
KINDS = ("hybrid", "hybrid_gs", "hybrid_ninf_gs")


@pytest.fixture(scope="module")
def dw():
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _design(dw, kind, nx, ns):
    sel = [0, nx, 1]
    inf = {k: v for k, v in OOI.items() if k not in ("cp_max", "cs_max")}
    if kind == "hybrid":
        return dw.dsp.hybrid_filter_design((nx, ns), sel, DX, FS, **inf)
    if kind == "hybrid_gs":
        return dw.dsp.hybrid_gs_filter_design((nx, ns), sel, DX, FS, **inf)
    return dw.dsp.hybrid_ninf_gs_filter_design((nx, ns), sel, DX, FS, **OOI)


def _check_plane(dw, kind, nx, ns):
    import torch
    from das4whales_b200 import fk
    mask = _design(dw, kind, nx, ns)
    assert mask.kind == kind
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    dev = mask._design_plane(plan)
    torch.cuda.synchronize()
    host = mask.todense()
    ref = torch.from_numpy(host).float().to(dev.device)
    del host
    nz = ref != 0
    assert torch.equal(dev != 0, nz), (kind, nx, ns)
    assert torch.equal(torch.signbit(dev[nz]), torch.signbit(ref[nz])), (kind, nx, ns)
    ulp = (dev.view(torch.int32) - ref.view(torch.int32)).abs().max().item()
    assert ulp <= 1, (kind, nx, ns, ulp)
    del dev, ref
    for eps in (0.0, 1e-5):
        a = fk.FkFilter(mask, eps=eps).rows_kept
        b = fk.FkFilter(fk.FkMask.from_dense(mask.todense()), eps=eps).rows_kept
        assert a == b, (kind, nx, ns, eps, a, b)
    mask._dense = None                     # drop the host plane before the next size
    fk.free_plans()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("nx,ns", [(551, 1200), (4897, 1200), (11020, 12000)])
def test_device_plane_matches_host_design(dw, kind, nx, ns):
    """Identical zero pattern, at most 1 float32 ulp apart, the same kept rows exactly and at eps = 1e-5.  4 897 channels
    (a prime) take the chirp-z column transform; 11 020 x 12 000 is the OOI record."""
    _check_plane(dw, kind, nx, ns)


def test_device_plane_matches_host_design_at_120000_samples(dw):
    """One 10 000 x 120 000 record (the elementwise kind: its host design is the one that fits in time and memory)."""
    _check_plane(dw, "hybrid", 10000, 120000)


@pytest.mark.parametrize("nx,ns", [(551, 1200), (4897, 1200)])
def test_filter_with_device_design_matches_host_designed_mask(dw, nx, ns):
    import torch
    from das4whales_b200 import fk
    x = torch.from_numpy(np.random.default_rng(nx).standard_normal((nx, ns)).astype(np.float32)).cuda()
    for kind in KINDS:
        mask = _design(dw, kind, nx, ns)
        y = dw.dsp.fk_filter_filt(x, mask)
        yh = dw.dsp.fk_filter_filt(x, fk.FkMask.from_dense(np.asarray(mask)))
        err = ((y - yh).abs().max() / yh.abs().max()).item()
        assert err <= 1e-6, (kind, nx, ns, err)


def test_filter_with_device_design_matches_float64_oracle(dw):
    from oracle import dsp_oracle as O
    nx, ns = 551, 1200
    sel = [0, nx, 1]
    x = np.random.default_rng(3).standard_normal((nx, ns))
    refs = {"hybrid": O.hybrid_filter_design((nx, ns), sel, DX, FS, OOI["cs_min"], OOI["cp_min"], OOI["fmin"], OOI["fmax"]),
            "hybrid_gs": O.hybrid_gs_filter_design((nx, ns), sel, DX, FS, OOI["cs_min"], OOI["cp_min"], OOI["fmin"],
                                                   OOI["fmax"]),
            "hybrid_ninf_gs": O.hybrid_ninf_gs_filter_design((nx, ns), sel, DX, FS, *(OOI[k] for k in
                                                             ("cs_min", "cp_min", "cp_max", "cs_max", "fmin", "fmax")))}
    for kind in KINDS:
        y = dw.dsp.fk_filter_filt(x.copy(), _design(dw, kind, nx, ns))
        ref = O.fk_filter_filt(x.copy(), np.asarray(refs[kind]))
        e = rel_err(y, ref)
        assert e[0] <= TOL and e[1] <= TOL, (kind, e)


def test_fkcomp_pipeline_matches_host_designed_masks(dw):
    import torch
    from das4whales_b200 import fk, pipeline
    nx, ns, sel = 400, 6000, [0, 400, 1]
    scale = 4.0838e-11 * 1550.0 / 2.0419
    counts = np.random.default_rng(5).integers(-20000, 20000, size=(nx, ns), dtype=np.int32)
    pipe = pipeline.FkCompPipeline(nx, ns, sel, DX, FS, scale)
    assert [pipe.masks[n].kind for n in pipeline.FKCOMP_MASKS] == ["hybrid_ninf", "hybrid_ninf_gs", "hybrid", "hybrid_gs"]
    ref = pipeline.FkCompPipeline(nx, ns, sel, DX, FS, scale)
    ref.bank = fk.FkFilterBank([m if m.kind not in fk.DESIGN_KINDS else fk.FkMask.from_dense(np.asarray(m))
                                for m in (ref.masks[n] for n in pipeline.FKCOMP_MASKS)], device=ref.device)
    raw = torch.from_numpy(counts).cuda()
    a = pipe.process_device(raw, with_traces=True)
    b = ref.process_device(raw, with_traces=True)
    for name in pipeline.FKCOMP_MASKS:
        yb = b["traces"][name]
        assert ((a["traces"][name] - yb).abs().max() / yb.abs().max()).item() <= 1e-6, name
        pa, pb = 10 ** (a["snr"][name].double() / 10), 10 ** (b["snr"][name].double() / 10)
        assert ((pa - pb).abs().max() / pb.abs().max()).item() <= 1e-6, name


def test_disp_comprate_numbers_equal_host_masks(dw):
    """The reference's tools.disp_comprate (tools.py:239-250) reads `.data.nbytes` and `nnz`: the host design's own."""
    from das4whales_b200 import fk
    nx, ns = 551, 1200
    for kind in KINDS:
        mask = _design(dw, kind, nx, ns)
        fk.FkFilter(mask)                                   # the device route first: it must not change what the host sees
        host = fk.FkMask.from_dense(mask.todense())
        assert mask.data.nbytes == host.data.nbytes and mask.nnz == host.nnz, kind
        assert np.array_equal(mask.data, host.data)
