"""CPU: the device design of the hybrid, hybrid_gs and hybrid_ninf_gs masks (d4w_mask_design), emulated on the host with the
kernels' own bodies, against the host design that `todense()` returns; the domain the device route covers, and the C entry's
argument checks."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import das4whales_b200 as dw
from das4whales_b200 import _lib, fk
from conftest import ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
DX, FS = 2.0419046878814697, 200.0
OOI = dict(cs_min=1350., cp_min=1450., cp_max=3300., cs_max=3450., fmin=14., fmax=30.)


def _design(kind, shape, sel, dx, fs, **kw):
    inf = {k: v for k, v in kw.items() if k not in ("cp_max", "cs_max")}
    if kind == "hybrid":
        return dw.dsp.hybrid_filter_design(shape, sel, dx, fs, **inf)
    if kind == "hybrid_gs":
        return dw.dsp.hybrid_gs_filter_design(shape, sel, dx, fs, **inf)
    return dw.dsp.hybrid_ninf_gs_filter_design(shape, sel, dx, fs, **kw)


# (shape, selected_channels, dx, fs, keyword arguments, kinds)
ALL = ("hybrid", "hybrid_gs", "hybrid_ninf_gs")
GS = ("hybrid_gs", "hybrid_ninf_gs")
CASES = [
    ((10, 10), [0, 1, 2], 1, 100, {}, ALL),                                   # the reference tests' arguments
    ((40, 240), [0, 40, 1], DX, FS, dict(cs_min=1400., cp_min=1450., fmin=15., fmax=25.), ALL),     # the golden shapes
    ((38, 120), [0, 38, 1], DX, FS, dict(cs_min=1400., cp_min=1450., fmin=15., fmax=25.), ALL),
    ((41, 240), [0, 41, 1], DX, FS, OOI, ALL),                                # odd nx
    ((40, 239), [0, 40, 1], DX, FS, OOI, ALL),                                # odd ns
    ((43, 167), [0, 43, 1], DX, FS, OOI, ALL),                                # both odd
    ((1, 240), [0, 1, 1], DX, FS, OOI, ALL),
    ((2, 240), [0, 2, 1], DX, FS, OOI, ALL),
    ((120, 600), [0, 120, 1], DX, FS, OOI, ALL),
    ((300, 400), [0, 600, 2], DX, FS, dict(cs_min=1450., cp_min=1450., fmin=14., fmax=30.), ("hybrid",)),   # ks == kp
    ((40, 240), [0, 40, 1], DX, 50., dict(fmin=15., fmax=25.), GS),          # col_hi = 0: fmax + 4 above every frequency
    ((41, 240), [0, 41, 1], DX, 50., dict(fmin=15., fmax=25.), GS),          # ... with an odd nx's centre row doubled
    ((40, 240), [0, 40, 1], DX, 50., dict(fmin=-30., fmax=10.), ALL),        # H reaches column 0 (and its mirror ns - 1)
    ((41, 120), [0, 41, 1], 6.0, 50., dict(cs_min=300., cp_min=320., cp_max=500., cs_max=600., fmin=-30., fmax=10.), ALL),
]


@pytest.fixture(scope="module")
def design_exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("design") / "mask_design_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", exe,
                        os.path.join(ROOT, "tests", "host_emul", "mask_design_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return exe


def _emulate(exe, mask, tmp_path):
    p = mask.params
    nx, ns = mask.shape
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("<5i", fk.DESIGN_KINDS[mask.kind], nx, ns, p["col_lo"], p["col_hi"]))
        f.write(struct.pack("<5d", p["kval"], p["fval"], p["cs_min"], p["cp_min"], p["cp_max"]))
        f.write(np.ascontiguousarray(p["H"], dtype="<f8").tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr
    return np.fromfile(fout, dtype="<f8").reshape(nx, ns)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_emulated_device_design_matches_host(design_exe, tmp_path, case):
    shape, sel, dx, fs, kw, kinds = CASES[case]
    for kind in kinds:
        mask = _design(kind, shape, sel, dx, fs, **kw)
        assert mask.kind == kind and mask._dense is None, (kind, "the design is deferred")
        host = mask.todense()
        assert host is mask.todense()                              # computed once, then cached
        emu = _emulate(design_exe, mask, tmp_path)
        assert np.array_equal(emu != 0, host != 0), (kind, shape)
        assert np.max(np.abs(emu - host)) <= 1e-13, (kind, shape, np.max(np.abs(emu - host)))


def test_col_hi_zero_case_keeps_its_column_range():
    m = dw.dsp.hybrid_gs_filter_design((40, 240), [0, 40, 1], DX, 50., fmin=15., fmax=25.)
    assert m.params["col_hi"] == 0 < m.params["col_lo"]
    # the host restatement of hybrid_filter_design cannot build this case; it raises as it did
    with pytest.raises(ValueError):
        dw.dsp.hybrid_filter_design((40, 240), [0, 40, 1], DX, 50., fmin=15., fmax=25.)


def test_edge_case_reaches_columns_0_and_ns_minus_1():
    m = dw.dsp.hybrid_ninf_gs_filter_design((40, 240), [0, 40, 1], DX, 50., fmin=-30., fmax=10.)
    assert m.params["H"][0] == 1 and m.params["col_lo"] == 0


# arguments the interval argument does not cover: the host design, wrapped as a dense mask, as before
OUT_OF_DOMAIN = [
    dict(cp_min=-1450.), dict(cs_min=0.), dict(cp_min=float("inf")), dict(cp_min=float("nan")), dict(fmin=25., fmax=15.),
    dict(fmin=20., fmax=20.), dict(fmax=float("inf")),
]


@pytest.mark.parametrize("kw", OUT_OF_DOMAIN)
def test_out_of_domain_arguments_give_todays_dense_mask(kw):
    shape, sel = (40, 240), [0, 40, 1]
    base = dict(cs_min=1400., cp_min=1450., cp_max=3400., cs_max=3500., fmin=15., fmax=25.)
    base.update(kw)
    inf = {k: v for k, v in base.items() if k not in ("cp_max", "cs_max")}
    with np.errstate(all="ignore"):
        cases = [(dw.dsp.hybrid_gs_filter_design, dw.dsp._hybrid_gs_host, inf,
                  (base["fmin"], base["fmax"], base["cp_min"])),
                 (dw.dsp.hybrid_ninf_gs_filter_design, dw.dsp._hybrid_ninf_gs_host, base,
                  (base["fmin"], base["fmax"], base["cp_min"], base["cp_max"])),
                 (dw.dsp.hybrid_filter_design, dw.dsp._hybrid_host, inf,
                  (base["cs_min"], base["cp_min"], base["fmin"], base["fmax"]))]
        for fn, host, args, hargs in cases:
            try:
                ref = host(shape, sel, DX, FS, *hargs)
            except ValueError:
                with pytest.raises(ValueError):
                    fn(shape, sel, DX, FS, **args)
                continue
            m = fn(shape, sel, DX, FS, **args)
            assert m.kind == "dense", (fn.__name__, kw)
            assert np.array_equal(m.todense(), ref, equal_nan=True), (fn.__name__, kw)


def test_negative_sampling_rate_takes_the_host_route():
    m = dw.dsp.hybrid_gs_filter_design((40, 240), [0, 40, 1], DX, -FS)
    assert m.kind == "dense"


def test_design_entry_checks_arguments():
    """D4W_ERR_ARG (ValueError) before any device work."""
    L = _lib.lib()
    assert L.d4w_mask_design_workspace_bytes(0, 10) == 0
    ws = L.d4w_mask_design_workspace_bytes(40, 240)
    assert ws >= 8 * 240
    H = np.zeros(240)
    H[150:170] = 1.0
    hp = _lib.ffi.cast("double*", H.ctypes.data)
    dummy = _lib.ffi.cast("void*", 256)
    out = _lib.ffi.cast("float*", 256)
    good = dict(kind=1, out=out, nx=40, ns=240, kval=0.01, fval=0.8, cs_min=1400., cp_min=1450., cp_max=3400., fmin=15.,
                fmax=25., col_lo=140, col_hi=180, H=hp, ws=dummy)
    bad = [dict(kind=3), dict(kind=-1), dict(out=_lib.ffi.NULL), dict(H=_lib.ffi.NULL), dict(ws=_lib.ffi.NULL), dict(nx=0),
           dict(ns=0), dict(fval=0.0), dict(fval=-0.8), dict(kval=float("inf")), dict(cp_min=-1.0), dict(cs_min=0.0),
           dict(cp_max=float("nan")), dict(fmin=25., fmax=15.), dict(fmax=float("inf")), dict(col_lo=-1), dict(col_hi=241),
           dict(kind=0, col_lo=180, col_hi=140)]
    H2 = H.copy()
    H2[100] = 1.0                                      # two bands: not a gs H
    H3 = H.copy()
    H3[160] = 0.5
    bad += [dict(H=_lib.ffi.cast("double*", H2.ctypes.data)), dict(H=_lib.ffi.cast("double*", H3.ctypes.data))]
    for b in bad:
        a = dict(good, **b)
        rc = L.d4w_mask_design(a["kind"], a["out"], a["nx"], a["ns"], a["kval"], a["fval"], a["cs_min"], a["cp_min"],
                               a["cp_max"], a["fmin"], a["fmax"], a["col_lo"], a["col_hi"], a["H"], a["ws"], _lib.ffi.NULL)
        assert rc == 1, b
