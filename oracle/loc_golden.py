"""oracle/loc_golden.py -- TEST INFRASTRUCTURE for localisation.

Loads the reference's loc module *unmodified* (it needs only NumPy) from the reference tree oracle/ref_loader.py points at,
runs it and the float64 restatement (oracle/loc_oracle.py) on identical seeded inputs, asserts they agree, and writes the
reference's outputs to tests/golden/loc.npz.  The reference tree exists only where fixtures are made, so the fixture is
what the GPU tests read.  The other fixtures (oracle/make_golden.py) are not rewritten.

    python -m oracle.loc_golden [out_dir]      # from the repo root; out_dir defaults to tests/golden
"""
import contextlib
import importlib.util
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import loc_oracle as LO, ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
LOC_C0 = 1490.0
# (whale x, y, z, fix_z): the first is reached from the reference's fixed first guess, the others are not (loc.py:84-86)
LOC_CASES = [(40000., 23000., -50., True), (12000., 30000., -50., True), (30000., 45000., -50., True),
             (40000., 23000., -50., False), (5000., 20000., -400., False)]

_cache = {}


def load_loc():
    """The reference's loc module (unmodified; it needs only NumPy)."""
    if "loc" in _cache:
        return _cache["loc"]
    src = os.path.join(ref_loader.REF_ROOT, "src", "das4whales", "loc.py")
    if not os.path.isfile(src):
        raise FileNotFoundError(f"reference loc.py not found under {ref_loader.REF_ROOT}")
    spec = importlib.util.spec_from_file_location("das4whales.loc", src)
    m = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = m
    spec.loader.exec_module(m)
    _cache["loc"] = m
    return m


def close(a, b, tol, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = np.max(np.abs(a - b)) / max(np.max(np.abs(a)), 1e-300)
    assert err <= tol, f"{what}: oracle vs reference rel err {err:.3e} > {tol}"


def make_loc(out_dir=OUT):
    """loc.npz: the reference's solve_lq (with its printed lines), cal_variance_residuals, calc_covariance_matrix and
    calc_uncertainty_position on a bent 800-channel cable, and the singular covariance branch (a constant-depth cable with
    the whale at that depth, free z)."""
    loc = load_loc()
    rng = np.random.default_rng(2024)
    cable = LO.bent_cable(800)
    out = dict(cable=cable, c0=LOC_C0, cases=np.array(LOC_CASES))
    for k, (x, y, z, fz) in enumerate(LOC_CASES):
        T = LO.arrivals(cable, (x, y, z), 3.0, LOC_C0, 2e-3, rng)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            n = loc.solve_lq(T, cable, LOC_C0, fix_z=bool(fz))
        var = loc.cal_variance_residuals(T, loc.calc_arrival_times(n[-1], cable, n[:3], LOC_C0), bool(fz))
        cbuf = io.StringIO()
        with contextlib.redirect_stdout(cbuf):
            cov = loc.calc_covariance_matrix(cable, n, LOC_C0, var, bool(fz))
            unc = loc.calc_uncertainty_position(cable, n, LOC_C0, var, bool(fz))
        n_o, _ = LO.gauss_newton(T, cable, LOC_C0, np.r_[LO.REF_GUESS, T.min()], 10, bool(fz))
        close(n, n_o, tol=0.0, what=f"loc solve {k}")
        close(var, LO.variance(T, cable, n, LOC_C0, bool(fz)), tol=1e-15, what=f"loc var {k}")
        C, _ = LO.covariance_unscaled(cable, n, LOC_C0, bool(fz))
        close(cov, var * C, tol=1e-15, what=f"loc cov {k}")
        out.update({f"T{k}": T, f"n{k}": n, f"stdout{k}": np.array(buf.getvalue()), f"var{k}": var, f"cov{k}": cov,
                    f"unc{k}": unc, f"covout{k}": np.array(cbuf.getvalue())})
    flat = cable.copy()
    flat[:, 2] = -100.0
    whale = np.array([20000., 30000., -100., 3.0])
    cbuf = io.StringIO()
    with contextlib.redirect_stdout(cbuf):
        cov = loc.calc_covariance_matrix(flat, whale, LOC_C0, 4e-6, False)
        unc = loc.calc_uncertainty_position(flat, whale, LOC_C0, 4e-6, False)
    assert cbuf.getvalue() == "Matrix is singular\nMatrix is singular\n", cbuf.getvalue()
    C, singular = LO.covariance_unscaled(flat, whale, LOC_C0, False)
    assert singular
    close(cov, 4e-6 * C, tol=1e-15, what="loc singular cov")
    out.update(flat_cable=flat, flat_whale=whale, flat_var=4e-6, flat_cov=cov, flat_unc=unc, flat_covout=np.array(cbuf.getvalue()))
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "loc.npz"), **out)


if __name__ == "__main__":
    make_loc(sys.argv[1] if len(sys.argv) > 1 else OUT)
