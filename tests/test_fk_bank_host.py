"""CPU: the f-k mask bank's P1-P5 bodies (csrc/fk_kernels.cuh) run on the host in the order d4w_fk_bank_apply
launches them, for small shapes of every column scheme, against the float64 filter of each mask.  Checks the union
slot tables, the exact zero rows of a mask's bank table outside its own support, and that the out-of-place middle pass
leaves the shared forward transform untouched."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from oracle import dsp_oracle as O
from conftest import rel_err, ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
EMUL = os.path.join(ROOT, "tests", "host_emul")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("bank_emul"))
    path = os.path.join(tmp, "fk_bank_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", path,
                        os.path.join(EMUL, "fk_bank_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return path


def _run(exe, tmp, x, masks, eps, taper):
    nx, ns = x.shape
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("4i", nx, ns, int(taper), len(masks)))
        f.write(np.asarray(eps, dtype=np.float64).tobytes())
        f.write(x.astype(np.float32).tobytes())
        for m in masks:
            f.write(np.asarray(m, dtype=np.float32).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    n = len(masks) * nx * ns
    y = np.frombuffer(raw[:4 * n], dtype=np.float32).reshape(len(masks), nx, ns)
    tail = np.frombuffer(raw[4 * n:], dtype=np.int32)
    return y, int(tail[0]), tail[1:1 + len(masks)].tolist(), bool(tail[-3]), bool(tail[-2]), int(tail[-1])


def _masks(rng, nx, ns):
    """Four dense masks: scattered rows spanning nine decades (pruned at eps), a band of low wavenumbers, a band of
    high ones disjoint from it, and a fan; so U is strictly larger than every mask's support."""
    c = np.arange(nx) - nx // 2
    scattered = rng.standard_normal((nx, ns)) * 10.0 ** rng.uniform(-9, 0, (nx, 1))
    scattered[rng.random(nx) < 0.3] = 0.0
    low = rng.standard_normal((nx, ns)) * (np.abs(c) <= max(1, nx // 20))[:, None]
    high = rng.standard_normal((nx, ns)) * ((np.abs(c) > nx // 4) & (np.abs(c) < nx // 3))[:, None]
    fan = O.fk_filter_design((nx, ns), [0, nx, 1], 2.0419046878814697, 200.0, 1400., 1450., 3400., 3500.)
    return [m.astype(np.float32).astype(np.float64) for m in (scattered, low, high, np.asarray(fan))]


# (nx, ns, column bodies emulated): 1 single-level (the dual-lane bodies, which also back the TMA kernels), 2 two-level
# (shared-memory or fused level B; the pipelined kernels run the same bodies), 4 chirp-z
CASES = [(40, 240, 1), (45, 175, 1), (63, 406, 1), (400, 24, 2), (1000, 24, 2), (10000, 16, 2), (4897, 24, 4),
         (103, 120, 4)]


@pytest.mark.parametrize("nx,ns,scheme", CASES)
def test_bank_bodies_against_float64(exe, tmp_path, nx, ns, scheme):
    rng = np.random.default_rng(nx + 3 * ns)
    masks = _masks(rng, nx, ns)
    eps = [1e-4, 0.0, 0.0, 0.0]
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    x64 = x.astype(np.float64)
    for taper in (False, True):
        y, nu, nact, w_untouched, zero_ok, got_scheme = _run(exe, str(tmp_path), x, masks, eps, taper)
        assert got_scheme == scheme
        kept = [np.nonzero(O.fold_rowmax(m) > np.float32(e))[0] for m, e in zip(masks, eps)]
        assert nact == [len(k) for k in kept]
        assert nu == len(set().union(*map(set, kept))) and all(n < nu for n in nact)
        assert w_untouched, "the middle pass must not write the shared forward transform"
        assert zero_ok, "a mask's bank table must be exactly zero outside its own support"
        for i, (m, e) in enumerate(zip(masks, eps)):
            xt = O.taper_data(x64.copy()) if taper else x64
            ref, k = O.fk_filter_filt_pruned(xt, m, e)
            assert k == nact[i]
            err = rel_err(y[i], ref)
            assert err[0] <= 5e-6 and err[1] <= 5e-6, (nx, ns, i, taper, err)
