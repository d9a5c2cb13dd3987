"""CPU: k_row_mid_fused is instantiated once per (first, last) radix pair (D4W_ROW_FUSED_PAIRS, fft_smem.cuh).  The list
must be exactly the pairs the row planner produces, and the specialised body must match a float64 FFT -> table -> IFFT."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import rel_err, ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
SRC = os.path.join(ROOT, "tests", "host_emul", "row_fused_emul.cu")
ENV = {k: v for k, v in os.environ.items() if not k.startswith("D4W_")}     # planner defaults


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("row_fused") / "row_fused_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def test_fused_pairs_are_the_planners(exe):
    """Every f-k / Hilbert / chirp-z row plan with split rows and in-register ends has its kernel, no kernel is unused,
    and every such plan takes the fused route by default."""
    lines = subprocess.run([exe, "pairs"], capture_output=True, text=True, check=True, env=ENV).stdout.split()
    assert "unfused" not in lines
    toks = [lines[i:i + 3] for i in range(0, len(lines), 3)]
    plan = {(int(a), int(b)) for k, a, b in toks if k == "plan"}
    built = {(int(a), int(b)) for k, a, b in toks if k == "built"}
    assert plan and plan == built, (sorted(plan - built), sorted(built - plan))


def test_fused_body_config2(exe, tmp_path):
    """ns = 120 000 (T1 = 12, T2 = 10 000 = 20 x 20 x 25): the (20, 25) body with a real mask table in place and out of
    place, and with a complex table shared by all rows (chirp-z rows), against float64."""
    ns = 120000
    rng = np.random.default_rng(3)
    w = (rng.standard_normal((2, ns)) + 1j * rng.standard_normal((2, ns))).astype(np.complex64)
    tab = rng.standard_normal((2, ns)).astype(np.float32)
    tc = (rng.standard_normal(ns) + 1j * rng.standard_normal(ns)).astype(np.complex64)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(w.tobytes() + tab.tobytes() + tc.tobytes())
    subprocess.run([exe, "body", str(ns), fin, fout], check=True, env=ENV)
    raw = np.fromfile(fout, dtype=np.int32, count=4)
    t1, t2, r0, rl = (int(v) for v in raw)
    assert (t1, t2, r0, rl) == (12, 10000, 20, 25)
    pos2k = np.fromfile(fout, dtype=np.int32, count=4 + t2)[4:]
    res = np.fromfile(fout, dtype=np.complex64, offset=4 * (4 + t2)).reshape(3, 2, ns)

    def ref(table, stride):
        out = np.empty((2, ns), dtype=np.complex128)
        for s in range(2):
            for k1 in range(t1):
                g = w[s, k1 * t2:(k1 + 1) * t2].astype(np.complex128)
                m = np.empty(t2, dtype=table.dtype)
                m[pos2k] = table[s * stride + k1 * t2: s * stride + (k1 + 1) * t2]
                out[s, k1 * t2:(k1 + 1) * t2] = t2 * np.fft.ifft(np.fft.fft(g) * m)      # the engine's inverse is unscaled
        return out

    yr = ref(tab.ravel().astype(np.float64), ns)
    yc = ref(tc.astype(np.complex128), 0)
    for got, want in ((res[0], yr), (res[1], yr), (res[2], yc)):
        assert rel_err(np.stack([got.real, got.imag]), np.stack([want.real, want.imag]))[0] <= 5e-6
    assert np.array_equal(res[0], res[1])
