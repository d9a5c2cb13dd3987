"""CPU: the chirp-z column passes of the f-k filter (csrc/fk_kernels.cuh body_col_fwd_czt / body_col_inv_czt), which take
channel counts with a prime factor above 61, run block by block on the host (tests/host_emul/fk_czt_emul.cu) and checked
against a float64 DFT over channels.  Also checks the chirp and kernel-spectrum tables the planner builds."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from conftest import ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
EMUL = os.path.join(ROOT, "tests", "host_emul")
CZT_MAX_NX = 12800           # 200 KB column budget / 8 B = 25 600-point chirp-z transform -> 2 nx - 1 <= 25 600


def _smooth5(n):
    for p in (2, 3, 5):
        while n % p == 0:
            n //= p
    return n == 1


def _largest_prime(n):
    p, big = 2, 1
    while p * p <= n:
        while n % p == 0:
            big, n = p, n // p
        p += 1
    return max(big, n)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("czt"))
    out = os.path.join(tmp, "fk_czt_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out,
                        os.path.join(EMUL, "fk_czt_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def _run(exe, tmp, nx, ns, taper, keep, x, w_in):
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("4i", nx, ns, int(taper), len(keep)))
        f.write(np.asarray(keep, dtype=np.int32).tobytes())
        f.write(x.astype(np.float32).tobytes())
        f.write(w_in.astype(np.complex64).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    czt, m, nc, nst = struct.unpack("4i", raw[:16])
    o = 16
    nk = len(keep)
    w = np.frombuffer(raw, np.complex64, nk * ns, o).reshape(nk, ns); o += nk * ns * 8
    y = np.frombuffer(raw, np.float32, nx * ns, o).reshape(nx, ns); o += nx * ns * 4
    chirp = np.frombuffer(raw, np.complex64, nx, o); o += nx * 8
    bhat = np.frombuffer(raw, np.complex64, m, o); o += m * 8
    pos2k = np.frombuffer(raw, np.int32, m, o)
    return dict(czt=czt, m=m, nc=nc, w=w, y=y, chirp=chirp, bhat=bhat, pos2k=pos2k)


def _max_rel(a, ref):
    return float(np.max(np.abs(a - ref)) / np.max(np.abs(ref)))


CASES = [(nx, ns, taper, pruned) for nx in (67, 127, 1021, 4897, 6122)
         for ns, taper, pruned in ((9, True, True), (10, False, False), (12, True, False), (7, False, True))]


@pytest.mark.parametrize("nx,ns,taper,pruned", CASES)
def test_czt_column_passes_vs_float64_dft(exe, tmp_path, nx, ns, taper, pruned):
    assert _largest_prime(nx) > 61
    rng = np.random.default_rng(nx * 31 + ns)
    half = nx // 2 + 1
    keep = np.sort(rng.choice(half, size=max(1, half // 3), replace=False)) if pruned else np.arange(half)
    if pruned and nx % 2 == 0:
        keep = np.union1d(keep, [0, nx // 2])                 # both self-conjugate rows, next to holes
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    w_in = (rng.standard_normal((len(keep), ns)) + 1j * rng.standard_normal((len(keep), ns))).astype(np.complex64)
    r = _run(exe, str(tmp_path), nx, ns, taper, keep, x, w_in)
    m = r["m"]
    assert r["czt"] == 1 and m >= 2 * nx - 1 and _smooth5(m) and not any(_smooth5(k) for k in range(2 * nx - 1, m))

    # forward: W[slot, t] = sum_n x_t[n] exp(-2 pi i n k / nx) at the kept k, tapered like dsp.taper_data
    xt = x.astype(np.float64)
    if taper:
        import scipy.signal as sps
        xt = xt * sps.windows.tukey(ns, alpha=0.03)[None, :]
    wref = np.fft.fft(xt, axis=0)[keep]
    assert _max_rel(r["w"].astype(np.complex128), wref) <= 2e-6, (nx, ns, taper, pruned)

    # inverse: y[n, t] = sum_k Y[k, t] exp(+2 pi i n k / nx), Y Hermitian-extended from the kept rows, pruned rows zero,
    # the self-conjugate rows (k = 0, nx/2) taken as real
    spec = np.zeros((half, ns), dtype=np.complex128)
    spec[keep] = w_in
    spec[0] = spec[0].real
    if nx % 2 == 0:
        spec[nx // 2] = spec[nx // 2].real
    yref = nx * np.fft.irfft(spec, n=nx, axis=0)
    assert _max_rel(r["y"].astype(np.float64), yref) <= 2e-6, (nx, ns, taper, pruned)


def test_czt_tables_near_capacity(exe, tmp_path):
    """The chirp c[n] = exp(-i pi (n^2 mod 2 nx) / nx) at the largest accepted awkward channel count, against the exact
    integer reduction evaluated in double; and the kernel spectrum bhat in the M plan's transform order against a
    float64 FFT.  An fp32 phase n^2 / nx is off by more than 1e-3 there, ten thousand times the table's rounding."""
    nx = max(n for n in range(CZT_MAX_NX - 200, CZT_MAX_NX + 1) if _largest_prime(n) > 61)
    ns = 2
    keep = [0, 1]
    x = np.zeros((nx, ns), np.float32)
    r = _run(exe, str(tmp_path), nx, ns, False, keep, x, np.zeros((2, ns), np.complex64))
    assert r["czt"] == 1 and r["m"] <= 25600
    n = np.arange(nx, dtype=np.int64)
    rr = (n * n) % (2 * nx)                                              # exact in int64
    ref = np.exp(-1j * np.pi * rr.astype(np.float64) / nx)
    assert np.max(np.abs(r["chirp"].astype(np.complex128) - ref)) <= 1.2e-7
    naive = np.exp(-1j * np.pi * (np.float32(n) ** 2 / np.float32(nx)).astype(np.float64))   # fp32 accumulated phase
    assert np.max(np.abs(naive - ref)) > 1e-3

    m = r["m"]
    b = np.zeros(m, np.complex128)
    b[:nx] = np.conj(ref)
    b[m - nx + 1:] = np.conj(ref[1:][::-1])
    bh = np.fft.fft(b) / m
    assert np.array_equal(np.sort(r["pos2k"]), np.arange(m))
    assert _max_rel(r["bhat"].astype(np.complex128), bh[r["pos2k"]]) <= 1e-6
