"""CPU: the f-k power spectrum's bodies (csrc/fk_kernels.cuh P1 / P2 and csrc/fk_spectrum.cuh's power pass) run on the
host in the order d4w_fk_spectrum_apply launches them, for small shapes of every column scheme and of both time splits
(T1 = 1 and T1 > 1), against the float64 |fftshift(fft2(x))|^2 slice.  The bands cover the whole plane (the Nyquist row
and column of even nx and ns included), a band that clips both halves of each axis, bands holding only +k' rows or only
-k' rows, and single rows and columns.  Also checks that every element of the band is stored exactly once."""
import os
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps

from test_hilbert_czt_host import NVCC, _compile

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
MAX_TOL, L2_TOL = 2e-5, 1e-5


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _compile(tmp_path_factory, "fk_spectrum_emul")


def _run(exe, tmp, x, band, taper):
    nx, ns = x.shape
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("7i", nx, ns, int(taper), *band))
        f.write(x.astype(np.float32).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    nk, nf = band[1] - band[0], band[3] - band[2]
    p = np.frombuffer(raw[:4 * nk * nf], dtype=np.float32).reshape(nk, nf)
    nact, all_written, acc_ok, scheme, t1 = np.frombuffer(raw[4 * nk * nf:], dtype=np.int32).tolist()
    return p, nact, bool(all_written), bool(acc_ok), scheme, t1


def _rows_touching(nx, k_lo, k_hi):
    """Half-plane rows k' in [0, nx/2] with +k' or -k' inside the band's rows (fftshift: row(k) = (k + nx/2) mod nx)."""
    return sum(1 for k in range(nx // 2 + 1)
               if k_lo <= (k + nx // 2) % nx < k_hi or k_lo <= (nx - k + nx // 2) % nx < k_hi)


def _bands(nx, ns):
    h = nx // 2
    return {
        "whole plane": (0, nx, 0, ns),
        "clips both halves": (nx // 4, 3 * nx // 4 + 1, ns // 3, ns - ns // 5),
        "+k' rows only": (h + 1, nx, 0, ns),
        "-k' rows only": (1, h, ns // 2, ns),
        "k = 0 row": (h, h + 1, 0, ns),
        "Nyquist row and column": (0, 1, 0, 1),
        "one column": (0, nx, ns // 2 + 1, ns // 2 + 2),
    }


# (nx, ns, column bodies emulated, T1): 1 single-level dual-lane bodies (which also back the TMA kernels), 2 two-level
# (shared-memory or fused level B; the pipelined kernels run the same bodies), 4 chirp-z
CASES = [(40, 240, 1, 1), (45, 175, 1, 1), (63, 406, 1, 1), (12, 16400, 1, 2), (13, 16875, 1, 3), (400, 24, 2, 1),
         (10000, 16, 2, 1), (4897, 24, 4, 1), (103, 120, 4, 1)]


@pytest.mark.parametrize("nx,ns,scheme,t1", CASES)
def test_power_pass_against_float64(exe, tmp_path, nx, ns, scheme, t1):
    rng = np.random.default_rng(nx + 7 * ns)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    for taper in (False, True):
        x64 = x.astype(np.float64) * (sps.windows.tukey(ns, 0.03)[None, :] if taper else 1.0)
        full = np.abs(np.fft.fftshift(np.fft.fft2(x64))) ** 2
        for what, band in _bands(nx, ns).items():
            p, nact, all_written, acc_ok, got_scheme, got_t1 = _run(exe, str(tmp_path), x, band, taper)
            assert (got_scheme, got_t1) == (scheme, t1)
            assert all_written and acc_ok, (what, all_written, acc_ok)
            assert nact == _rows_touching(nx, band[0], band[1]), what
            ref = full[band[0]:band[1], band[2]:band[3]]
            d = p - ref
            emax = float(np.max(np.abs(d)) / np.max(ref))
            el2 = float(np.linalg.norm(d) / np.linalg.norm(ref))
            assert emax <= MAX_TOL and el2 <= L2_TOL, (nx, ns, what, taper, emax, el2)
