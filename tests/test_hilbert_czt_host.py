"""CPU: the chirp-z Hilbert rows (row lengths with no T1 x T2 split, csrc/hilbert_czt.cuh) run on the host through
tests/host_emul/row_czt_emul.cu -- the planner's choices, the chirp and kernel-spectrum tables, and the whole-row and split
kernel bodies against float64 scipy.signal.hilbert.  Also pins the f-k filter's chirp-z channel tables, which share the
table builder, byte for byte to tests/golden/czt_col_tables.npz."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps

from conftest import ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
EMUL = os.path.join(ROOT, "tests", "host_emul")
ROUTES = [{}, {"D4W_ROW_FUSED": "0"}]


def _compile(tmp_path_factory, name):
    out = os.path.join(str(tmp_path_factory.mktemp(name)), name)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out,
                        os.path.join(EMUL, name + ".cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _compile(tmp_path_factory, "row_czt_emul")


def _smooth5(n):
    for p in (2, 3, 5):
        while n % p == 0:
            n //= p
    return n == 1


def _env(extra):
    env = {k: v for k, v in os.environ.items() if k not in ("D4W_ROW_FUSED", "D4W_T1")}
    env.update(extra)
    return env


def _plans(exe, lengths, extra=None):
    r = subprocess.run([exe, "plan"] + [str(n) for n in lengths], capture_output=True, text=True, check=True, env=_env(extra or {}))
    out = {}
    for line in r.stdout.splitlines():
        f = line.split(" ", 2)
        out[int(f[0])] = (f[1], f[2])
    return out


def test_planner_choices(exe):
    p = _plans(exe, [600, 12000, 36000, 120000, 240000, 1126, 1501, 8191, 8193, 15001, 127997, 128001])
    # lengths with a direct split keep exactly their plan
    assert p[600] == ("direct", "1 600") and p[12000] == ("direct", "1 12000")
    assert p[36000] == ("direct", "4 9000") and p[120000] == ("direct", "12 10000") and p[240000] == ("direct", "25 9600")
    czt = {n: tuple(int(v) for v in p[n][1].split()) for n in (1126, 1501, 8191, 8193, 15001, 127997)}
    assert all(p[n][0] == "czt" for n in czt)
    # (M, T1, T2, fused): whole row in one CTA while M <= 16 384, split rows above
    assert czt[1126] == (2304, 1, 2304, 0) and czt[1501] == (3072, 1, 3072, 0) and czt[8191] == (16384, 1, 16384, 0)
    assert czt[8193] == (16875, 3, 5625, 1) and czt[15001] == (30375, 3, 10125, 1) and czt[127997] == (256000, 25, 10240, 1)
    for n, (m, t1, t2, _) in czt.items():
        assert m >= 2 * n - 1 and _smooth5(m) and t1 * t2 == m and not any(_smooth5(k) for k in range(2 * n - 1, m)), n
    assert p[128001][0] == "error" and "128000" in p[128001][1]
    # D4W_ROW_FUSED=0 selects k_row_mid for the split rows, as on the direct route
    q = _plans(exe, [8193, 15001], {"D4W_ROW_FUSED": "0"})
    assert q[8193] == ("czt", "16875 3 5625 0") and q[15001] == ("czt", "30375 3 10125 0")


def _tables(exe, tmp_path, n, extra=None):
    fout = os.path.join(str(tmp_path), f"tab{n}.bin")
    subprocess.run([exe, "tables", str(n), fout], check=True, env=_env(extra or {}))
    raw = open(fout, "rb").read()
    m, t1, t2, fused = struct.unpack("4i", raw[:16])
    o = 16
    chirp = np.frombuffer(raw, np.complex64, n, o); o += n * 8
    bhat = np.frombuffer(raw, np.complex64, m, o); o += m * 8
    tab = np.frombuffer(raw, np.int32, m, o)
    return dict(m=m, t1=t1, t2=t2, fused=fused, chirp=chirp, bhat=bhat, tab=tab)


def _exact_chirp(n):
    k = np.arange(n, dtype=np.int64)
    return np.exp(-1j * np.pi * ((k * k) % (2 * n)).astype(np.float64) / n)


def test_chirp_near_limit(exe, tmp_path):
    """c[t] at N = 127 997 against the exact integer reduction; an fp32 phase t^2 / N misses the same bound by far."""
    n = 127997
    r = _tables(exe, tmp_path, n)
    ref = _exact_chirp(n)
    bound = 1.2e-7
    assert np.max(np.abs(r["chirp"].astype(np.complex128) - ref)) <= bound
    t = np.arange(n, dtype=np.float32)
    naive = np.exp(-1j * np.pi * (t * t / np.float32(n)).astype(np.float64))
    assert np.max(np.abs(naive - ref)) > 1000 * bound


@pytest.mark.parametrize("n,extra,fused", [(1501, {}, 0), (8193, {}, 1), (8193, {"D4W_ROW_FUSED": "0"}, 0)])
def test_kernel_spectrum_table_orders(exe, tmp_path, n, extra, fused):
    """B^ = FFT_M(conj c, wrapped) / M in the middle pass's table order (k_row_mid: kt1 + T1 * pos2k_row[pos];
    k_row_mid_fused: its own order) against a float64 FFT."""
    r = _tables(exe, tmp_path, n, extra)
    m = r["m"]
    assert r["fused"] == fused
    assert np.array_equal(np.sort(r["tab"]), np.arange(m))
    c = _exact_chirp(n)
    b = np.zeros(m, np.complex128)
    b[:n] = np.conj(c)
    b[m - n + 1:] = np.conj(c[1:][::-1])
    bh = np.fft.fft(b) / m
    got = r["bhat"].astype(np.complex128)
    assert np.max(np.abs(got - bh[r["tab"]])) / np.max(np.abs(bh)) <= 1e-6


def test_channel_tables_bit_identical(tmp_path_factory, tmp_path):
    """The f-k filter's chirp-z channel tables now come from the shared builder: byte for byte what they were."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "czt_col_tables.npz"))
    nx, m = int(g["nx"]), int(g["m"])
    exe = _compile(tmp_path_factory, "fk_czt_emul")
    ns = 2
    fin, fout = os.path.join(str(tmp_path), "in.bin"), os.path.join(str(tmp_path), "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("4i", nx, ns, 0, 2))
        f.write(np.asarray([0, 1], np.int32).tobytes())
        f.write(np.zeros((nx, ns), np.float32).tobytes())
        f.write(np.zeros((2, ns), np.complex64).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    czt, m2 = struct.unpack("2i", raw[:8])
    assert czt == 1 and m2 == m
    o = 16 + 2 * ns * 8 + nx * ns * 4
    assert raw[o:o + nx * 8] == g["chirp"].tobytes()
    assert raw[o + nx * 8:o + nx * 8 + m * 8] == g["bhat"].tobytes()


def _run(exe, tmp, x, mode, extra):
    nrows, n = x.shape
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("3i", n, nrows, mode))
        f.write(np.ascontiguousarray(x, np.float32).tobytes())
    subprocess.run([exe, "run", fin, fout], check=True, env=_env(extra))
    raw = open(fout, "rb").read()
    m, t1, pair = struct.unpack("3i", raw[:12])
    return m, t1, pair, np.frombuffer(raw, np.float32, nrows * n, 12).reshape(nrows, n)


@pytest.mark.parametrize("extra", ROUTES)
@pytest.mark.parametrize("n", [751, 1126, 8193, 8194])
def test_bodies_vs_scipy_hilbert(exe, tmp_path, n, extra):
    """Whole-row body (751 odd, 1 126 even) and the five split bodies (8 193 odd, 8 194 even; T1 = 3) in all four modes,
    with 1, 2 and 3 rows (an odd row count leaves the last pair half empty)."""
    for nrows in (1, 2, 3):
        rng = np.random.default_rng(n * 7 + nrows)
        x = rng.standard_normal((nrows, n)).astype(np.float32)
        x64 = x.astype(np.float64)
        a = sps.hilbert(x64, axis=1)
        var = x64.var(axis=1, keepdims=True)
        refs = {0: np.abs(a), 2: a.imag, 3: np.abs(a) / np.sqrt(var)}
        for mode, ref in refs.items():
            m, t1, pair, y = _run(exe, str(tmp_path), x, mode, extra)
            assert (t1 == 1) == (n < 8192) and pair == (t1 > 1)
            e = np.max(np.abs(y - ref)) / np.max(np.abs(ref))
            assert e <= 2e-6, (n, nrows, mode, e)
        _, _, _, y = _run(exe, str(tmp_path), x, 1, extra)
        lin, lref = 10 ** (y.astype(np.float64) / 10), np.abs(a) ** 2 / var
        assert np.max(np.abs(lin - lref)) / np.max(lref) <= 1e-5, (n, nrows)
