"""CPU: the SAME __host__ __device__ kernel bodies the GPU runs (csrc/fk_kernels.cuh,
fft_smem.cuh) executed block-by-block on the host and checked against the oracle.  Catches
indexing / twiddle / fold / untangle errors without a GPU."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps

from oracle import dsp_oracle as O
from conftest import rel_err, ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
EMUL = os.path.join(ROOT, "tests", "host_emul")
DX, FS = 2.0419046878814697, 200.0


def _build(name, tmp):
    exe = os.path.join(tmp, name)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a",
                        "-o", exe, os.path.join(EMUL, name + ".cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return exe


@pytest.fixture(scope="module")
def tmpdir_mod(tmp_path_factory):
    return str(tmp_path_factory.mktemp("emul"))


def test_fft_engine_emulation(tmpdir_mod):
    exe = _build("fft_engine_emul", tmpdir_mod)
    for maxr in ("25", "16", "8"):
        r = subprocess.run([exe, maxr], capture_output=True, text=True)
        assert r.returncode == 0 and "OK" in r.stdout, r.stdout


def test_pfa_2520_engine_emulation(tmpdir_mod):
    """prime-factor 2520-point transform of the matched filter (csrc/fft_pfa.cuh): radix 5/7/8/9 dual butterflies, CRT maps"""
    exe = _build("pfa_emul", tmpdir_mod)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout


def _run(exe, tmp, nx, ns, kind, taper, x, kval, fval, c, H=None, dense=None, col=(0, 0), env=None):
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("6i", nx, ns, kind, int(taper), col[0], col[1]))
        f.write(struct.pack("6d", kval, fval, *c))
        f.write(x.astype(np.float32).tobytes())
        if kind == 1:
            f.write(np.asarray(H, dtype=np.float64).tobytes())
        if kind == 2:
            f.write(np.asarray(dense, dtype=np.float32).tobytes())
    e = dict(os.environ)
    e.update(env or {})
    subprocess.run([exe, fin, fout], check=True, env=e)
    raw = open(fout, "rb").read()
    return np.frombuffer(raw[: nx * ns * 4], dtype=np.float32).reshape(nx, ns), struct.unpack("5i", raw[nx * ns * 4:])


CASES = [(40, 240, 1, False, None), (45, 175, 1, True, None), (38, 120, 2, False, None),
         (100, 1200, 1, True, {"D4W_T1": "12"}), (100, 1200, 1, True, {"D4W_T1": "12", "D4W_ROW_FUSED": "1"}),
         (30, 600, 1, False, {"D4W_T1": "5", "D4W_COL_NC": "1"}),
         (250, 360, 1, False, {"D4W_T1": "6", "D4W_COL_NC": "4"}),
         (10000, 16, 1, False, None),      # the bench column plan (two-level 25 x 400, fused 20 x 20 level B)
         (10000, 10, 1, True, {"D4W_COLB_RA": "16"}), (10000, 8, 1, False, {"D4W_COLB_RA": "25"}),
         (10000, 8, 1, False, {"D4W_COLB_FUSED": "0"}),      # shared-memory engine level B
         (10000, 44, 1, True, {"D4W_COL_CHUNK_PAIRS": "8"}),  # three time chunks, the last one ragged
         (6400, 36, 1, True, {"D4W_COL_X1": "16", "D4W_COL_CHUNK_PAIRS": "8", "D4W_COLB_FUSED": "0"}),
         (6400, 12, 1, False, {"D4W_COL_X1": "16"}), (8000, 8, 1, True, {"D4W_COL_X1": "20"}),
         (10000, 8, 1, False, {"D4W_COL_TWO_LEVEL": "0"}),   # single-level dual column kernels (20x20x25)
         (400, 24, 1, True, None), (320, 12, 1, True, {"D4W_COL_X1": "16"}), (500, 16, 1, False, {"D4W_COL_X1": "20"}),
         (10000, 16, 1, True, {"D4W_COL_PIPE3": "1"}),        # X1 = 10, three-stage 10 x 10 x 10 level B (k_col3_pipe's bodies)
         (1000, 24, 1, False, {"D4W_COL_PIPE3": "1", "D4W_PIPE3_CQ": "4", "D4W_PIPE3_THREADS": "32"})]    # 5 x 5 x 4, 3 chunks


def test_fk_pipeline_emulation(tmpdir_mod):
    exe = _build("fk_pipeline_emul", tmpdir_mod)
    rng = np.random.default_rng(0)
    for nx, ns, step, taper, env in CASES:
        x32 = rng.standard_normal((nx, ns)).astype(np.float32)
        x64 = x32.astype(np.float64)
        sel = [0, nx * step, step]
        kval, fval = 1.0 / (nx * (step * DX)), 1.0 / (ns * (1 / FS))
        c = (1400., 1450., 3400., 3500.)
        M = O.fk_filter_design((nx, ns), sel, DX, FS, *c)
        ref = O.fk_filter_filt(x64.copy(), M, tapering=taper)
        y, tail = _run(exe, tmpdir_mod, nx, ns, 0, taper, x32, kval, fval, c, env=env)
        assert 0 < tail[0] < nx // 2 + 1, "fan mask support must prune wavenumber rows"
        assert rel_err(y, ref)[0] <= 5e-6, (nx, ns, "fan")
        y2, _ = _run(exe, tmpdir_mod, nx, ns, 2, taper, x32, kval, fval, c, dense=np.ascontiguousarray(M), env=env)
        assert rel_err(y2, ref)[0] <= 5e-6, (nx, ns, "dense")
        if ns % 2 == 0:
            cc = (1350., 1450., 3300., 3450.)
            Mh = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *cc, 14., 30.)
            freq = np.fft.fftshift(np.fft.fftfreq(ns, d=1 / FS))
            b, a = sps.butter(8, [14 / (FS / 2), 30 / (FS / 2)], "bp")
            H = np.concatenate((np.zeros(ns // 2), np.abs(sps.freqz(b, a, worN=ns // 2)[1]) ** 2))
            i0, i1 = int(np.argmax(freq >= 0)), int(np.argmax(freq >= 44))
            refh = O.fk_filter_filt(x64.copy(), Mh, tapering=taper)
            yh, _ = _run(exe, tmpdir_mod, nx, ns, 1, taper, x32, kval, fval, cc, H=H, col=(i0, i1), env=env)
            assert rel_err(yh, refh)[0] <= 5e-6, (nx, ns, "hybrid_ninf")


SUPPORT_CASES = [(40, 240, None), (45, 175, None), (400, 24, None), (320, 12, None),
                 (10000, 16, None),                                   # two-level 25 x 400, fused 20 x 20 level B
                 (10000, 8, {"D4W_COLB_FUSED": "0"}), (10000, 8, {"D4W_COL_TWO_LEVEL": "0"}),
                 (1000, 24, {"D4W_COL_PIPE3": "1", "D4W_PIPE3_CQ": "4", "D4W_PIPE3_THREADS": "32"}),
                 (6400, 12, {"D4W_COL_X1": "16"}), (8000, 8, {"D4W_COL_X1": "20"})]


def test_fk_pipeline_emulation_dense_supports(tmpdir_mod):
    """Dense masks whose wavenumber support has holes, a single row whose conjugate partner row is empty, or only the
    DC and Nyquist rows: the kept-row tables of every column scheme (slot positions, two-level plane entries and need
    tables) against the float64 filter."""
    exe = _build("fk_pipeline_emul", tmpdir_mod)
    rng = np.random.default_rng(4)
    for nx, ns, env in SUPPORT_CASES:
        x32 = rng.standard_normal((nx, ns)).astype(np.float32)
        for support in ("scattered", "one_row", "dc_nyquist"):
            m = rng.standard_normal((nx, ns))                  # signed, not symmetric
            if support == "scattered":
                rows = rng.random(nx) < 0.1
            elif support == "one_row":                         # shifted row nx//2 + 3 is k = 3; row k = -3 stays empty
                rows = np.arange(nx) == nx // 2 + 3
            else:                                              # k = 0, and k = -nx/2 (the Nyquist row when nx is even)
                rows = (np.arange(nx) == nx // 2) | (np.arange(nx) == 0)
            m[~rows] = 0.0
            m = m.astype(np.float32).astype(np.float64)
            ref = O.fk_filter_filt(x32.astype(np.float64), m)
            y, tail = _run(exe, tmpdir_mod, nx, ns, 2, False, x32, 0.0, 0.0, (0.0,) * 4, dense=m, env=env)
            assert tail[0] == np.count_nonzero(O.fold_rowmax(m)), (nx, ns, env, support)
            assert rel_err(y, ref)[0] <= 5e-6, (nx, ns, env, support)


def test_peak_picker_emulation(tmpdir_mod):
    """The device peak picker's per-sample body (flat tops, hierarchical prominence walk over 64-sample blocks and
    64-block superblocks) on the host against scipy.signal.find_peaks, index for index, on the same float32 rows."""
    exe = _build("peaks_emul", tmpdir_mod)
    rng = np.random.default_rng(17)
    for ns in (2, 3, 5, 64, 65, 130, 4097, 9000):
        rows = [rng.standard_normal(ns), np.abs(np.sin(np.arange(ns) * 0.01)) * (1 + 0.05 * rng.standard_normal(ns)),
                np.round(rng.standard_normal(ns) * 2) / 2, np.full(ns, 1.5), np.arange(ns, dtype=np.float64),
                -np.arange(ns, dtype=np.float64), np.concatenate([np.zeros(ns // 2), np.ones(ns - ns // 2)]),
                np.where(np.arange(ns) % 7 == 3, 2.0, np.round(rng.standard_normal(ns)))]
        x = np.stack(rows).astype(np.float32)
        for thr in (0.0, 0.3, 1.0, 2.5):
            fin, fout = os.path.join(tmpdir_mod, "pk.in"), os.path.join(tmpdir_mod, "pk.out")
            with open(fin, "wb") as f:
                f.write(struct.pack("<iid", x.shape[0], ns, thr))
                f.write(x.tobytes())
            subprocess.run([exe, fin, fout], check=True)
            flags = np.frombuffer(open(fout, "rb").read(), dtype=np.uint8).reshape(x.shape)
            for r in range(x.shape[0]):
                ref = sps.find_peaks(x[r].astype(np.float64), prominence=thr)[0]
                assert np.array_equal(np.nonzero(flags[r])[0], ref), (ns, thr, r)
