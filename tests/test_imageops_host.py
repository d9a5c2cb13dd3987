"""CPU: the image operators of improcess outside the Gabor path.  The Radon restatement (oracle/radon_oracle.py) against
invariants that need no skimage and against the fixture; the fixture against live cv2 / scipy / torch through the
unmodified reference; the restated OpenCV rules (Gaussian kernel, bilateral filter) against cv2; the k_radon ray body run
on the host (tests/host_emul/radon_emul.cu) against the restatement; and every ValueError before device work."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from das4whales_b200 import improcess
from oracle import imageops_golden as G, radon_oracle as R, ref_loader

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
EMUL = os.path.join(ROOT, "tests", "host_emul")


def relmax(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


# ------------------------------------------------------------------------------ Radon restatement: invariants
def test_radon_zero_degrees_is_column_sums():
    img = np.random.default_rng(1).random((13, 22))
    padded, _ = R.pad_square(img)
    assert np.array_equal(R.radon(img, [0.0])[:, 0], padded.sum(0))


@pytest.mark.parametrize("shape", [(13, 22), (21, 9), (16, 16)])
def test_radon_ninety_degrees_is_row_sums(shape):
    # at 90 degrees bin b samples row 2c - b of the padded square (c = n // 2), so the row sums come out reversed about c
    img = np.random.default_rng(2).random(shape)
    padded, _ = R.pad_square(img)
    n, c = padded.shape[0], padded.shape[0] // 2
    rows = padded.sum(1)
    want = np.array([rows[2 * c - b] if 0 <= 2 * c - b < n else 0.0 for b in range(n)])
    assert np.max(np.abs(R.radon(img, [90.0])[:, 0] - want)) <= 1e-12 * rows.max()


def test_radon_single_pixel_is_the_bilinear_sinusoid():
    img = np.zeros((9, 14))
    img[2, 11] = 1.0
    theta = np.array([0.0, 17.0, 45.0, 90.0, 133.0, 179.5, -40.0])
    out = R.radon(img, theta)
    _, (pr, pc) = R.pad_square(img)
    n = out.shape[0]
    c = n // 2
    py, px = pr + 2, pc + 11
    r = np.arange(n, dtype=np.float64)
    for k, t in enumerate(np.deg2rad(theta)):
        co, si = np.cos(t), np.sin(t)
        for b in range(n):
            x = co * b + si * r - c * (co + si - 1)
            y = -si * b + co * r - c * (co - si - 1)
            want = np.sum(np.maximum(0, 1 - np.abs(x - px)) * np.maximum(0, 1 - np.abs(y - py)))
            assert abs(out[b, k] - want) <= 1e-12
        # the peak sits on the sinusoid of the bin whose ray passes through the pixel
        b_star = co * (px - c) - si * (py - c) + c
        assert abs(np.argmax(out[:, k]) - b_star) <= 1.0


def test_radon_zero_image():
    assert not np.any(R.radon(np.zeros((7, 12)), np.linspace(-90, 270, 17)))


def test_radon_keeps_mass_inside_the_circle():
    # every rotation of a smooth blob well inside the circle keeps its mass, up to the resampling error of bilinear sampling
    y, x = np.mgrid[0:30, 0:30]
    img = np.exp(-((y - 13.2) ** 2 + (x - 15.6) ** 2) / (2 * 3.0 ** 2))
    out = R.radon(img, np.arange(0, 180, 7.5))
    assert np.max(np.abs(out.sum(0) - img.sum())) <= 1e-3 * img.sum()


def test_radon_bins_match_full_transform():
    img = G.radon_image()
    full = R.radon(img, G.RADON_THETA)
    bins = np.arange(full.shape[0])
    for k, t in enumerate(G.RADON_THETA):
        assert np.max(np.abs(R.radon_bins(img, bins, np.full(bins.size, t)) - full[:, k])) <= 1e-12 * np.abs(full).max()


def test_radon_square_matches_the_restatement():
    for shape in [(1, 1), (3, 5), (23, 31), (1102, 1200), (11020, 12000), (40, 7)]:
        n, pr, pc = improcess._radon_square(*shape)
        if max(shape) < 2000:
            padded, before = R.pad_square(np.ones(shape))
            assert padded.shape == (n, n) and before == [pr, pc]
        assert n == int(np.ceil(np.sqrt(2) * max(shape)))
    assert improcess._radon_square(11020, 12000) == (16971, 2975, 2485)


# ------------------------------------------------------------------------------ fixture against the restatements
def test_fixture_radon_is_the_restatement(golden):
    g = golden("imageops")
    img = g["radon_img"]
    assert np.array_equal(g["radon_default"], R.radon(img))
    assert g["radon_default"].shape == (44, 180)
    assert np.array_equal(g["radon_theta_out"], R.radon(img, g["radon_theta"]))
    assert np.array_equal(g["radon_u8"], R.radon(g["u8"][:20, :17], g["radon_theta"]))


def test_fixture_gaussian_is_the_restated_kernel(golden):
    import cv2
    g = golden("imageops")
    for size in g["gauss_sizes"]:
        for sigma in list(g["gauss_sigmas"]) + [-1.0]:
            assert np.max(np.abs(improcess._gaussian_kernel(int(size), sigma) - cv2.getGaussianKernel(int(size), sigma).ravel())) <= 1e-15
    for size in (1, 9, 11):
        assert np.max(np.abs(improcess._gaussian_kernel(size, 0.0) - cv2.getGaussianKernel(size, 0.0).ravel())) <= 1e-15
    f64 = g["f64"]
    for size in g["gauss_sizes"]:
        k = improcess._gaussian_kernel(int(size), 1.5)
        want = cv2.filter2D(f64, cv2.CV_64F, np.outer(k, k), borderType=cv2.BORDER_REFLECT_101)
        assert relmax(g[f"gauss_f64_{size}"], want) <= 1e-12


def test_fixture_bilateral_is_the_restated_rules(golden):
    g = golden("imageops")
    u8, f32 = g["u8"], g["f32"]
    rng = float(f32.max() - f32.min())
    for k, (d, sc, ss) in enumerate(g["bilateral_cases"]):
        assert np.max(np.abs(G.bilateral(u8, int(d), sc, ss).astype(int) - g[f"bil_u8_{k}"])) <= 1
        assert np.max(np.abs(G.bilateral(f32, int(d), sc, ss) - g[f"bil_f32_{k}"])) <= 1e-6 * rng
        if sc <= 0 or ss <= 0:                  # cv2 returns the input itself, whatever the other sigma
            assert np.array_equal(g[f"bil_u8_{k}"], u8) and np.array_equal(g[f"bil_f32_{k}"], f32)
            assert np.array_equal(G.bilateral(u8, int(d), sc, ss), u8) and np.array_equal(G.bilateral(f32, int(d), sc, ss), f32)
    assert sum(1 for _, sc, ss in g["bilateral_cases"] if (sc <= 0) != (ss <= 0)) >= 3
    assert np.max(np.abs(G.bilateral(g["const"], 9, 30.0, 30.0) - g["bil_const"])) <= 1e-6 * 0.375


def test_fixture_diagonal_and_gradient_closed_forms(golden):
    from scipy.signal import correlate
    g = golden("imageops")
    f64 = g["f64"]
    k5 = improcess._DIAG5[::-1, ::-1] + improcess._DIAG5[::-1, :]
    assert relmax(g["diag_edges_f64"], correlate(f64, k5, mode="same", method="direct")) <= 1e-12
    k3 = improcess._DIAG3 + improcess._DIAG3[::-1, :]
    assert relmax(g["diag_det_f64"], correlate(f64.astype(np.float32).astype(np.float64), k3, mode="same", method="direct")) <= 1e-6
    for k, (dft, dfx) in enumerate(g["grad_directions"]):
        assert g[f"grad_{k}"].shape == ((f64.shape[0] if dfx == 0 else f64.shape[0] - dfx if dft == 0 else f64.shape[0] - 2 * dfx),
                                        f64.shape[1] - dft)


@pytest.mark.skipif(not ref_loader.available(), reason="reference not available")
def test_fixture_is_the_live_reference(golden):
    import torch  # noqa: F401  (the reference's diagonal_edge_detection)
    g = golden("imageops")
    imp = G.load_reference()
    u8, f32, f64 = g["u8"], g["f32"], g["f64"]
    for k, (d, sc, ss) in enumerate(g["bilateral_cases"]):
        assert np.array_equal(imp.bilateral_filter(u8, int(d), sc, ss), g[f"bil_u8_{k}"])
        assert np.array_equal(imp.bilateral_filter(f32, int(d), sc, ss), g[f"bil_f32_{k}"])
    for size in g["gauss_sizes"]:
        for sigma in g["gauss_sigmas"]:
            assert np.array_equal(imp.gaussian_filter(f32, int(size), sigma), g[f"gauss_f32_{size}_{sigma}"])
    assert np.array_equal(imp.detect_diagonal_edges(f64, 0), g["diag_edges_f64"])
    assert np.array_equal(imp.diagonal_edge_detection(f32, 0).numpy(), g["diag_det_f32"])
    for k, direction in enumerate(g["grad_directions"]):
        assert np.array_equal(imp.gradient_oriented(f64, tuple(direction)), g[f"grad_{k}"])
    with pytest.raises(ValueError):
        imp.gradient_oriented(f64, (0, 0))
    assert np.array_equal(imp.compute_radon_transform(g["radon_img"], g["radon_theta"]), g["radon_theta_out"])


# ------------------------------------------------------------------------------ host emulation of k_radon
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = os.path.join(str(tmp_path_factory.mktemp("radon")), "radon_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out,
                        os.path.join(EMUL, "radon_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def emulate(exe, tmp, img, theta):
    h, w = img.shape
    n, pr, pc = improcess._radon_square(h, w)
    a = np.deg2rad(np.asarray(theta, np.float64))
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(np.array([h, w, n, pr, pc, len(a)], np.int64).tobytes())
        f.write(np.ascontiguousarray(np.stack([np.cos(a), np.sin(a)], 1)).tobytes())
        f.write(np.ascontiguousarray(img, np.float32).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    return np.fromfile(fout, np.float64).reshape(n, len(a))


@pytest.mark.parametrize("shape", [(13, 20), (21, 9), (1, 1), (1, 17), (30, 30)])
def test_radon_emulation_vs_restatement(exe, tmp_path, shape):
    img = np.random.default_rng(sum(shape)).random(shape).astype(np.float32)
    theta = [0.0, 45.0, 90.0, 179.5, -30.0, -90.25, 13.7, 360.0, -179.0]
    e = emulate(exe, str(tmp_path), img, theta)
    assert relmax(e, R.radon(img.astype(np.float64), theta)) <= 1e-6


# ------------------------------------------------------------------------------ argument checks
def test_value_errors_before_any_device_work():
    img = np.zeros((8, 9), np.float32)
    bad = [
        lambda: improcess.compute_radon_transform(np.zeros((2, 3, 4))),
        lambda: improcess.compute_radon_transform(np.zeros((4, 4), np.int32)),
        lambda: improcess.compute_radon_transform(img, theta=[]),
        lambda: improcess.compute_radon_transform(img, theta=np.zeros((2, 2))),
        lambda: improcess.compute_radon_transform(img, theta=[0.0, np.nan]),
        lambda: improcess.compute_radon_transform(img, theta=["a"]),
        lambda: improcess.bilateral_filter(img.astype(np.float64), 5, 10, 10),
        lambda: improcess.bilateral_filter(img.astype(np.uint16), 5, 10, 10),
        lambda: improcess.bilateral_filter(np.zeros((4, 4, 3), np.uint8), 5, 10, 10),
        lambda: improcess.bilateral_filter(img, 5.5, 10, 10),
        lambda: improcess.bilateral_filter(img, 5, np.inf, 10),
        lambda: improcess.bilateral_filter(img, 131, 10, 10),
        lambda: improcess.bilateral_filter(img, 0, 10, 50),
        lambda: improcess.bilateral_filter(np.zeros((0, 5), np.float32), 5, 10, 10),
        lambda: improcess.compute_radon_transform(np.zeros((4, 0))),
        lambda: improcess.gaussian_filter(np.zeros((0, 0)), 3, 1.0),
        lambda: improcess.gradient_oriented(np.zeros((0, 4)), (1, 0)),
        lambda: improcess.gaussian_filter(img, 4, 1.0),
        lambda: improcess.gaussian_filter(img, 0, 1.0),
        lambda: improcess.gaussian_filter(img, -3, 1.0),
        lambda: improcess.gaussian_filter(img, 3.5, 1.0),
        lambda: improcess.gaussian_filter(img, 3, "x"),
        lambda: improcess.gaussian_filter(np.zeros(5), 3, 1.0),
        lambda: improcess.detect_diagonal_edges(np.zeros((2, 2, 2)), 0),
        lambda: improcess.diagonal_edge_detection(np.zeros(5), 0),
        lambda: improcess.diagonal_edge_detection(np.zeros((3, 3), np.complex64), 0),
        lambda: improcess.gradient_oriented(img, (0, 0)),
        lambda: improcess.gradient_oriented(img, (-1, 2)),
        lambda: improcess.gradient_oriented(img, (1.5, 2)),
        lambda: improcess.gradient_oriented(img, 3),
        lambda: improcess.gradient_oriented(np.zeros(5), (1, 0)),
    ]
    for k, f in enumerate(bad):
        with pytest.raises(ValueError):
            f()


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    img = np.ones((8, 9), np.float32)
    calls = [lambda: improcess.compute_radon_transform(img), lambda: improcess.bilateral_filter(img, 5, 10, 10),
             lambda: improcess.bilateral_filter(img, 5, 0, 10), lambda: improcess.gaussian_filter(img, 3, 0),
             lambda: improcess.detect_diagonal_edges(img, 0), lambda: improcess.diagonal_edge_detection(img, 0),
             lambda: improcess.gradient_oriented(img, (1, 0)), lambda: improcess.gradient_oriented(img, (20, 0))]
    for f in calls:
        with pytest.raises(RuntimeError):
            f()
