"""GPU: the image operators of improcess outside the Gabor path against the fixture of the reference
(tests/golden/imageops.npz, oracle/imageops_golden.py) and the float64 Radon restatement (oracle/radon_oracle.py).

Bounds: Radon within 1e-5 of max|R| (float32 pixels and weights, double coordinates and sums: the measured error is
~3e-8); bilateral within one count for uint8 and 1e-5 of the image range for float32; the filter2D operators and
gradient_oriented within 1e-5 relative (float32 arithmetic against the reference's float64)."""
import numpy as np
import pytest

from das4whales_b200 import improcess
from oracle import radon_oracle as R

pytestmark = pytest.mark.gpu
TOL = 1e-5


def relmax(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


# ------------------------------------------------------------------------------ Radon
def test_radon_fixture(golden):
    g = golden("imageops")
    img = g["radon_img"]
    out = improcess.compute_radon_transform(img)
    assert out.dtype == np.float64 and out.shape == (44, 180)
    assert relmax(out, g["radon_default"]) <= TOL
    assert relmax(improcess.compute_radon_transform(img, g["radon_theta"]), g["radon_theta_out"]) <= TOL
    assert relmax(improcess.compute_radon_transform(g["u8"][:20, :17], g["radon_theta"]), g["radon_u8"]) <= TOL


@pytest.mark.parametrize("shape", [(37, 52), (64, 9), (5, 71), (1, 1)])
@pytest.mark.parametrize("nth", [1, 360])
def test_radon_shapes_and_angles(shape, nth):
    rng = np.random.default_rng(shape[0] * 100 + nth)
    img = rng.random(shape)
    theta = np.array([33.3]) if nth == 1 else np.linspace(-180, 180, 360, endpoint=False)
    want = R.radon(img, theta)
    out = improcess.compute_radon_transform(img, theta)
    assert relmax(out, want) <= TOL
    import torch
    t = improcess.compute_radon_transform(torch.from_numpy(img).cuda(), theta)
    assert t.is_cuda and t.dtype == torch.float32
    assert relmax(t.cpu().numpy(), want) <= TOL


def test_radon_integer_and_bool_inputs():
    import torch
    rng = np.random.default_rng(4)
    theta = [0.0, 30.0, 91.0]
    for img in (rng.integers(0, 256, (19, 26)).astype(np.uint8), rng.integers(0, 65536, (19, 26)).astype(np.uint16),
                rng.random((19, 26)) > 0.5):
        want = R.radon(img, theta)
        assert relmax(improcess.compute_radon_transform(img, theta), want) <= TOL
    u8 = rng.integers(0, 256, (19, 26)).astype(np.uint8)
    t = improcess.compute_radon_transform(torch.from_numpy(u8).cuda(), theta)
    assert relmax(t.cpu().numpy(), R.radon(u8, theta)) <= TOL


def test_radon_reruns_are_bit_identical():
    import torch
    img = torch.rand((301, 407), device="cuda")
    a = improcess.compute_radon_transform(img, np.arange(0, 180, 0.5))
    b = improcess.compute_radon_transform(img, np.arange(0, 180, 0.5))
    assert torch.equal(a, b)


def test_radon_full_size_trace2image():
    import torch
    g = torch.Generator(device="cuda").manual_seed(3)
    trace = torch.randn((11020, 12000), generator=g, device="cuda", dtype=torch.float32)
    image = improcess.trace2image(trace)
    out = improcess.compute_radon_transform(image)
    assert out.shape == (16971, 180) and out.is_cuda
    rng = np.random.default_rng(2)
    bins, angles = rng.integers(2000, 15000, 48), rng.integers(0, 180, 48)
    want = R.radon_bins(image.cpu().numpy(), bins, angles)
    got = out[torch.from_numpy(bins).cuda(), torch.from_numpy(angles).cuda()].double().cpu().numpy()
    assert np.max(np.abs(got - want)) <= TOL * out.abs().max().item()


# ------------------------------------------------------------------------------ bilateral
def test_bilateral_fixture(golden):
    import torch
    g = golden("imageops")
    u8, f32 = g["u8"], g["f32"]
    rng = float(f32.max() - f32.min())
    for k, (d, sc, ss) in enumerate(g["bilateral_cases"]):
        out = improcess.bilateral_filter(u8, int(d), sc, ss)
        assert out.dtype == np.float64 and np.max(np.abs(out - g[f"bil_u8_{k}"])) <= 1, (d, sc, ss)
        out = improcess.bilateral_filter(f32, int(d), sc, ss)
        assert np.max(np.abs(out - g[f"bil_f32_{k}"])) <= TOL * rng, (d, sc, ss)
        t = improcess.bilateral_filter(torch.from_numpy(f32).cuda(), int(d), sc, ss)
        assert t.is_cuda and np.max(np.abs(t.cpu().numpy() - g[f"bil_f32_{k}"])) <= TOL * rng
        if sc <= 0 or ss <= 0:                  # cv2 returns the input itself
            assert np.array_equal(improcess.bilateral_filter(u8, int(d), sc, ss), g[f"bil_u8_{k}"])
            assert np.array_equal(improcess.bilateral_filter(f32, int(d), sc, ss), g[f"bil_f32_{k}"])
            assert np.array_equal(t.cpu().numpy(), f32)
    out = improcess.bilateral_filter(g["const"], 9, 30.0, 30.0)
    assert np.max(np.abs(out - g["bil_const"])) <= TOL * 0.375


def test_bilateral_large_image_against_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(8)
    u8 = rng.integers(0, 256, (333, 517)).astype(np.uint8)
    f32 = rng.random((333, 517)).astype(np.float32) * 40 - 7
    for d, sc, ss in [(5, 30.0, 30.0), (9, 75.0, 75.0), (0, 20.0, 4.0), (9, 75.0, 0.0), (5, 0.0, 30.0)]:
        assert np.max(np.abs(improcess.bilateral_filter(u8, d, sc, ss) - cv2.bilateralFilter(u8, d, sc, ss))) <= 1
        assert np.max(np.abs(improcess.bilateral_filter(f32, d, sc, ss) - cv2.bilateralFilter(f32, d, sc, ss))) <= TOL * 40


# ------------------------------------------------------------------------------ filter2D operators and the gradient
def test_gaussian_fixture(golden):
    g = golden("imageops")
    for size in g["gauss_sizes"]:
        for sigma in g["gauss_sigmas"]:
            assert relmax(improcess.gaussian_filter(g["f32"], int(size), sigma), g[f"gauss_f32_{size}_{sigma}"]) <= TOL
        assert relmax(improcess.gaussian_filter(g["f64"], int(size), 1.5), g[f"gauss_f64_{size}"]) <= TOL


def test_diagonal_operators_fixture(golden):
    import torch
    g = golden("imageops")
    assert relmax(improcess.detect_diagonal_edges(g["f64"], 0.5), g["diag_edges_f64"]) <= TOL
    assert relmax(improcess.detect_diagonal_edges(g["u8"], 0.5), g["diag_edges_u8"]) <= TOL
    for key in ("f32", "f64"):
        out = improcess.diagonal_edge_detection(g[key], 0.5)
        assert isinstance(out, torch.Tensor) and out.device.type == "cpu" and out.dtype == torch.float32
        assert relmax(out.numpy(), g[f"diag_det_{key}"]) <= TOL
    t = improcess.diagonal_edge_detection(torch.from_numpy(g["f32"]).cuda(), 0.5)
    assert t.is_cuda and relmax(t.cpu().numpy(), g["diag_det_f32"]) <= TOL


def test_gradient_oriented_fixture(golden):
    import torch
    g = golden("imageops")
    for k, (dft, dfx) in enumerate(g["grad_directions"]):
        out = improcess.gradient_oriented(g["f64"], (int(dft), int(dfx)))
        assert out.dtype == np.float64 and relmax(out, g[f"grad_{k}"]) <= TOL
        t = improcess.gradient_oriented(torch.from_numpy(g["f64"]).cuda(), (int(dft), int(dfx)))
        assert t.is_cuda and relmax(t.cpu().numpy(), g[f"grad_{k}"]) <= TOL
    x = g["f64"]
    assert improcess.gradient_oriented(x, (x.shape[1], 0)).shape == x[:, :-x.shape[1]].shape
    assert improcess.gradient_oriented(x, (1, x.shape[0])).shape == (0, x.shape[1] - 1)
