"""oracle/imageops_golden.py -- TEST INFRASTRUCTURE for the image operators of improcess outside the Gabor path.

Loads the reference's improcess module *unmodified* (oracle/ref_loader.load_improcess) and runs its
compute_radon_transform, bilateral_filter, gaussian_filter, detect_diagonal_edges, diagonal_edge_detection and
gradient_oriented on seeded images, writing the results to tests/golden/imageops.npz.  Everything but the Radon transform
is a real cv2 / scipy / torch call.  skimage is not installed where the fixtures are made, so skimage.transform.radon is
replaced by the float64 restatement of oracle/radon_oracle.py; the reference wrapper's own argument handling still runs.

`bilateral` restates cv2.bilateralFilter for one channel in NumPy, so the CPU tests can hold each OpenCV rule the GPU
kernel follows against live cv2.

    python -m oracle.imageops_golden [out_dir]      # from the repo root; out_dir defaults to tests/golden
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import radon_oracle, ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
BILATERAL = [(5, 30.0, 30.0), (5, 0.0, -1.0), (9, 75.0, 0.0), (5, 0.0, 30.0), (0, 20.0, -2.0), (9, 75.0, 5.0), (9, 12.0, 2.0), (0, 20.0, 3.0), (0, 50.0, 1.5)]
GAUSS_SIZES, GAUSS_SIGMAS = (3, 5, 7, 31), (0.0, 1.5, 8.0)
GRAD_DIRECTIONS = [(3, 0), (0, 2), (2, 1)]
RADON_THETA = np.array([0.0, 12.5, 45.0, 90.0, 133.3, 179.5, -20.0])


def images(seed=2025, shape=(36, 45)):
    """a smooth field with lines and noise as uint8, float32 and float64"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:shape[0], 0:shape[1]].astype(np.float64)
    f = 110 + 60 * np.sin(x / 7.0) * np.cos(y / 11.0) + 70 * (np.abs(x - 0.8 * y - 10) < 2) + rng.normal(0, 12, shape)
    u8 = np.clip(np.rint(f), 0, 255).astype(np.uint8)
    return u8, (f / 255).astype(np.float32), f / 255


def radon_image(seed=7, shape=(23, 31)):
    rng = np.random.default_rng(seed)
    return rng.random(shape) * (np.arange(shape[1]) % 5 == 0) + 0.25 * rng.random(shape)


def bilateral(img, d, sigma_color, sigma_space):
    """cv2.bilateralFilter(img, d, sigma_color, sigma_space) restated for a 2-D uint8 or float32 image"""
    if sigma_color <= 0 or sigma_space <= 0:
        return img.copy()
    radius = max(int(np.rint(sigma_space * 1.5)) if d <= 0 else d // 2, 1)
    cc, sc = -0.5 / sigma_color ** 2, -0.5 / sigma_space ** 2
    src = img.astype(np.float32)
    if img.dtype == np.float32:
        lo, hi = float(src.min()), float(src.max())
        if abs(lo - hi) < np.finfo(np.float32).eps:
            scale, lut = np.float32(0), np.r_[1, np.zeros(4097)].astype(np.float32)
        else:
            scale = np.float32(4096 / (hi - lo))
            lut = np.exp((np.arange(4098, dtype=np.float32) / scale).astype(np.float64) ** 2 * cc).astype(np.float32)
    else:
        lut = np.exp(np.arange(256, dtype=np.float64) ** 2 * cc).astype(np.float32)
    pad = np.pad(src, radius, mode="reflect")                       # numpy 'reflect' is OpenCV's BORDER_REFLECT_101
    h, w = src.shape
    s, ws = np.zeros_like(src), np.zeros_like(src)
    for i in range(-radius, radius + 1):
        for j in range(-radius, radius + 1):
            r = np.sqrt(float(i * i + j * j))
            if r > radius:
                continue
            v = pad[radius + i:radius + i + h, radius + j:radius + j + w]
            if img.dtype == np.float32:
                alpha = np.abs(v - src) * scale
                k = np.floor(alpha).astype(np.int64)
                alpha = alpha - k.astype(np.float32)
                cw = lut[k] + alpha * (lut[k + 1] - lut[k])
            else:
                cw = lut[np.abs(v - src).astype(np.int64)]
            wt = np.float32(np.exp(r * r * sc)) * cw
            s += v * wt
            ws += wt
    out = s / ws
    return np.clip(np.rint(out), 0, 255).astype(np.uint8) if img.dtype == np.uint8 else out


def load_reference():
    """the reference's improcess module, with skimage.transform.radon -> radon_oracle.radon"""
    imp = ref_loader.load_improcess()

    def radon(image, theta=None, circle=True):
        assert circle is False
        return radon_oracle.radon(image, theta)
    imp.radon = radon
    return imp


def make_imageops(out_dir=OUT):
    imp = load_reference()
    u8, f32, f64 = images()
    out = dict(u8=u8, f32=f32, f64=f64, bilateral_cases=np.array(BILATERAL), gauss_sizes=np.array(GAUSS_SIZES),
               gauss_sigmas=np.array(GAUSS_SIGMAS), grad_directions=np.array(GRAD_DIRECTIONS), radon_theta=RADON_THETA)
    for k, (d, sc, ss) in enumerate(BILATERAL):
        out[f"bil_u8_{k}"] = imp.bilateral_filter(u8, d, sc, ss)
        out[f"bil_f32_{k}"] = imp.bilateral_filter(f32, d, sc, ss)
    const = np.full((20, 27), 0.375, np.float32)
    out["const"] = const
    out["bil_const"] = imp.bilateral_filter(const, 9, 30.0, 30.0)
    for size in GAUSS_SIZES:
        for sigma in GAUSS_SIGMAS:
            out[f"gauss_f32_{size}_{sigma}"] = imp.gaussian_filter(f32, size, sigma)
        out[f"gauss_f64_{size}"] = imp.gaussian_filter(f64, size, 1.5)
    out["diag_edges_f64"] = imp.detect_diagonal_edges(f64, 0.5)
    out["diag_edges_u8"] = imp.detect_diagonal_edges(u8, 0.5)
    out["diag_det_f32"] = imp.diagonal_edge_detection(f32, 0.5).numpy()
    out["diag_det_f64"] = imp.diagonal_edge_detection(f64, 0.5).numpy()
    for k, direction in enumerate(GRAD_DIRECTIONS):
        out[f"grad_{k}"] = imp.gradient_oriented(f64, direction)
    rimg = radon_image()
    out["radon_img"] = rimg
    out["radon_default"] = imp.compute_radon_transform(rimg)
    out["radon_theta_out"] = imp.compute_radon_transform(rimg, RADON_THETA)
    out["radon_u8"] = imp.compute_radon_transform(u8[:20, :17], RADON_THETA)
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "imageops.npz"), **out)


if __name__ == "__main__":
    make_imageops(sys.argv[1] if len(sys.argv) > 1 else OUT)
