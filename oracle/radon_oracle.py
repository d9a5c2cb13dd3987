"""oracle/radon_oracle.py -- skimage.transform.radon(image, theta, circle=False) restated in float64 NumPy.

The reference's compute_radon_transform (das4whales/improcess.py:347-367) is this one skimage call.  skimage is not
installed where the fixtures are made, so this restatement is written from skimage's published algorithm
(skimage/transform/radon_transform.py, and the order-1 constant-mode bilinear sampling of skimage/transform/_warps_cy.pyx
and _shared/interpolation.pxd) and cannot be compared with skimage itself.  tests/test_imageops_host.py pins it instead
by invariants that need no skimage: at 0 degrees it is the padded image's column sums, at 90 degrees its row sums, a
single pixel gives the bilinear weights along the analytic sinusoid, a zero image gives zeros, and every projection of
an image well inside the circle keeps the image's total mass.

    img_as_float:  uint8 / 255, uint16 / 65535, bool -> 0 / 1, floats as they are
    padding:       n = s + ceil(sqrt(2) max(h, w) - s) on both axes (a square), (s + p) // 2 - s // 2 of the p pads before
    angle a:       inverse map [[cos, sin, -c (cos + sin - 1)], [-sin, cos, -c (cos - sin - 1)]] of (col, row), c = n // 2
    sampling:      bilinear between floor and ceil of each coordinate, zero outside the padded image, no clipping
    output:        [n, len(theta)], column a = the column sums of the warped image
"""
import numpy as np

_SCALE = {np.dtype(np.uint8): 255.0, np.dtype(np.uint16): 65535.0, np.dtype(np.bool_): 1.0}


def img_as_float(image):
    image = np.asarray(image)
    if image.dtype in _SCALE:
        return image.astype(np.float64) / _SCALE[image.dtype]
    if image.dtype.kind != "f":
        raise ValueError(f"unsupported dtype {image.dtype}")
    return image.astype(np.float64)


def pad_square(image):
    """the zero-padded square of radon(circle=False), and the padding before each axis"""
    diagonal = np.sqrt(2) * max(image.shape)
    pad = [int(np.ceil(diagonal - s)) for s in image.shape]
    before = [(s + p) // 2 - s // 2 for s, p in zip(image.shape, pad)]
    padded = np.pad(image, [(b, p - b) for b, p in zip(before, pad)], mode="constant", constant_values=0)
    assert padded.shape[0] == padded.shape[1]
    return padded, before


def bilinear(img, y, x):
    """order-1 sampling of img at (y, x) with zeros outside (skimage's bilinear_interpolation, mode 'constant')"""
    rows, cols = img.shape
    minr, minc = np.floor(y), np.floor(x)
    maxr, maxc = np.ceil(y), np.ceil(x)
    dr, dc = y - minr, x - minc

    def px(r, c):
        ok = (r >= 0) & (r < rows) & (c >= 0) & (c < cols)
        return np.where(ok, img[np.clip(r, 0, rows - 1).astype(np.int64), np.clip(c, 0, cols - 1).astype(np.int64)], 0.0)

    top = (1 - dc) * px(minr, minc) + dc * px(minr, maxc)
    bottom = (1 - dc) * px(maxr, minc) + dc * px(maxr, maxc)
    return (1 - dr) * top + dr * bottom


def radon(image, theta=None):
    """skimage.transform.radon(image, theta, circle=False), float64"""
    if theta is None:
        theta = np.arange(180)
    padded, _ = pad_square(img_as_float(image))
    n = padded.shape[0]
    center = n // 2
    row, col = np.mgrid[0:n, 0:n].astype(np.float64)
    out = np.zeros((n, len(theta)))
    for i, angle in enumerate(np.deg2rad(np.asarray(theta, dtype=np.float64))):
        cos_a, sin_a = np.cos(angle), np.sin(angle)
        x = cos_a * col + sin_a * row + -center * (cos_a + sin_a - 1)
        y = -sin_a * col + cos_a * row + -center * (cos_a - sin_a - 1)
        out[:, i] = bilinear(padded, y, x).sum(0)
    return out


def radon_bins(image, bins, angles):
    """R[bins[k], k] for degree angles[k]: sampled entries of radon(image, theta) at any size, one ray at a time"""
    diagonal = np.sqrt(2) * max(image.shape)
    pad = [int(np.ceil(diagonal - s)) for s in image.shape]
    before = [(s + p) // 2 - s // 2 for s, p in zip(image.shape, pad)]
    n = image.shape[0] + pad[0]
    img = img_as_float(image)
    center = n // 2
    r = np.arange(n, dtype=np.float64)
    out = np.empty(len(bins))
    for k, (b, a) in enumerate(zip(bins, np.deg2rad(np.asarray(angles, dtype=np.float64)))):
        cos_a, sin_a = np.cos(a), np.sin(a)
        x = cos_a * b + sin_a * r + -center * (cos_a + sin_a - 1) - before[1]
        y = -sin_a * b + cos_a * r + -center * (cos_a - sin_a - 1) - before[0]
        out[k] = bilinear(img, y, x).sum()
    return out
