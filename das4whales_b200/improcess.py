"""das4whales_b200.improcess -- the image-domain ("Gabor") detector of DAS4Whales on the GPU.

Drop-in for the functions of `das4whales.improcess` that scripts/main_gabordetect.py calls
(/root/reference/src/das4whales/improcess.py): scale_pixels (:23-41), trace2image (:44-63), angle_fromspeed (:66-95),
gabor_filt_design (:98-140), binning (:395-421), apply_smooth_mask (:424-454); plus `filter2D`, the GPU stand-in for the
`cv2.filter2D(img, cv2.CV_64F, kernel)` calls the script makes (:109, :135), and `gabor_detect`, which chains the whole
script section :78-169 on the device.  The reference's other image operators follow at the end: compute_radon_transform
(:347), bilateral_filter (:319), gaussian_filter (:370), detect_diagonal_edges (:172), diagonal_edge_detection (:229) and
gradient_oriented (:143) (csrc/imageops_kernels.cuh and filter2D).  Everything numeric runs in libd4w.so
(csrc/image_kernels.cuh); OpenCV / torchvision / skimage are not used.

ndarray in -> float64 ndarray out (like the reference); CUDA tensor in -> float32 CUDA tensor out.
"""
import numpy as np

from . import _lib
from . import rows as _rows
from .dsp import _is_tensor, _to_device, _to_host64


def _torch():
    return _rows._torch()


def _dev2d(a):
    """ndarray / tensor (any real or bool dtype) -> contiguous float32 CUDA tensor [h, w]"""
    torch = _torch()
    if _is_tensor(a):
        t = a if a.is_cuda else a.cuda()
        return t.to(torch.float32).contiguous()
    arr = np.asarray(a)
    if arr.dtype == np.bool_:
        arr = arr.astype(np.float32)
    return _to_device(arr)


def scale_pixels(img):
    """(img - min) / (max - min)  (reference: improcess.py:23-41)"""
    return _scale(img, 1.0)


def _scale(img, mul):
    torch = _torch()
    x = _dev2d(img)
    y = torch.empty_like(x)
    ws = torch.empty(2, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_scale_pixels(_lib.ptr(x, "float*"), _lib.ptr(y, "float*"), x.numel(), float(mul), _lib.ptr(ws),
                                               _lib.stream_ptr()), "scale_pixels")
    return y if _is_tensor(img) else _to_host64(y)


def trace2image(trace):
    """|hilbert(trace)| / std_row(trace), min-max scaled to 0..255 (reference: improcess.py:44-63).  The envelope, the
    division by the row sigma and the scaling all run on the GPU (d4w_hilbert mode 3, d4w_scale_pixels)."""
    torch = _torch()
    x = _to_device(trace)
    env = _rows.envelope_over_std(x)
    ws = torch.empty(2, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_scale_pixels(_lib.ptr(env, "float*"), _lib.ptr(env, "float*"), env.numel(), 255.0, _lib.ptr(ws),
                                               _lib.stream_ptr()), "trace2image")
    return env if _is_tensor(trace) else _to_host64(env)


def angle_fromspeed(c0, fs, dx, selected_channels):
    """Angle (degrees) between sound-speed lines and the time axis of the t-x image (reference: improcess.py:66-95)."""
    ratio = c0 / (fs * dx * selected_channels[2])
    print('Detection speed ratio: ', ratio)
    theta_c0 = np.arctan(ratio) * 180 / np.pi
    print('Angle: ', theta_c0)
    return theta_c0


def _gabor_kernel(ksize, sigma, theta, lambd, gamma, psi):
    """cv2.getGaborKernel((ksize, ksize), sigma, theta, lambd, gamma, psi, CV_64F) restated (OpenCV imgproc/src/gabor.cpp):
    half-width xmax = ksize // 2, so the kernel is (2 * (ksize // 2) + 1) square -- 101 x 101 for ksize = 100 -- and
    kernel[ymax - y, xmax - x] = exp(-(xr^2 / 2 sx^2 + yr^2 / 2 sy^2)) * cos(2 pi xr / lambd + psi)."""
    sigma_x, sigma_y = sigma, sigma / gamma
    xmax = ymax = ksize // 2
    c, s = np.cos(theta), np.sin(theta)
    y, x = np.mgrid[-ymax:ymax + 1, -xmax:xmax + 1].astype(np.float64)
    xr = x * c + y * s
    yr = -x * s + y * c
    v = np.exp(-0.5 / sigma_x ** 2 * xr * xr - 0.5 / sigma_y ** 2 * yr * yr) * np.cos(2 * np.pi / lambd * xr + psi)
    return np.ascontiguousarray(v[::-1, ::-1])


def gabor_filt_design(theta_c0, plot=False):
    """Pair of oriented 101 x 101 Gabor kernels for lines along the sound speed (reference: improcess.py:98-140).
    Host side (10 201 values each)."""
    ksize, sigma, lambd, gamma = 100, 4, 20, 0.15
    theta = np.pi / 2 + np.deg2rad(theta_c0)
    gabor_filtup = _gabor_kernel(ksize, sigma, theta, lambd, gamma, 0.0)
    gabor_filtdown = np.flipud(gabor_filtup)
    if plot:
        import matplotlib.pyplot as plt
        plt.figure(figsize=(6, 4))
        for i, g in enumerate((gabor_filtup, gabor_filtdown)):
            plt.subplot(121 + i)
            plt.imshow(g, origin='lower', cmap='RdBu_r', vmin=-1, vmax=1, aspect='equal')
            plt.xlabel('Time indices')
            plt.colorbar(orientation='horizontal')
        plt.tight_layout()
        plt.show()
    return gabor_filtup, gabor_filtdown


def _resize(x, oh, ow):
    torch = _torch()
    ih, iw = x.shape
    out = torch.empty((oh, ow), dtype=torch.float32, device=x.device)
    tmp = torch.empty((ih, ow), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_resize_aa(_lib.ptr(x, "float*"), ih, iw, _lib.ptr(out, "float*"), oh, ow, _lib.ptr(tmp, "float*"),
                                            _lib.stream_ptr()), "binning")
    return out


def binning(image, ft, fx):
    """Resize an image by ft along time (axis 1) and fx along distance (axis 0) -- torchvision
    `Resize((int(H * fx), int(W * ft)))`, i.e. bilinear interpolation with antialiasing (reference: improcess.py:395-421).
    A boolean image comes back boolean (torchvision resizes it in float32 and casts back: any contributing pixel set)."""
    is_bool = (image.dtype == np.bool_) if isinstance(image, np.ndarray) else (_is_tensor(image) and str(image.dtype) == "torch.bool")
    x = _dev2d(image)
    oh, ow = int(x.shape[0] * fx), int(x.shape[1] * ft)
    y = _resize(x, oh, ow)
    if is_bool:
        y = y != 0
        return y if _is_tensor(image) else y.cpu().numpy()
    return y if _is_tensor(image) else _to_host64(y)


def filter2D(src, ddepth, kernel, in_threshold=None, out_threshold=None, border="reflect101"):
    """GPU stand-in for `cv2.filter2D(src, cv2.CV_64F, kernel)` as scripts/main_gabordetect.py:109,135 call it:
    correlation (no kernel flip), anchor at the kernel centre, BORDER_REFLECT_101.  `ddepth` is accepted and ignored
    (ndarray in -> float64 out, tensor in -> float32 out).  in_threshold / out_threshold binarise the source / the result
    on the fly (`src > thr`), which lets the script's two threshold steps run inside the same kernel."""
    torch = _torch()
    x = _dev2d(src)
    K = torch.from_numpy(np.ascontiguousarray(kernel, dtype=np.float32)).to(x.device)
    if K.ndim != 2 or x.ndim != 2:
        raise ValueError("filter2D expects a 2-D image and a 2-D kernel")
    out = torch.empty_like(x)
    nan = float("nan")
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_filter2d(_lib.ptr(x, "float*"), x.shape[0], x.shape[1], _lib.ptr(K, "float*"), K.shape[0], K.shape[1],
                                           nan if in_threshold is None else float(in_threshold),
                                           nan if out_threshold is None else float(out_threshold),
                                           0 if border == "reflect101" else 1, _lib.ptr(out, "float*"), _lib.stream_ptr()), "filter2D")
    if _is_tensor(src):
        return out
    return _to_host64(out)


def apply_smooth_mask(array, mask, sigma=1.5):
    """array * mask (reference: improcess.py:424-454 -- the Gaussian-smoothed mask is computed there but the product uses
    the raw mask, :452).  When `mask` is smaller than `array` by an integer factor it is first resized to the array's
    shape like `binning(mask, f, f)` does, fused with the product (d4w_mask_upsample_mul)."""
    torch = _torch()
    x = _to_device(array)
    m = _dev2d(mask)
    nx, ns = x.shape
    out = torch.empty_like(x)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_mask_upsample_mul(_lib.ptr(x, "float*"), nx, ns, _lib.ptr(m, "float*"), m.shape[0], m.shape[1],
                                                    _lib.ptr(out, "float*"), _lib.ffi.NULL, _lib.stream_ptr()), "apply_smooth_mask")
    return out if _is_tensor(array) else _to_host64(out)


def gabor_detect(trf_fk, fs, dx, selected_channels, c0=1500., bin_factor=10, threshold=9100., threshold2=150.,
                 return_all=False):
    """The image-domain detector of scripts/main_gabordetect.py:78-169 on the device, end to end:
    trace2image -> binning(1/bin_factor) -> filter2D(up) + filter2D(down) -> > threshold -> filter2D pair on the binary image
    -> > threshold2 -> binning(mask, bin_factor) -> trace * mask.  Both Gabor correlations of a step are one pass with the
    kernel up + down (filter2D is linear in the kernel).  Returns the masked trace (and, with return_all, the intermediate
    images as a dict)."""
    torch = _torch()
    x = _to_device(trf_fk)
    nx, ns = x.shape
    image = trace2image(x)
    imagebin = binning(image, 1 / bin_factor, 1 / bin_factor)
    theta_c0 = np.arctan(c0 / (fs * dx * selected_channels[2])) * 180 / np.pi
    up, down = gabor_filt_design(theta_c0)
    kpair = up + down
    fimage = filter2D(imagebin, None, kpair)
    mask = filter2D(fimage, None, kpair, in_threshold=threshold, out_threshold=threshold2)      # float 0 / 1
    out = torch.empty_like(x)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_mask_upsample_mul(_lib.ptr(x, "float*"), nx, ns, _lib.ptr(mask, "float*"), mask.shape[0], mask.shape[1],
                                                    _lib.ptr(out, "float*"), _lib.ffi.NULL, _lib.stream_ptr()), "gabor mask")
    res = out if _is_tensor(trf_fk) else _to_host64(out)
    if not return_all:
        return res
    conv = (lambda t: t) if _is_tensor(trf_fk) else (lambda t: t.to(torch.float64).cpu().numpy())
    return res, {"image": conv(image), "imagebin": conv(imagebin), "fimage": conv(fimage), "mask": conv(mask) != 0}


# ------------------------------------------------------------------------------ the operators outside the Gabor path
# improcess.py:143-169, :172-266, :319-392 of the reference.  Arguments are checked on the host before any device work.
def _dtype_name(img):
    """numpy-style name of an ndarray's or a tensor's dtype ('uint8', 'float32', ...)"""
    return str(img.dtype).split(".")[-1] if _is_tensor(img) else np.asarray(img).dtype.name


def _check_image(img, what):
    """(image as ndarray or tensor, dtype name) of a non-empty 2-D real image; ValueError otherwise"""
    if not _is_tensor(img):
        img = np.asarray(img)
    name = _dtype_name(img)
    if img.ndim != 2 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError(f"{what}: expected a non-empty 2-D image, got shape {tuple(img.shape)}")
    if name not in ("bool", "uint8", "uint16", "int8", "int16", "int32", "int64", "float16", "float32", "float64"):
        raise ValueError(f"{what}: unsupported dtype {name}")
    return img, name


def _as_int(v, what):
    try:
        i = int(v)
    except (TypeError, ValueError):
        raise ValueError(f"{what} must be an integer") from None
    if i != v:
        raise ValueError(f"{what} must be an integer")
    return i


def _as_real(v, what):
    try:
        f = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"{what} must be a real number") from None
    if not np.isfinite(f):
        raise ValueError(f"{what} must be finite")
    return f


def _out(y, like):
    return y if _is_tensor(like) else _to_host64(y)


# skimage's img_as_float: the integer scale of each accepted dtype
_RADON_SCALE = {"bool": 1.0, "uint8": 255.0, "uint16": 65535.0, "float16": 1.0, "float32": 1.0, "float64": 1.0}


def _radon_square(h, w):
    """(n, pad_rows, pad_cols): skimage's radon(circle=False) zero-pads an h x w image to an n x n square,
    n = ceil(sqrt(2) max(h, w)), with (s + p) // 2 - s // 2 of the p = n - s padding rows / columns before the image."""
    diagonal = np.sqrt(2) * max(h, w)
    pad = [int(np.ceil(diagonal - s)) for s in (h, w)]
    before = [(s + p) // 2 - s // 2 for s, p in zip((h, w), pad)]
    return h + pad[0], before[0], before[1]


def compute_radon_transform(image, theta=None):
    """skimage.transform.radon(image, theta, circle=False) (reference: improcess.py:347-367): the sum of every column of
    the padded image rotated by each angle (degrees, default 0..179), bilinear, zero outside.  Returns [n, len(theta)],
    n = ceil(sqrt(2) max(h, w)).  uint8 / uint16 / bool images are scaled as skimage.img_as_float scales them; other integer
    dtypes raise ValueError.  Ray sums run in double on the GPU (d4w_radon), so the result does not depend on the launch."""
    image, name = _check_image(image, "compute_radon_transform")
    if name not in _RADON_SCALE:
        raise ValueError(f"compute_radon_transform: unsupported dtype {name} (skimage.img_as_float takes floats, uint8, uint16, bool)")
    th = np.arange(180) if theta is None else theta
    try:
        th = np.asarray(th.cpu() if _is_tensor(th) else th, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError("compute_radon_transform: theta must be a 1-D array of angles in degrees") from None
    if th.ndim != 1 or th.size < 1 or not np.all(np.isfinite(th)):
        raise ValueError("compute_radon_transform: theta must be a 1-D array of at least one finite angle")
    h, w = image.shape
    n, pad_r, pad_c = _radon_square(h, w)
    angles = np.deg2rad(th)
    cs = np.ascontiguousarray(np.stack([np.cos(angles), np.sin(angles)], axis=1))
    torch = _torch()
    x = _dev2d(image)
    dcs = torch.from_numpy(cs).to(x.device)
    out = torch.empty((n, th.size), dtype=torch.float64, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_radon(_lib.ptr(x, "float*"), h, w, n, pad_r, pad_c, _lib.ptr(dcs, "double*"), th.size,
                                        _lib.ptr(out, "double*"), _lib.stream_ptr()), "compute_radon_transform")
    if _RADON_SCALE[name] != 1.0:
        out /= _RADON_SCALE[name]          # the transform is linear: scaling the sums is img_as_float's scaling, exactly
    return out.to(torch.float32) if _is_tensor(image) else out.cpu().numpy()


def bilateral_filter(img, diameter, sigma_color, sigma_space):
    """cv2.bilateralFilter(img, diameter, sigma_color, sigma_space) of a single-channel uint8 or float32 image (reference:
    improcess.py:319-344; cv2 rejects other depths, so they raise ValueError here).  OpenCV's rules, as cv2 4.13 applies
    them: either sigma <= 0 returns the image unchanged, for both depths; the radius is round(1.5 sigma_space) for
    diameter <= 0, diameter // 2 otherwise, at least 1 (here at most 64); the taps are those within the radius, border
    reflect-101; uint8 weighs colours by an exact table and rounds the result, float32 by a 4 096-bin table over the image's
    range (colour weight 1 throughout for a constant image).  The result holds the uint8 values for a uint8 image (float64 /
    float32 out, as the rest of the module)."""
    img, name = _check_image(img, "bilateral_filter")
    if name not in ("uint8", "float32"):
        raise ValueError(f"bilateral_filter: OpenCV filters uint8 and float32 images only, got {name}")
    d = _as_int(diameter, "bilateral_filter: diameter")
    sc = _as_real(sigma_color, "bilateral_filter: sigma_color")
    ss = _as_real(sigma_space, "bilateral_filter: sigma_space")
    copy = sc <= 0 or ss <= 0                              # cv2 returns the image unchanged then
    radius = 1 if copy else max(int(np.rint(ss * 1.5)) if d <= 0 else d // 2, 1)
    if radius > 64:
        raise ValueError(f"bilateral_filter: radius {radius} > 64 is not supported")
    torch = _torch()
    x = _dev2d(img)
    if copy:
        return _out(x.clone(), img)
    h, w = x.shape
    out = torch.empty_like(x)
    ws = torch.empty(_lib.lib().D4W_BILATERAL_WS_BYTES, dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_bilateral(_lib.ptr(x, "float*"), h, w, int(name == "uint8"), radius, sc, ss, _lib.ptr(ws),
                                            _lib.ptr(out, "float*"), _lib.stream_ptr()), "bilateral_filter")
    return _out(out, img)


# OpenCV's getGaussianKernel uses fixed tables for sigma <= 0 and these sizes (checked against cv2 4.13, which also has 9)
_GAUSS_TABLES = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
                 7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125],
                 9: [4 / 256, 13 / 256, 30 / 256, 51 / 256, 60 / 256, 51 / 256, 30 / 256, 13 / 256, 4 / 256]}


def _gaussian_kernel(size, sigma):
    """cv2.getGaussianKernel(size, sigma) restated: a fixed table for sigma <= 0 and size <= 9, otherwise
    exp(-x^2 / (2 s^2)) normalised to sum 1 over x = i - (size - 1) / 2, s = sigma, or ((size - 1) / 2 - 1) 0.3 + 0.8 for
    sigma <= 0."""
    if sigma <= 0 and size in _GAUSS_TABLES:
        return np.array(_GAUSS_TABLES[size])
    s = sigma if sigma > 0 else ((size - 1) * 0.5 - 1) * 0.3 + 0.8
    x = np.arange(size) - (size - 1) * 0.5
    t = np.exp(-0.5 / (s * s) * x * x)
    return t / t.sum()


def gaussian_filter(img, size, sigma):
    """cv2.GaussianBlur(img, (size, size), sigma) (reference: improcess.py:370-392): one filter2D pass (reflect-101) with
    the outer product of _gaussian_kernel(size, sigma).  `size` must be odd and positive.  An integer image is filtered as
    its values; the result is not rounded back to the input depth."""
    img, _ = _check_image(img, "gaussian_filter")
    size = _as_int(size, "gaussian_filter: size")
    if size < 1 or size % 2 == 0:
        raise ValueError("gaussian_filter: size must be odd and positive")
    g = _gaussian_kernel(size, _as_real(sigma, "gaussian_filter: sigma"))
    return filter2D(img, None, np.outer(g, g))


_DIAG5 = np.array([[0, 1, 1, 1, 1], [-1, 0, 1, 1, 1], [-1, -1, 0, 1, 1], [-1, -1, -1, 0, 1], [-1, -1, -1, -1, 0]], np.float64)
_DIAG3 = np.array([[2, -1, -1], [-1, 2, -1], [-1, -1, 2]], np.float64)


def detect_diagonal_edges(matrix, threshold):
    """fftconvolve(matrix, K, 'same') + fftconvolve(matrix, fliplr(K), 'same') with the reference's 5 x 5 diagonal kernel K
    (reference: improcess.py:172-226; `threshold` is unused there too).  A convolution is a correlation with the kernel
    turned by 180 degrees, so this is one zero-border filter2D pass with rot180(K) + rot180(fliplr(K))."""
    matrix, _ = _check_image(matrix, "detect_diagonal_edges")
    return filter2D(matrix, None, _DIAG5[::-1, ::-1] + _DIAG5[::-1, :], border="zeros")


def diagonal_edge_detection(img, threshold):
    """conv2d(img, W, padding=1) + conv2d(img, flip(W, 0), padding=1) with the reference's 3 x 3 kernel W (reference:
    improcess.py:229-266): one zero-border filter2D pass with W + flip(W, 0).  Returns what the reference returns, a
    float32 torch tensor: on the CPU for an ndarray, on the input's device for a tensor."""
    img, _ = _check_image(img, "diagonal_edge_detection")
    y = filter2D(_dev2d(img), None, _DIAG3 + _DIAG3[::-1, :], border="zeros")
    return y.to(img.device) if _is_tensor(img) else y.cpu()


def gradient_oriented(image, direction):
    """The reference's oriented difference (improcess.py:143-169) for shifts dft, dfx >= 0:
    dfx = 0: -(x[:, :-dft] - x[:, dft:]); dft = 0: -(x[dfx:, :] - x[:-dfx, :]);
    otherwise -(x[dfx:-dfx, :-dft] - 0.5 x[2 dfx:, dft:] - 0.5 x[:-2 dfx, dft:]).  (0, 0) raises ValueError, as the
    reference's broadcast fails.  An integer image is taken as its values (no unsigned wrap-around)."""
    image, _ = _check_image(image, "gradient_oriented")
    try:
        dft, dfx = direction
    except (TypeError, ValueError):
        raise ValueError("gradient_oriented: direction must be a pair (dft, dfx)") from None
    dft, dfx = _as_int(dft, "gradient_oriented: dft"), _as_int(dfx, "gradient_oriented: dfx")
    if dft < 0 or dfx < 0:
        raise ValueError("gradient_oriented: dft and dfx must be >= 0")
    if dft == 0 and dfx == 0:
        raise ValueError("gradient_oriented: direction (0, 0) has no gradient (the reference's shapes do not broadcast)")
    h, w = image.shape
    oh = max(0, h if dfx == 0 else h - dfx if dft == 0 else h - 2 * dfx)
    ow = max(0, w - dft)
    torch = _torch()
    x = _dev2d(image)
    out = torch.empty((oh, ow), dtype=torch.float32, device=x.device)
    if oh and ow:
        with torch.cuda.device(x.device.index):
            _lib.check(_lib.lib().d4w_grad_oriented(_lib.ptr(x, "float*"), h, w, dft, dfx, _lib.ptr(out, "float*"),
                                                    _lib.stream_ptr()), "gradient_oriented")
    return out if _is_tensor(image) else out.to(torch.float64).cpu().numpy()
