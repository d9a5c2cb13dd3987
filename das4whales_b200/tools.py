"""das4whales_b200.tools -- the compute functions of `das4whales.tools` (/root/reference/src/das4whales/tools.py) on the GPU,
without xarray or dask: inputs are [ns] or [nx, ns] ndarrays or CUDA tensors with time on the last axis, and the reference's
map_blocks over dask chunks becomes an explicit chunk size (dask-style uniform blocks, the last one ragged).

`fk_filt` is tools.fk_filt / fk_filt_chunk (tools.py:8-81): per block, linear detrend (d4w_detrend_linear), f-k filter with
the block's own Gaussian-blurred fan designed on the device (d4w_fan_blur, sigma = 40).  `energy_TimeDomain` is
tools.energy_TimeDomain (:84-157), sum x^2 per time chunk (d4w_row_moments).  `filtfilt` is tools.filtfilt / filtfilt_chunk
(:161-209), scipy.signal.filtfilt(b, a) per time chunk on the SOS kernel.  `spec` is tools.spec / tools.__spec_chunk
(:212-236): the Welch power spectral density of every whole chunk of every channel, all of them in one d4w_welch call.
An ndarray in gives float64 ndarrays back; a tensor in gives float32 CUDA tensors (the energy stays float64).
"""
import numpy as np
import scipy.signal as _sps

from . import dsp as _dsp
from . import fk as _fk
from . import rows as _rows

# sections the zero-phase SOS kernel (d4w_sosfiltfilt) takes
SOS_MAX_SECTIONS = 16


def spec(x, fs=200., chunk=3000, nperseg=1024):
    """Welch PSD per chunk: scipy.signal.welch(x[..., c * chunk:(c + 1) * chunk], fs=fs, nperseg=nperseg) for every whole
    chunk c < ns // chunk (the reference's template has int(ns / 3000) rows; a trailing partial chunk is not used).
    x: [ns] or [nx, ns], an ndarray or a CUDA tensor.  Returns (f, Pxx): f = rfftfreq(nperseg, 1 / fs) float64, Pxx
    [ns // chunk, nperseg // 2 + 1] or [nx, ns // chunk, nperseg // 2 + 1] -- float64 for an ndarray in, float32 CUDA for a
    tensor in."""
    tensor = _dsp._is_tensor(x)
    a = x if tensor else np.asarray(x)
    if a.ndim not in (1, 2):
        raise ValueError(f"spec takes [ns] or [nx, ns], not {a.ndim}-D input")
    if (a.is_complex() if tensor else np.iscomplexobj(a)):
        raise ValueError("spec takes real input only")
    ns, chunk = int(a.shape[-1]), int(chunk)
    if chunk < 1 or ns < chunk:
        raise ValueError(f"spec: {ns} samples hold no whole chunk of {chunk}")
    win, nperseg = _dsp.welch_window("hann_periodic", nperseg, chunk)
    lay = _dsp.welch_layout(ns, nperseg, None, None, chunk)
    xd = _dsp._to_device(a)
    if xd.ndim == 1:
        xd = xd.reshape(1, -1)
    p = _rows.welch(xd, lay.nperseg, lay.step, lay.nfft, win, True, _dsp.welch_scale(win, fs, "density"), "mean", chunk=chunk)
    f = np.fft.rfftfreq(lay.nfft, 1 / fs)
    if a.ndim == 1:
        p = p[0]
    if tensor:
        return f, p
    return f, p.to(_dsp._fk._torch().float64).cpu().numpy()


def _blocks(n, c, what):
    """dask-style uniform blocks of an axis of n samples: [(start, stop)], the last one ragged; c = None is one block"""
    if c is None:
        return [(0, n)]
    if isinstance(c, bool) or not isinstance(c, (int, np.integer)) or c < 1:
        raise ValueError(f"{what} = {c!r} must be None or a positive integer")
    return [(s, min(s + int(c), n)) for s in range(0, n, int(c))]


def _input(x, name, ndims=(1, 2)):
    tensor = _dsp._is_tensor(x)
    a = x if tensor else np.asarray(x)
    if a.ndim not in ndims:
        raise ValueError(f"{name} takes {' or '.join(('[ns]', '[nx, ns]')[d - 1] for d in ndims)} input, not {a.ndim}-D")
    if (a.is_complex() if tensor else np.iscomplexobj(a)):
        raise ValueError(f"{name} takes real input only")
    return tensor, a


def fk_filt(data, tint, fs, xint, dx, c_min, c_max, chunks=None):
    """tools.fk_filt: on every block of `chunks` = (cx, ct) (None, or None in either place: the whole axis), the reference's
    fk_filt_chunk -- scipy.signal.detrend(block), fft2, x the block's Gaussian-blurred fan (sigma 40, float32), ifft2, real --
    written back in place of the block.  Blocks of one shape share one fan design and one f-k plan.  A block whose blurred
    fan is constant gets NaN, as the reference's 0 / 0 mask gives.  data: [nx, ns] ndarray (float64 result) or CUDA tensor
    (float32 result).  ValueError, naming dsp.supported_shape, for a block shape the f-k planner does not take."""
    tensor, a = _input(data, "fk_filt", ndims=(2,))
    nx, ns = (int(n) for n in a.shape)
    cx, ct = (None, None) if chunks is None else tuple(chunks)
    rb, tb = _blocks(nx, cx, "chunks[0]"), _blocks(ns, ct, "chunks[1]")
    torch = _fk._torch()
    xd = _dsp._to_device(a)
    dev = xd.device.index
    out = torch.empty_like(xd)
    designs = {}
    for r0, r1 in rb:
        for t0, t1 in tb:
            shape = (r1 - r0, t1 - t0)
            if shape not in designs:
                _fk.get_plan(shape[0], shape[1], dev)          # the planner's ValueError before any design work
                # numpy.fft.fftfreq steps of the block (tools.py:32-33)
                kval, fval = 1.0 / (shape[0] * (xint * dx)), 1.0 / (shape[1] * (tint / fs))
                g = _rows.blurred_fan(shape[0], shape[1], kval, fval, c_min, c_max, 40, device=dev)
                designs[shape] = None if bool(torch.isnan(g[0, 0])) else _fk.FkFilter(g, shape=shape, device=dev)
            flt = designs[shape]
            blk = out[r0:r1, t0:t1]
            if flt is None:
                blk.fill_(float("nan"))
                continue
            buf = blk if blk.is_contiguous() else None
            buf = _rows.detrend_linear(xd[r0:r1, t0:t1], out=buf)
            flt(buf, out=buf)
            if buf is not blk:
                blk.copy_(buf)
    return out if tensor else _dsp._to_host64(out)


def energy_TimeDomain(x, chunk=None):
    """tools.energy_TimeDomain: sum of x^2 over every time chunk (chunk=None: the whole row), in float64 on the GPU.
    Returns [ceil(ns / chunk)] or [nx, ceil(ns / chunk)] float64 (an ndarray, or a CUDA tensor for a tensor in); the last
    chunk is ragged."""
    tensor, a = _input(x, "energy_TimeDomain")
    ns = int(a.shape[-1])
    _blocks(ns, chunk, "chunk")
    xd = _dsp._to_device(a)
    e = _rows.row_moments(xd.reshape(-1, ns), chunk)[:, :, 2]
    e = e[0] if a.ndim == 1 else e
    return e.contiguous() if tensor else e.cpu().numpy()


def filtfilt(x, b, a, padtype="odd", padlen=None, chunk=None):
    """tools.filtfilt: scipy.signal.filtfilt(b, a, chunk, axis=-1) of every time chunk (chunk=None: the whole row), run as the
    zero-phase SOS filter of scipy.signal.tf2sos(b, a) with filtfilt's odd extension of padlen = 3 max(len(a), len(b))
    samples by default (what dsp.bp_filt does for the reference's filtfilt).  ValueError for another padtype, a chunk not
    longer than padlen, or a design of more than 16 second-order sections."""
    if padtype != "odd":
        raise ValueError(f"padtype = {padtype!r}: only filtfilt's default 'odd' extension is computed")
    tensor, arr = _input(x, "filtfilt")
    b, a = np.atleast_1d(np.asarray(b, dtype=np.float64)), np.atleast_1d(np.asarray(a, dtype=np.float64))
    if b.ndim != 1 or a.ndim != 1 or not len(a) or a[0] == 0:
        raise ValueError("b and a must be 1-D coefficient arrays with a[0] != 0")
    sos = _sps.tf2sos(b, a)
    if sos.shape[0] > SOS_MAX_SECTIONS:
        raise ValueError(f"the design has {sos.shape[0]} second-order sections; the SOS kernel takes up to {SOS_MAX_SECTIONS}")
    padlen = 3 * max(len(a), len(b)) if padlen is None else int(padlen)
    ns = int(arr.shape[-1])
    blocks = _blocks(ns, chunk, "chunk")
    if padlen < 0 or min(t1 - t0 for t0, t1 in blocks) <= padlen:
        raise ValueError(f"The length of the input vector x must be greater than padlen, which is {padlen}.")
    xd = _dsp._to_device(arr).reshape(-1, ns)
    nx = xd.shape[0]
    c = blocks[0][1]
    m = ns // c
    if m * c == ns:                                          # whole chunks: one call on the [nx m, c] view
        y = _rows.sosfiltfilt(sos, xd.reshape(nx * m, c), padlen=padlen).reshape(nx, ns)
    else:
        y = _fk._torch().empty_like(xd)
        if m:
            y[:, :m * c] = _rows.sosfiltfilt(sos, xd[:, :m * c].reshape(nx * m, c), padlen=padlen).reshape(nx, m * c)
        y[:, m * c:] = _rows.sosfiltfilt(sos, xd[:, m * c:].contiguous(), padlen=padlen)
    y = y[0] if arr.ndim == 1 else y
    return y if tensor else _dsp._to_host64(y)
