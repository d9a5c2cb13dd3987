"""das4whales_b200.tools -- the channel-parallel part of `das4whales.tools` (/root/reference/src/das4whales/tools.py).

`spec` is tools.spec / tools.__spec_chunk (tools.py:212-236) without xarray or dask: the Welch power spectral density of
every whole chunk of every channel, all of them in one d4w_welch call on the GPU.
"""
import numpy as np

from . import dsp as _dsp
from . import rows as _rows


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
