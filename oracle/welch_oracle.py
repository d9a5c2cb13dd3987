"""oracle/welch_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Float64 restatement of the reference's per-channel power spectral density, tools.spec / tools.__spec_chunk
(das4whales/tools.py:212-236): scipy.signal.welch(chunk, fs=200, nperseg=1024) of every 3 000-sample chunk, one spectrum per
whole chunk.  The reference module imports xarray and dask, which are not dependencies here, so it cannot be loaded
unmodified; its xarray map_blocks over time chunks is restated as a loop over whole chunks.  Only tests/ may import this
module; das4whales_b200/ never does.
"""
import numpy as np
import scipy.signal as sps


def welch(x, **kw):
    """scipy.signal.welch itself, in float64 along the last axis"""
    return sps.welch(np.asarray(x, dtype=np.float64), **kw)


def spec(x, fs=200., chunk=3000, nperseg=1024):
    """tools.spec: (f, Pxx [..., ns // chunk, nperseg // 2 + 1]), one __spec_chunk welch call per whole chunk"""
    x = np.asarray(x, dtype=np.float64)
    nch = x.shape[-1] // chunk
    parts = [sps.welch(x[..., c * chunk:(c + 1) * chunk], fs=fs, nperseg=nperseg) for c in range(nch)]
    return parts[0][0], np.stack([p for _, p in parts], axis=-2)
