"""oracle/tools_golden.py -- TEST INFRASTRUCTURE.

Runs the UNMODIFIED reference tools module (das4whales/tools.py, loaded through oracle/ref_loader.py) -- its chunk functions fk_filt_chunk,
_energy_TimeDomain_chunk and filtfilt_chunk -- on seeded float64 blocks and writes the results to tests/golden/tools.npz,
after checking them against the restatements of oracle/tools_oracle.py.  xarray, dask and pandas are not installed where
the fixtures are made: `load_tools` stubs them with a DataArray that holds an ndarray (.values, .dims, .coords, .name,
.attrs, ** and .sum(dim, keepdims)), which is all the chunk functions touch.

    python -m oracle.tools_golden [out_dir]      # from the repo root; out_dir defaults to tests/golden
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_loader, tools_oracle as T  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
DX, FS = 2.0419046878814697, 200.0
# (nx, ns, c_min, c_max): odd and even sizes on both axes, and the reference's own 2 x 5 test case (its fan blurs to a
# constant, so the mask and the output are NaN)
FK_CASES = [(40, 240, 1450., 3400.), (41, 245, 1450., 3400.), (33, 120, 1400., 3500.), (64, 75, 1450., 3400.), (2, 5, 1400., 3500.)]
# Butterworth designs in (b, a) form: (order, critical frequencies in Hz, type)
IIR_CASES = [(2, [20.], "low"), (4, [5.], "high"), (5, [10., 30.], "bandpass"), (8, [15., 25.], "bandpass")]


class DataArray:
    def __init__(self, data, dims=None, coords=None, name=None, attrs=None):
        self.values = np.asarray(data)
        self.dims = tuple(dims) if dims is not None else tuple(f"dim_{i}" for i in range(self.values.ndim))
        self.coords = {} if coords is None else coords
        self.name, self.attrs = name, ({} if attrs is None else attrs)

    def __array__(self, dtype=None, copy=None):
        return self.values if dtype is None else self.values.astype(dtype)

    @property
    def shape(self):
        return self.values.shape

    def __pow__(self, p):
        return DataArray(self.values ** p, self.dims, self.coords, self.name, self.attrs)

    def sum(self, dim, keepdims=False):
        return DataArray(self.values.sum(axis=self.dims.index(dim), keepdims=keepdims), self.dims, self.coords)


def load_tools():
    """The reference's tools module (unmodified source) with xarray / dask / pandas stubbed."""
    ref_loader.load()                                   # stubs matplotlib, registers the das4whales package
    for n in ("xarray", "dask", "dask.array", "pandas"):
        try:
            importlib.import_module(n)
        except Exception:
            ref_loader._stub(n)
    xr = sys.modules["xarray"]
    if not hasattr(xr, "DataArray"):
        xr.DataArray = DataArray
    spec = importlib.util.spec_from_file_location("das4whales.tools", os.path.join(ref_loader._SRC, "tools.py"))
    m = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = m
    spec.loader.exec_module(m)
    return m


def make_tools(out_dir=OUT):
    import scipy.signal as sps
    tools = load_tools()
    rng = np.random.default_rng(11)
    out = {}
    for i, (nx, ns, cmin, cmax) in enumerate(FK_CASES):
        x = rng.standard_normal((nx, ns)) + 0.01 * np.arange(ns)[None, :] + 0.5      # a trend for the detrend to remove
        y = tools.fk_filt_chunk(DataArray(x, dims=["distance", "time"]), 1, FS, 1, DX, cmin, cmax).values
        ref = T.fk_filt_chunk(x, 1, FS, 1, DX, cmin, cmax)
        assert np.array_equal(np.isnan(y), np.isnan(ref)) and np.allclose(y, ref, rtol=0, atol=1e-12, equal_nan=True), (nx, ns)
        out[f"fk_x_{i}"], out[f"fk_y_{i}"] = x, y
    x = rng.standard_normal((5, 3001)) * np.linspace(1, 3, 5)[:, None]
    out["energy_x"] = x
    for chunk in (3001, 1000, 333):
        blocks = [tools._energy_TimeDomain_chunk(DataArray(x[:, t0:t1], dims=["distance", "time"]), "time").values
                  for t0, t1 in T.blocks(x.shape[1], chunk)]
        e = np.concatenate(blocks, axis=-1)
        assert np.allclose(e, T.energy_time_domain(x, chunk), rtol=1e-14, atol=0)
        out[f"energy_{chunk}"] = e
    x = rng.standard_normal((2, 2600))                 # 2 whole chunks of 1000 and a ragged 600, longer than every padlen
    out["iir_x"] = x
    for i, (order, fc, kind) in enumerate(IIR_CASES):
        b, a = sps.butter(order, np.asarray(fc) / (FS / 2), kind)
        out[f"iir_b_{i}"], out[f"iir_a_{i}"] = b, a
        for chunk in (2600, 1000):
            blocks = [tools.filtfilt_chunk(DataArray(x[:, t0:t1], dims=["distance", "time"]), dim="time", b=b, a=a).values
                      for t0, t1 in T.blocks(x.shape[1], chunk)]
            y = np.concatenate(blocks, axis=-1)
            assert np.allclose(y, T.filtfilt(x, b, a, chunk), rtol=0, atol=1e-12)
            out[f"iir_y_{i}_{chunk}"] = y
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "tools.npz"), **out)


if __name__ == "__main__":
    make_tools(sys.argv[1] if len(sys.argv) > 1 else OUT)
