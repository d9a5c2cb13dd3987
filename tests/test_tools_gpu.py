"""GPU: the tools module and the device-designed fan of dsp.fk_filt against float64 references."""
import numpy as np
import pytest
import scipy.signal as sps

from conftest import rel_err
from oracle import dsp_oracle as O, tools_oracle as T, tools_golden as G

pytestmark = pytest.mark.gpu
DX, FS = G.DX, G.FS
TOL = 1e-4          # test_rows_gpu.py's bound for the row / SOS kernels
FK_MAX, FK_L2 = 1e-4, 1e-5


@pytest.fixture(scope="module")
def dw():
    import __graft_entry__
    __graft_entry__.build()
    import das4whales_b200
    return das4whales_b200


def _kf(shape, tint=1, fs=FS, xint=1, dx=DX):
    return 1.0 / (shape[0] * (xint * dx)), 1.0 / (shape[1] * (tint / fs))


@pytest.mark.parametrize("nx,ns", [(40, 240), (551, 1200), (4897, 1200), (2000, 12000)])
def test_device_fan_sigma_20(dw, nx, ns):
    """dsp.fk_filt's fan: 4897 channels is a chirp-z channel count of the f-k filter"""
    g = dw.rows.blurred_fan(nx, ns, *_kf((nx, ns)), 1450., 3400., 20).cpu().numpy()
    ref = O.fk_filt_mask((nx, ns), 1, FS, 1, DX, 1450., 3400.)
    err = float(np.max(np.abs(g - ref)))
    print(f"fan sigma 20 {nx} x {ns}: max abs err {err:.2e}")
    assert err <= 2e-7


@pytest.mark.parametrize("nx,ns", [(41, 239), (551, 1200), (10000, 300)])
def test_device_fan_sigma_40(dw, nx, ns):
    g = dw.rows.blurred_fan(nx, ns, *_kf((nx, ns)), 1400., 3500., 40).cpu().numpy()
    ref = T.fan_mask((nx, ns), 1, FS, 1, DX, 1400., 3500., sigma=40)
    err = float(np.max(np.abs(g - ref)))
    print(f"fan sigma 40 {nx} x {ns}: max abs err {err:.2e}")
    assert err <= 2e-7


def test_device_fan_constant_is_nan(dw):
    assert dw.rows.blurred_fan(2, 5, *_kf((2, 5)), 1400., 3500., 20).isnan().all()


@pytest.mark.parametrize("nx,ns", [(300, 1200), (551, 1200), (1000, 960)])
def test_dsp_fk_filt_device_design(dw, nx, ns):
    x = np.random.default_rng(nx).standard_normal((nx, ns))
    y = dw.dsp.fk_filt(x, 1, FS, 1, DX, 1450., 3400.)
    e = rel_err(y, O.fk_filt(x, 1, FS, 1, DX, 1450., 3400.))
    print(f"dsp.fk_filt {nx} x {ns}: max-norm {e[0]:.2e}, l2 {e[1]:.2e}")
    assert e[0] <= FK_MAX and e[1] <= FK_L2


def test_tools_fk_filt_golden(dw, golden):
    g = golden("tools")
    for i, (nx, ns, cmin, cmax) in enumerate(G.FK_CASES):
        y = dw.tools.fk_filt(g[f"fk_x_{i}"], 1, FS, 1, DX, cmin, cmax)
        ref = g[f"fk_y_{i}"]
        if np.isnan(ref).all():
            assert np.isnan(y).all(), (nx, ns)
            continue
        e = rel_err(y, ref)
        print(f"tools.fk_filt {nx} x {ns}: max-norm {e[0]:.2e}, l2 {e[1]:.2e}")
        assert e[0] <= FK_MAX and e[1] <= FK_L2, (nx, ns, e)


@pytest.mark.parametrize("nx,ns,chunks", [(600, 2400, (None, 600)), (600, 2500, (250, 1000)), (131, 1200, (50, None)),
                                          (120, 700, (100, 240))])
def test_tools_fk_filt_blocks(dw, nx, ns, chunks):
    """uniform blocks with ragged last ones: each block detrended and filtered with its own fan, as map_blocks does"""
    import torch
    rng = np.random.default_rng(ns)
    x = rng.standard_normal((nx, ns)) + 0.003 * np.arange(ns)[None, :]
    ref = T.fk_filt(x, 1, FS, 1, DX, 1450., 3400., chunks)
    y = dw.tools.fk_filt(x, 1, FS, 1, DX, 1450., 3400., chunks=chunks)
    e = rel_err(y, ref)
    print(f"tools.fk_filt {nx} x {ns} chunks {chunks}: max-norm {e[0]:.2e}, l2 {e[1]:.2e}")
    assert y.dtype == np.float64 and e[0] <= FK_MAX and e[1] <= FK_L2
    yt = dw.tools.fk_filt(torch.from_numpy(x.astype(np.float32)).cuda(), 1, FS, 1, DX, 1450., 3400., chunks=chunks)
    assert yt.dtype == torch.float32 and yt.is_cuda
    assert rel_err(yt.cpu().numpy(), ref)[0] <= FK_MAX


def test_tools_fk_filt_unsupported_block(dw):
    x = np.zeros((40, 134))                        # 67 samples per block: a prime factor above 61
    with pytest.raises(ValueError, match="supported_shape"):
        dw.tools.fk_filt(x, 1, FS, 1, DX, 1450., 3400., chunks=(None, 67))


def test_detrend_and_moments(dw):
    import torch
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((70, 5000)) * 3 + np.arange(5000)[None, :] * rng.standard_normal((70, 1)) + 100).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    for r0, r1, t0, t1 in ((0, 70, 0, 5000), (3, 50, 1234, 4321), (10, 11, 7, 8), (0, 70, 4000, 4002)):
        y = dw.rows.detrend_linear(xd[r0:r1, t0:t1]).cpu().numpy()
        blk = x[r0:r1, t0:t1].astype(np.float64)
        ref = sps.detrend(blk, axis=-1)
        bound = 1e-6 * np.max(np.abs(blk), axis=1)
        assert np.all(np.max(np.abs(y - ref), axis=1) <= bound), (r0, r1, t0, t1)
    m = dw.rows.row_moments(xd, 1000).cpu().numpy()
    x64 = x.astype(np.float64).reshape(70, 5, 1000)
    t = np.arange(1000)
    assert np.allclose(m[:, :, 0], x64.sum(-1), rtol=1e-9, atol=1e-6)
    assert np.allclose(m[:, :, 1], (x64 * t).sum(-1), rtol=1e-9)
    assert np.allclose(m[:, :, 2], (x64 ** 2).sum(-1), rtol=1e-12)


def test_energy(dw, golden):
    import torch
    g = golden("tools")
    x = g["energy_x"]
    for chunk in (3001, 1000, 333):
        e = dw.tools.energy_TimeDomain(x, chunk)
        ref = g[f"energy_{chunk}"]
        assert e.dtype == np.float64 and e.shape == ref.shape
        assert np.max(np.abs(e - ref) / ref) <= 1e-6, chunk
    et = dw.tools.energy_TimeDomain(torch.from_numpy(x.astype(np.float32)).cuda(), 1000)
    assert et.dtype == torch.float64 and et.is_cuda
    assert np.max(np.abs(et.cpu().numpy() - g["energy_1000"]) / g["energy_1000"]) <= 1e-6
    e1 = dw.tools.energy_TimeDomain(x[2], None)
    assert e1.shape == (1,) and abs(e1[0] - np.sum(x[2] ** 2)) <= 1e-6 * e1[0]


@pytest.mark.parametrize("i", range(len(G.IIR_CASES)))
def test_filtfilt(dw, golden, i):
    """Butterworth designs in (b, a) form: low-pass 2, high-pass 4, band-pass 5 and bp_filt's band-pass 8"""
    import torch
    g = golden("tools")
    x, b, a = g["iir_x"], g[f"iir_b_{i}"], g[f"iir_a_{i}"]
    for chunk in (2600, 1000):
        y = dw.tools.filtfilt(x, b, a, chunk=chunk)
        e = rel_err(y, g[f"iir_y_{i}_{chunk}"])
        print(f"filtfilt {G.IIR_CASES[i]} chunk {chunk}: max-norm {e[0]:.2e}")
        assert y.dtype == np.float64 and e[0] <= TOL, (chunk, e)
    xl = np.random.default_rng(i).standard_normal((5, 6000))
    for chunk in (None, 1500, 1400):                       # one block, whole chunks, ragged
        ref = T.filtfilt(xl, b, a, chunk)
        assert rel_err(dw.tools.filtfilt(xl, b, a, chunk=chunk), ref)[0] <= TOL, chunk
    yt = dw.tools.filtfilt(torch.from_numpy(xl[1].astype(np.float32)).cuda(), b, a, chunk=1400)
    assert yt.dtype == torch.float32 and yt.shape == (6000,)
    assert rel_err(yt.cpu().numpy(), T.filtfilt(xl[1], b, a, 1400))[0] <= TOL
