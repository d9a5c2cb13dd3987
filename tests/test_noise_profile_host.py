"""CPU tests of the cable noise profile's host side (dsp.noise_window, dsp.noise_profile_from_stats): the window index
arithmetic of scripts/main_bathynoise.py:251, the profile assembled from the [nx, 5] env_stats record against the
float64 oracle, IEEE handling of zero channels, and no CPU fallback."""
import numpy as np
import pytest

from oracle import noise_oracle as N

FS = 200.0


@pytest.fixture(scope="module")
def dsp():
    from das4whales_b200 import dsp
    return dsp


@pytest.mark.parametrize("tnoise,fs", [((19., 26.), 200.), ((15., 19.), 200.), ((0.0, 0.01), 200.), ((1.3, 2.7), 173.),
                                       ((19.999, 26.001), 200.)])
def test_noise_window_is_the_scripts_int_t_fs(dsp, tnoise, fs):
    i0, i1 = dsp.noise_window(24000, fs, tnoise)
    assert (i0, i1) == tuple(N.noise_window(fs, tnoise)) == (int(tnoise[0] * fs), int(tnoise[1] * fs))


def test_noise_window_of_the_script_is_1400_samples(dsp):
    assert dsp.noise_window(12000, FS) == (3800, 5200)


@pytest.mark.parametrize("tnoise,ns", [((26., 19.), 12000), ((19., 19.), 12000), ((19., 19.004), 12000), ((-1., 5.), 12000),
                                       ((19., 60.01), 12000), ((61., 62.), 12000)])
def test_noise_window_rejects_empty_or_outside(dsp, tnoise, ns):
    with pytest.raises(ValueError):
        dsp.noise_window(ns, FS, tnoise)


def test_noise_window_may_end_at_ns(dsp):
    assert dsp.noise_window(12000, FS, (50., 60.)) == (10000, 12000)


def _records(x, tnoise, fs=FS):
    i0, i1 = N.noise_window(fs, tnoise)
    return N.env_stats(x), N.env_stats(x[:, i0:i1])


@pytest.mark.parametrize("ns", [1400, 1401, 3000])
def test_profile_from_records_matches_oracle(dsp, ns):
    rng = np.random.default_rng(ns)
    x = rng.standard_normal((7, ns)) * 1e-9 * np.linspace(0.5, 3.0, 7)[:, None]
    x[3] += 2e-9 * np.sin(2 * np.pi * 20 * np.arange(ns) / FS)
    tnoise = (1.0, 4.5)
    full, win = _records(x, tnoise)
    prof = dsp.noise_profile_from_stats(full, win)
    ref = N.cable_noise_profile(x, FS, tnoise)
    assert tuple(prof) == dsp.NOISE_PROFILE_KEYS == tuple(ref)
    for k in dsp.NOISE_PROFILE_KEYS:
        assert prof[k].dtype == np.float64 and prof[k].shape == (7,) and prof[k].flags.c_contiguous
        np.testing.assert_allclose(prof[k], ref[k], rtol=1e-12, atol=0, err_msg=k)


def test_profile_zero_channel_is_nan_and_minus_inf(dsp):
    x = np.random.default_rng(0).standard_normal((3, 2000))
    x[1] = 0.0
    full, win = _records(x, (1.0, 5.0))
    prof = dsp.noise_profile_from_stats(full, win)
    ref = N.cable_noise_profile(x, FS, (1.0, 5.0))
    assert np.isnan(prof["SNR_1d"][1]) and np.isnan(ref["SNR_1d"][1])
    assert prof["noise_power_db"][1] == -np.inf == ref["noise_power_db"][1]
    for k in ("med", "mean", "std", "std_med_diff", "noise_power", "noise_mean"):
        assert prof[k][1] == 0.0, k
    assert np.all(np.isfinite(prof["SNR_1d"][[0, 2]])) and np.all(np.isfinite(prof["noise_power_db"][[0, 2]]))


def test_profile_p_ref(dsp):
    x = np.random.default_rng(1).standard_normal((2, 800))
    full, win = _records(x, (0.5, 3.0))
    a = dsp.noise_profile_from_stats(full, win, p_ref=1e-11)["noise_power_db"]
    b = dsp.noise_profile_from_stats(full, win, p_ref=1e-6)["noise_power_db"]
    np.testing.assert_allclose(a - b, 100.0, rtol=1e-12)


def test_no_cpu_fallback(dsp):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        dsp.cable_noise_profile(np.zeros((4, 6000)), FS)
    with pytest.raises(ValueError):                     # the window is checked before anything runs
        dsp.cable_noise_profile(np.zeros((4, 1000)), FS)
