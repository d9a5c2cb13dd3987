"""oracle/noise_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Float64 NumPy/SciPy restatement of the per-channel noise analysis of the reference's scripts/main_bathynoise.py
(:183-194 and :248-259), written from the script's behaviour.  The script itself cannot be imported (it downloads a file
and plots).  Only tests/ may import this module; das4whales_b200/ never does.
"""
import numpy as np
import scipy.signal as sps


def noise_window(fs, tnoise=(19., 26.)):
    """[i0, i1) of trf_fk[:, i0:i1] (:251, :256)"""
    return [int(t * fs) for t in tnoise]


def env_stats(x):
    """the record rows.env_stats computes, in float64: [nx, 5] = {median |hilbert|, mean |hilbert|, mean, mean x^2, var}"""
    x = np.asarray(x, dtype=np.float64)
    env = np.abs(sps.hilbert(x, axis=1))
    return np.stack([np.median(env, axis=1), np.mean(env, axis=1), np.mean(x, axis=1), np.mean(x ** 2, axis=1),
                     np.var(x, axis=1)], axis=1)


def cable_noise_profile(trf_fk, fs, tnoise=(19., 26.), p_ref=1e-11):
    """the script's per-channel quantities for the f-k filtered strain trf_fk [nx, ns]"""
    trf_fk = np.asarray(trf_fk, dtype=np.float64)
    env = np.abs(sps.hilbert(trf_fk, axis=1))
    med = np.median(env, axis=1)                                   # :183
    mean = np.mean(env, axis=1)                                    # :185
    std = np.std(trf_fk, axis=1)                                   # :189
    with np.errstate(divide="ignore", invalid="ignore"):
        std_med_diff = std - med                                   # :192
        SNR_1d = 20 * np.log10(std / med)                          # :194
        i0, i1 = noise_window(fs, tnoise)                          # :251
        noise = trf_fk[:, i0:i1]                                   # :256
        noise_power = np.mean(noise ** 2, axis=1)                  # :257
        noise_power_db = 10 * np.log10(noise_power / p_ref ** 2)   # :258
        noise_mean = np.mean(np.abs(sps.hilbert(noise, axis=1)), axis=1)   # :259
    return {"med": med, "mean": mean, "std": std, "std_med_diff": std_med_diff, "SNR_1d": SNR_1d,
            "noise_power": noise_power, "noise_power_db": noise_power_db, "noise_mean": noise_mean}


def image(trf_fk):
    """the t-x image of :139: |hilbert(trf_fk * 1e9)| / std(trf_fk * 1e9)"""
    y = np.asarray(trf_fk, dtype=np.float64) * 1e9
    return np.abs(sps.hilbert(y, axis=1)) / np.std(y, axis=1, keepdims=True)
