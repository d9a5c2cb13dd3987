"""One call of every per-channel operator (no warm-up) so that `ncu -k regex:...` captures each kernel once:
    ncu --set full --clock-control none -k regex:"k_xcorr|k_row_stats|k_hsplit|k_hilbert_row|k_sos_pass|k_stft_mag|k_row_median|k_speccorr|k_row_max|k_snr_plain|k_peak|k_raw2strain" \
        -o gpurun_out/r01g_rows python scripts/gpu_profile_rows.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import das4whales_b200 as dw
from das4whales_b200 import rows, synth

NX, NS, FS = int(os.environ.get("PROF_NX", 2000)), 120000, 200.0
x = synth.synth_strain(NX, NS, seed=5)
t = np.arange(NS) / FS
tpls = [dw.detect.gen_template_fincall(t, FS, 17.8, 28.8, 0.68), dw.detect.gen_template_fincall(t, FS, 14.7, 21.8, 0.78)]
hf, lf = dw.detect.compute_cross_correlograms(x, tpls)             # k_row_stats, k_xcorr
env = rows.envelope(hf)                                            # k_hsplit_fwd2, k_row_mid_fused, k_hsplit_inv2
snr = dw.dsp.snr_tr_array(hf, env=True); snr2 = dw.dsp.snr_tr_array(hf, env=False)   # k_snr_plain
bp = dw.dsp.bp_filt(x, FS, 14.0, 30.0)                             # k_sos_pass
picks = rows.find_peaks_flags(env, 6.0)                            # k_peak_levels, k_peak_pick
raw = torch.randint(-2 ** 20, 2 ** 20, (NX, NS), dtype=torch.int32, device="cuda")
st = rows.raw2strain(raw, 1e-9)                                    # k_raw2strain
sub = x[:200].contiguous()
kern = {"f0": 27.0, "f1": 16.0, "dur": 0.9, "bdwidth": 4.0}
sc = dw.detect.compute_cross_correlogram_spectrocorr(sub, FS, (12.0, 36.0), kern, 0.8, 0.95)   # k_stft_mag, k_row_max, k_row_median, k_speccorr
torch.cuda.synchronize()
print("ok")
