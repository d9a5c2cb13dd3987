"""Time detect.compute_cross_correlograms (HF + LF fin-whale templates) at 10 000 x 120 000."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import das4whales_b200 as dw
from das4whales_b200 import synth
nx, ns, FS = 10000, 120000, 200.0
x = synth.synth_strain(nx, ns, seed=3)
t = np.arange(ns) / FS
tpls = [dw.detect.gen_template_fincall(t, FS, 17.8, 28.8, 0.68), dw.detect.gen_template_fincall(t, FS, 14.7, 21.8, 0.78)]
o = dw.detect.compute_cross_correlograms(x, tpls); del o
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize(); e0.record()
for _ in range(5):
    o = dw.detect.compute_cross_correlograms(x, tpls); del o
e1.record(); torch.cuda.synchronize()
print("xcorr HF+LF ms:", round(e0.elapsed_time(e1) / 5, 2))
