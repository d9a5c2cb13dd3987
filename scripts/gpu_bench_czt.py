"""Per-pass device time (P1-P5, CUDA events) and the whole f-k step for a chirp-z channel count (7346 x 12 000, the
tapered hybrid_ninf mask of the reference scripts) and, as the reference point, the smooth 11 020 x 12 000.
One JSON line per shape.  Usage: python scripts/gpu_bench_czt.py [reps]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import das4whales_b200 as dw
from das4whales_b200.fk import FkFilter
DX, FS = 2.0419046878814697, 200.0
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20


def timed(fn):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


for nx, ns in ((7346, 12000), (11020, 12000)):
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(nx))
    m = dw.dsp.hybrid_ninf_filter_design((nx, ns), [0, nx, 1], DX, FS, 1350., 1450., 3300, 3450, 14., 30.)
    flt = FkFilter(m)
    y = torch.empty_like(x)
    passes = {f"P{i}": round(timed(lambda i=i: flt.run_pass(i, x, y, tapering=True)), 3) for i in range(1, 6)}
    step = timed(lambda: flt(x, out=y, tapering=True))
    p = flt.plan
    print(json.dumps({"nx": nx, "ns": ns, "col_scheme": p.col_scheme, "tile": p.tile, "col_stages": p.col_stages,
                      "t1": p.t1, "t2": p.t2, "rows_kept": flt.rows_kept, "pass_ms": passes, "step_ms": round(step, 3),
                      "gpu": torch.cuda.get_device_name()}), flush=True)
    del flt, x, y
    torch.cuda.empty_cache()
