"""Sweep f-k plan knobs (env vars read at plan creation) at the BASELINE config-2 shape and print
per-pass device times.  One subprocess per configuration.
    python scripts/gpu_tune_fk.py            # run the sweep
    python scripts/gpu_tune_fk.py --one      # time the current environment's configuration"""
import json, os, subprocess, sys, itertools
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NX, NS = int(os.environ.get("TUNE_NX", 10000)), int(os.environ.get("TUNE_NS", 120000))

def one():
    import torch
    import das4whales_b200 as dw
    from das4whales_b200 import synth
    from das4whales_b200.fk import FkFilter
    mask = dw.dsp.fk_filter_design((NX, NS), [0, NX, 1], 2.0419046878814697, 200.0)
    flt = FkFilter(mask)
    x = synth.plane_wave(NX, NS, 400, 24000)
    y = torch.empty_like(x)
    for _ in range(2):
        flt(x, out=y)
    err = float((y - x).abs().max())
    reps = 4
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(6)] for _ in range(reps)]
    torch.cuda.synchronize()
    for r in range(reps):
        ev[r][0].record()
        for i in range(5):
            flt.run_pass(i + 1, x, y)
            ev[r][i + 1].record()
    torch.cuda.synchronize()
    ms = [sum(ev[r][i].elapsed_time(ev[r][i + 1]) for r in range(reps)) / reps for i in range(5)]
    if os.environ.get("D4W_FK_DEBUG"):
        from das4whales_b200 import _lib
        buf = _lib.ffi.new("unsigned long long[8]")
        _lib.lib().d4w_fk_debug_phases(flt.plan.ptr, buf)      # reset
        flt(x, out=y); torch.cuda.synchronize()
        _lib.check(_lib.lib().d4w_fk_debug_phases(flt.plan.ptr, buf), "dbg")
        nsm = torch.cuda.get_device_properties(x.device).multi_processor_count
        print("phase Mcycles per SM (one apply): fwd load/fft/out =", [round(buf[i] / nsm / 1e6, 3) for i in range(3)],
              " inv drain/fill/fft/store =", [round(buf[i] / nsm / 1e6, 3) for i in range(4, 8)])
    print(json.dumps({"ms": [round(m, 3) for m in ms], "total": round(sum(ms), 3), "err": err,
                      "t1": flt.plan.t1, "t2": flt.plan.t2, "tile": flt.plan.tile}))

if "--one" in sys.argv:
    one()
    sys.exit(0)

configs = []
for thr, maxr in itertools.product((256, 512), (16, 10, 8)):
    configs.append({"D4W_COL_THREADS": thr, "D4W_COL_MAX_RADIX": maxr})
configs.append({"D4W_COL_DUAL": 0, "D4W_COL_THREADS": 512})
for t1, rthr, rmaxr in ((12, 256, 16), (12, 512, 16), (12, 256, 10), (24, 256, 16), (25, 256, 16), (20, 256, 16), (15, 256, 16), (12, 256, 25)):
    configs.append({"D4W_T1": t1, "D4W_ROW_THREADS": rthr, "D4W_ROW_MAX_RADIX": rmaxr})
if len(sys.argv) > 1 and sys.argv[1] == "--col":
    configs = configs[:7]
for cfg in configs:
    env = dict(os.environ)
    env.update({k: str(v) for k, v in cfg.items()})
    r = subprocess.run([sys.executable, __file__, "--one"], env=env, capture_output=True, text=True)
    out = r.stdout.strip().splitlines()
    print(cfg, out[-1] if out else ("ERR " + r.stderr.strip()[-300:]), flush=True)
