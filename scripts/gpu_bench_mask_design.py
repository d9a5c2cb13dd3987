"""Design time of the hybrid, hybrid_gs and hybrid_ninf_gs f-k masks on the device, with FkCompPipeline's parameters
(14-30 Hz, 1350 / 1450 / 3300 / 3450 m/s): CUDA-event time of each device design plus its table build (what the filter
runs for a new mask: d4w_mask_design, the dense support scan and the transform-order table) at 11 020 x 12 000 and
10 000 x 120 000 after a warm-up, and the construction time of FkCompPipeline at both shapes (host clock around work that
ends in a device synchronise).  Prints one JSON line per measurement with the card's name and power limit, read in the
same run.  `--host` instead times the host designs (what todense() runs) at 11 020 x 12 000 on the CPU.
Usage: python scripts/gpu_bench_mask_design.py [--host] [reps]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

DX, FS = 2.0419046878814697, 200.0
SPEEDS = dict(cs_min=1350., cp_min=1450., cp_max=3300., cs_max=3450., fmin=14., fmax=30.)
INF = {k: v for k, v in SPEEDS.items() if k not in ("cp_max", "cs_max")}
HOST = "--host" in sys.argv
args = [a for a in sys.argv[1:] if a != "--host"]
REPS = max(2, int(args[0]) if args else 5)


def designs(dsp, nx, ns):
    sel = [0, nx, 1]
    return {"hybrid": lambda: dsp.hybrid_filter_design((nx, ns), sel, DX, FS, **INF),
            "hybrid_gs": lambda: dsp.hybrid_gs_filter_design((nx, ns), sel, DX, FS, **INF),
            "hybrid_ninf_gs": lambda: dsp.hybrid_ninf_gs_filter_design((nx, ns), sel, DX, FS, **SPEEDS)}


if HOST:
    from das4whales_b200 import dsp
    nx, ns = 11020, 12000
    total = 0.0
    for name, make in designs(dsp, nx, ns).items():
        m = make()
        t0 = time.perf_counter()
        d = m.todense()
        s = time.perf_counter() - t0
        total += s
        rows = int(np.count_nonzero(np.any(d != 0, axis=1)))
        print(json.dumps(dict(case="host_design", design=name, nx=nx, ns=ns, s=round(s, 2), rows_nonzero=rows,
                              cpus=os.cpu_count())), flush=True)
        del d, m
    print(json.dumps(dict(case="host_design_total", nx=nx, ns=ns, s=round(total, 2), cpus=os.cpu_count())), flush=True)
    sys.exit(0)

import torch
from das4whales_b200 import dsp, fk, pipeline


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:                     # noqa: BLE001
        return None


gpu, watts = torch.cuda.get_device_name(), power_limit_w()


def emit(**kw):
    print(json.dumps(dict(kw, gpu=gpu, power_limit_w=watts)), flush=True)


def device_design(mask, plan):
    """a fresh device design and table build of `mask` for `plan` (the per-plan cache is bypassed)"""
    return fk._DenseMaskHolder(plan, mask._design_plane(plan)).dm


for nx, ns in ((11020, 12000), (10000, 120000)):
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    for name, make in designs(dsp, nx, ns).items():
        m = make()
        device_design(m, plan)                                        # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        plane_ms = []
        for _ in range(REPS):                                         # the design kernels alone
            e0.record()
            p = m._design_plane(plan)
            e1.record(); torch.cuda.synchronize()
            plane_ms.append(e0.elapsed_time(e1))
            del p
        e0.record()
        for _ in range(REPS):                                         # design + support scan + table (synchronises)
            dm = device_design(m, plan)
        e1.record(); torch.cuda.synchronize()
        emit(case="device_design", design=name, nx=nx, ns=ns, design_ms=round(float(np.median(plane_ms)), 3),
             design_and_table_ms=round(e0.elapsed_time(e1) / REPS, 3), rows_kept=int(dm.rows))
        del dm
    pipeline.FkCompPipeline(nx, ns, [0, nx, 1], DX, FS, 1.0)          # warm-up
    fk.free_plans()
    torch.cuda.synchronize()
    t = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        pipe = pipeline.FkCompPipeline(nx, ns, [0, nx, 1], DX, FS, 1.0)
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
        del pipe
        fk.free_plans()                                               # every construction plans and designs from scratch
    emit(case="FkCompPipeline_construct", nx=nx, ns=ns, ms=round(1e3 * float(np.median(t)), 1),
         ms_min=round(1e3 * min(t), 1))
    torch.cuda.empty_cache()
