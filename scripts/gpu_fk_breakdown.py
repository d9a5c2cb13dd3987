"""Per-kernel breakdown of the flagship f-k filter (10 000 x 120 000 fp32, fan mask, the workload of bench.py).

    python scripts/gpu_fk_breakdown.py [--rounds R] [--out DIR]

Prints the card (name, power limit, SM clock), then for each of the five passes the median device time over R rounds
(CUDA events, each pass launched alone), the HBM bytes the plan must move in it (FkFilter.traffic_bytes) and the rate
that gives, the median time of a whole filter call, and a torch.profiler table of every kernel the call launches (a
separate run, so the timings above carry no tracing overhead).  With --out, the table and the numbers go to
DIR/fk_breakdown.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NX, NS = 10000, 120000
DX, FS = 2.0419046878814697, 200.0
FAN = (1400.0, 1450.0, 3400.0, 3500.0)
NAMES = ["p1_col_fwd", "p2_row_split", "p3_row_mid", "p4_row_unsplit", "p5_col_inv"]


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        return subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as exc:       # noqa: BLE001
        return f"nvidia-smi unavailable: {exc!r}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import das4whales_b200 as dw
    from das4whales_b200 import synth
    from das4whales_b200.fk import FkFilter
    assert torch.cuda.is_available(), "needs a GPU"
    mask = dw.dsp.fk_filter_design((NX, NS), [0, NX, 1], DX, FS, *FAN)
    flt = FkFilter(mask)
    x = synth.synth_strain(NX, NS, seed=1234)
    y = torch.empty_like(x)
    for _ in range(3):
        flt(x, out=y)
    torch.cuda.synchronize()
    ev = lambda: torch.cuda.Event(enable_timing=True)      # noqa: E731
    pass_ms = [[] for _ in NAMES]
    step_ms = []
    for _ in range(args.rounds):
        for i in range(5):
            a, b = ev(), ev()
            a.record()
            for _ in range(args.steps):
                flt.run_pass(i + 1, x, y)
            b.record()
            torch.cuda.synchronize()
            pass_ms[i].append(a.elapsed_time(b) / args.steps)
        a, b = ev(), ev()
        a.record()
        for _ in range(args.steps):
            flt(x, out=y)
        b.record()
        torch.cuda.synchronize()
        step_ms.append(a.elapsed_time(b) / args.steps)
    traffic = flt.traffic_bytes()
    step = statistics.median(step_ms)
    res = {"card": card(), "shape": [NX, NS], "rows_kept": flt.rows_kept, "col_scheme": flt.plan.col_scheme,
           "t1": flt.plan.t1, "t2": flt.plan.t2, "rounds": args.rounds, "steps_per_round": args.steps,
           "step_ms": {"median": round(step, 4), "min": round(min(step_ms), 4), "max": round(max(step_ms), 4)},
           "passes": {}}
    for i, n in enumerate(NAMES):
        m = statistics.median(pass_ms[i])
        res["passes"][n] = {"ms": round(m, 4), "spread_ms": round(max(pass_ms[i]) - min(pass_ms[i]), 4),
                            "share": round(m / sum(statistics.median(p) for p in pass_ms), 4),
                            "plan_bytes": traffic[n], "gbs": round(traffic[n] / (m * 1e-3) / 1e9, 1) if m > 0 else None}
    # torch.profiler: every kernel of 3 filter calls, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            flt(x, out=y)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "memset" not in e.name.lower() and "memcpy" not in e.name.lower():
            k = kern.setdefault(e.name, [0.0, 0])
            k[0] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
            k[1] += 1
    res["profiler_kernels"] = sorted(({"kernel": k[:160], "ms_per_call": round(v[0] / 3, 4), "launches_per_call": v[1] // 3}
                                      for k, v in kern.items()), key=lambda d: -d["ms_per_call"])
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fk_breakdown.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
