"""Per-kernel breakdown of the flagship f-k filter (10 000 x 120 000 fp32, fan mask, the workload of bench.py).

    python scripts/gpu_fk_breakdown.py [--rounds R] [--out DIR]

Prints the card (name, power limit, SM clock), then for each of the five passes the median device time over R rounds
(CUDA events, each pass launched alone), the HBM bytes the plan must move in it (FkFilter.traffic_bytes) and the rate
that gives, the median time of a whole filter call, and a torch.profiler table of every kernel the call launches (a
separate run, so the timings above carry no tracing overhead).  With --out, the table and the numbers go to
DIR/fk_breakdown.json.

For the two-level column passes P1 and P5 it also reports the L2 sector bytes the plan moves and the rate that gives:
x (or y), the level-A/B intermediate V written by one level and read by the other, and the kept rows W.  Level A moves
V in whole 32-byte sectors with the blocked position order of the kernels in this tree; --v-layout natural counts V's
level-A side at the half-sector efficiency of the earlier order (for timing a build of an earlier commit)."""
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


def two_level_shape(nx):
    """(X1, X2) of the planner's two-level column split: X1 the largest of 25, 20, 16 dividing nx with 8 <= X2 <= 1024"""
    for x1 in (25, 20, 16):
        if nx % x1 == 0 and 8 <= nx // x1 <= 1024:
            return x1, nx // x1
    return None


def col_l2_sector_bytes(nx, ns, rows_kept, v_layout):
    """L2 sector bytes of one two-level column pass (P1 or P5), from the plan's shape.  Every access is a whole
    32-byte sector except level A's V accesses in the natural order, where each 16-byte access fills half of one."""
    x1, x2 = two_level_shape(nx)
    planes = x1 // 2 + 1
    xy = nx * ns * 4                                   # x in (P1) or y out (P5)
    v = planes * x2 * (ns // 2) * 16                   # V: one 16-byte element per plane, c2 row and sample pair
    w = rows_kept * ns * 8                             # kept wavenumber rows, complex64
    v_a = v * (2 if v_layout == "natural" else 1)
    return {"x_or_y": xy, "v_level_a": v_a, "v_level_b": v, "w": w, "total": xy + v_a + v + w}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out")
    ap.add_argument("--v-layout", choices=("blocked", "natural"), default="blocked",
                    help="position order of V inside a chunk row in the build being timed")
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
        if n in ("p1_col_fwd", "p5_col_inv") and flt.plan.col_scheme in (2, 3):
            l2 = col_l2_sector_bytes(NX, NS, flt.rows_kept, args.v_layout)
            res["passes"][n]["l2_sector_bytes"] = l2
            res["passes"][n]["l2_sector_gbs"] = round(l2["total"] / (m * 1e-3) / 1e9, 1) if m > 0 else None
    res["v_layout"] = args.v_layout
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
