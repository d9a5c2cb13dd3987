"""Device time (CUDA events, after warm-up) of an f-k mask bank (fk.FkFilterBank: one forward transform, then P3-P5 per
mask) against n separate FkFilter calls on the same device tensor, in alternated rounds, with the per-pass split of
both (each pass timed alone over REPS launches, run_pass).  Checks that every bank output equals its FkFilter output.
  * 11 020 x 12 000 with the four masks of scripts/main_fkcomp.py:73-95 (nf_cos, nf_gs, inf_cos, inf_gs);
  * 10 000 x 120 000 with four analytic masks: fan and hybrid_ninf at two speed bands each.
Prints one JSON line per measurement with the card's name and power limit, and the acceptance figure: the bank's saving
against (n - 1) x (P1 + P2) of the single-mask plan.
Usage: python scripts/gpu_bench_fk_bank.py [reps]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import dsp, fk
REPS = max(5, int(sys.argv[1]) if len(sys.argv) > 1 else 10)
WARMUP = 3
ROUNDS = 5
DX, FS = 2.0419046878814697, 200.0


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:                     # noqa: BLE001
        return None


def timed(fn, reps=REPS):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def line(**kw):
    print(json.dumps(dict(kw, reps=REPS, warmup=WARMUP, gpu=gpu, power_limit_w=watts)), flush=True)


def fkcomp_masks(nx, ns):
    sel, c = [0, nx, 1], (1350., 1450., 3300., 3450.)
    fin = dict(cs_min=c[0], cp_min=c[1], cp_max=c[2], cs_max=c[3], fmin=14., fmax=30.)
    inf = dict(cs_min=c[0], cp_min=c[1], fmin=14., fmax=30.)
    return (["nf_cos", "nf_gs", "inf_cos", "inf_gs"],
            [dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, **fin), dsp.hybrid_ninf_gs_filter_design((nx, ns), sel, DX, FS, **fin),
             dsp.hybrid_filter_design((nx, ns), sel, DX, FS, **inf), dsp.hybrid_gs_filter_design((nx, ns), sel, DX, FS, **inf)])


def analytic_masks(nx, ns):
    sel = [0, nx, 1]
    bands = ((1350., 1450., 3300., 3450.), (1400., 1500., 2500., 2700.))
    names, masks = [], []
    for i, b in enumerate(bands):
        names += [f"fan_{i}", f"hybrid_ninf_{i}"]
        masks += [dsp.fk_filter_design((nx, ns), sel, DX, FS, *b),
                  dsp.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, *b, fmin=14., fmax=30.)]
    return names, masks


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
for (nx, ns), design in (((11020, 12000), fkcomp_masks), ((10000, 120000), analytic_masks)):
    names, masks = design(nx, ns)
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns))
    bank = fk.FkFilterBank(masks)
    singles = [fk.FkFilter(m) for m in masks]
    outs = [torch.empty_like(x) for _ in masks]
    equal = all(torch.equal(a, f(x)) for a, f in zip(bank(x, outs=outs), singles))
    assert equal
    n = len(masks)
    b_ms, s_ms = [], []
    for _ in range(ROUNDS):                    # alternated windows, so both sides see the same clocks and neighbours
        b_ms.append(timed(lambda: bank(x, outs=outs)))
        s_ms.append(timed(lambda: [f(x, out=o) for f, o in zip(singles, outs)]))
    # per-pass split: passes 1-2 once for the bank, passes 3-5 per mask; each single filter's passes
    split_b = {p: timed(lambda p=p: bank.run_pass(p, x, outs)) for p in (1, 2)}
    for p in (3, 4, 5):
        split_b[p] = sum(timed(lambda p=p, i=i: bank.run_pass(p, x, outs, mask=i)) for i in range(n))
    split_s = [{p: timed(lambda p=p, f=f, o=o: f.run_pass(p, x, o)) for p in range(1, 6)} for f, o in zip(singles, outs)]
    bank_ms, sep_ms = float(np.median(b_ms)), float(np.median(s_ms))
    p12 = float(np.mean([s[1] + s[2] for s in split_s]))
    line(nx=nx, ns=ns, masks=names, op=f"FkFilterBank of {n} masks", ms=round(bank_ms, 3),
         ms_rounds=[round(v, 3) for v in b_ms], rows_kept=bank.rows_kept,
         pass_ms={f"p{p}": round(v, 3) for p, v in split_b.items()}, outputs_equal_single_filters=equal)
    line(nx=nx, ns=ns, masks=names, op=f"{n} separate FkFilter calls", ms=round(sep_ms, 3),
         ms_rounds=[round(v, 3) for v in s_ms], rows_kept=[f.rows_kept for f in singles],
         pass_ms=[{f"p{p}": round(v, 3) for p, v in s.items()} for s in split_s])
    line(nx=nx, ns=ns, op="bank saving vs (n - 1) x (P1 + P2)", saving_ms=round(sep_ms - bank_ms, 3),
         n_minus_1_p1_p2_ms=round((n - 1) * p12, 3), ratio=round((sep_ms - bank_ms) / max((n - 1) * p12, 1e-9), 3),
         bank_over_separate=round(bank_ms / sep_ms, 3))
    del x, bank, singles, outs, masks
    fk.free_plans()
    torch.cuda.empty_cache()
