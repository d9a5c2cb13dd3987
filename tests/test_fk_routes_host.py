"""CPU guard for the f-k filter's route table: the host planner (build_fk_hostplan, compiled from
tests/host_emul/fk_route_probe.cu with an H100's 232 448 bytes of opt-in shared memory and no D4W_* variable set) still
plans every shape of ROUTES as the table says, and the routes that shapes reach by themselves are exactly REACHABLE.
tests/test_fk_routes_gpu.py runs one case per route on the device against float64; a planner change that moves a shape
to another kernel, or makes a new kernel reachable, fails here first.

KNOB_ONLY lists the column and row kernels that are built but that no shape reaches without a D4W_* environment
variable forcing them."""
import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from conftest import ROOT
from test_hilbert_czt_host import NVCC, _compile

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

FIELDS = ("scheme", "nc", "dual", "tma", "x1", "x2", "np", "ra", "rb", "pipe", "chunk_pairs", "t1", "row_fused",
          "col_threads")

# (nx, ns): scheme nc dual tma | X1 X2 np ra rb pipe chunk_pairs | T1 row_fused col_threads
# scheme is fk._Plan.col_scheme: 0 single-level (scalar when nc = 1, else dual cp.async), 1 single-level TMA, 2 two-level
# (level A in registers, level B in shared memory: the generic engine when ra = 0, else the fused ra x rb kernel),
# 3 pipelined two-level.  col_threads is the block size (and template) of the single-level column kernels.
ROUTES = {
    # scalar k_col_fwd / k_col_inv<512>: one column fits a tile, two do not, and no two-level split
    (13122, 1200): (0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),   # 2 x 3^8: no factor 16 / 20 / 25
    (15625, 1210): (0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),   # ns % 4 != 0 rules out the two-level split
    (20000, 1210): (0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),
    # dual cp.async k_col_fwd_dual / k_col_inv_dual
    (5510, 1200): (0, 4, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 256),    # 2 x 5 x 19 x 29: radix 19 / 29 stages
    (5510, 1210): (0, 4, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 256),
    (64, 400): (0, 8, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 512),
    (63, 405): (0, 8, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 512),
    # persistent TMA k_col_fwd_tma / k_col_inv_tma
    (6561, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),    # 3^8
    (7203, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),    # 3 x 7^4
    (6859, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 256),    # 19^3
    (8303, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 256),    # 19 x 19 x 23
    (8019, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),
    (9261, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),
    (12005, 1200): (1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 512),
    # two-level, shared-memory engine level B (k_colA_* + k_colB_fwd / k_colB_inv)
    (1024, 4096): (2, 8, 1, 0, 16, 64, 8, 0, 0, 0, 1536, 1, 0, 512),
    (11020, 1200): (2, 2, 1, 1, 20, 551, 4, 0, 0, 0, 256, 1, 0, 256),
    (6000, 1200): (2, 4, 1, 0, 25, 240, 8, 0, 0, 0, 256, 1, 0, 256),
    (20000, 1200): (2, 1, 0, 0, 25, 800, 4, 0, 0, 0, 256, 1, 0, 512),
    (25000, 1200): (2, 1, 0, 0, 25, 1000, 2, 0, 0, 0, 256, 1, 0, 512),
    (20000, 1920): (2, 1, 0, 0, 25, 800, 4, 0, 0, 0, 256, 1, 0, 512),
    # two-level, fused level B k_colB_fwd_fused / k_colB_inv_fused<ra, rb>
    (4096, 1200): (2, 4, 1, 0, 16, 256, 8, 16, 16, 0, 256, 1, 0, 512),
    (5120, 1200): (2, 4, 1, 0, 20, 256, 8, 16, 16, 0, 256, 1, 0, 256),
    (6400, 1200): (2, 2, 1, 1, 25, 256, 8, 16, 16, 0, 256, 1, 0, 256),
    (8000, 1200): (2, 2, 1, 1, 25, 320, 8, 20, 16, 0, 256, 1, 0, 256),
    (8000, 2400): (2, 2, 1, 1, 25, 320, 8, 20, 16, 0, 256, 1, 0, 256),
    (12500, 1200): (2, 2, 1, 1, 25, 500, 4, 20, 25, 0, 256, 1, 0, 256),
    (15625, 1200): (2, 1, 0, 0, 25, 625, 4, 25, 25, 0, 256, 1, 0, 512),
    # pipelined single launch k_col2_pipe<25, 20, 20>
    (10000, 2480): (3, 2, 1, 1, 25, 400, 8, 20, 20, 1, 80, 1, 0, 256),    # 1 240 pairs: the last 80-pair chunk is ragged
    (10000, 16400): (3, 2, 1, 1, 25, 400, 8, 20, 20, 1, 80, 2, 0, 256),   # time split T1 = 2 (T2 = 8 200)
    (10000, 30000): (3, 2, 1, 1, 25, 400, 8, 20, 20, 1, 80, 3, 1, 256),
    (10000, 2200): (3, 2, 1, 1, 25, 400, 8, 20, 20, 1, 80, 1, 0, 256),
}

# (scheme, dual, X1, ra, rb, pipe, column template) over every channel count 8 .. 28 000 at ns = 1 200 and 1 210.  dual
# and the template (col_threads) belong to the single-level schemes (0, 1, 4); the two-level ones launch no single-level
# column kernel and carry 0 for both.
SWEEP_NS = (1200, 1210)
SWEEP_NX = (8, 28000)
REACHABLE = {
    (0, 0, 0, 0, 0, 0, 512),        # scalar k_col_*<512>
    (0, 1, 0, 0, 0, 0, 256),        # dual k_col_*_dual<256> (a radix above 16)
    (0, 1, 0, 0, 0, 0, 512),        # dual k_col_*_dual<512>
    (1, 1, 0, 0, 0, 0, 256),        # k_col_*_tma<256>
    (1, 1, 0, 0, 0, 0, 512),        # k_col_*_tma<512>
    (2, 0, 16, 0, 0, 0, 0), (2, 0, 20, 0, 0, 0, 0), (2, 0, 25, 0, 0, 0, 0),      # two-level, shared-memory engine level B
    (2, 0, 16, 16, 16, 0, 0), (2, 0, 20, 16, 16, 0, 0), (2, 0, 25, 16, 16, 0, 0),   # fused (16, 16): nx 4096, 5120, 6400
    (2, 0, 25, 20, 16, 0, 0),       # fused (20, 16): nx 8000
    (2, 0, 25, 20, 25, 0, 0),       # fused (20, 25): nx 12500
    (2, 0, 25, 25, 25, 0, 0),       # fused (25, 25): nx 15625
    (3, 0, 25, 20, 20, 1, 0),       # pipelined k_col2_pipe<25, 20, 20>: nx 10000
    (4, 0, 0, 0, 0, 0, 512),        # chirp-z (tests/test_fk_czt_gpu.py)
}
REACHABLE_FUSED = {(16, 16), (20, 16), (20, 25), (25, 25), (20, 20)}
REACHABLE_PIPE = {(25, 20, 20)}

# Built, but reached only through an environment variable:
KNOB_ONLY = {
    "k_colB_fwd_fused / k_colB_inv_fused<16, 20>, <16, 25>, <25, 16>, <25, 20>":
        "D4W_COLB_RA: for X2 = 320, 400 and 500 the order {20, 16, 25} always takes ra = 20 first",
    "k_col2_pipe<X1, ra, rb> other than <25, 20, 20>":
        "D4W_COL_X1 / D4W_COLB_RA: a 400-point level B implies 25 | nx, and X1 = 25 wins",
    "k_col2_pipe<25, 20, 20, OCC = 4>": "D4W_PIPE_OCC=4",
    "k_col3_pipe (X1 = 10, three-stage level B)": "D4W_COL_PIPE3=1",
    "k_col_fwd_tma / k_col_inv_tma<416>": "D4W_COL_THREADS between 257 and 416",
    "k_col_fwd / k_col_inv<256> and <1024>": "D4W_COL_THREADS <= 256 or > 512 (the scalar kernels run 512 threads)",
    "k_row_mid_dual": "D4W_ROW_DUAL=1",
}
KNOB_ONLY_FUSED = {(16, 20), (16, 25), (25, 16), (25, 20)}
KNOB_ONLY_PIPE = {(25, 16, 25), (20, 20, 20), (20, 16, 25), (16, 20, 20), (16, 16, 25)}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _compile(tmp_path_factory, "fk_route_probe")


def _clean_env():
    return {k: v for k, v in os.environ.items() if not k.startswith("D4W_")}


def _parse(stdout):
    out = {}
    for line in stdout.splitlines():
        f = line.split()
        key = (int(f[0]), int(f[1]))
        out[key] = None if f[2] == "error" else tuple(int(v) for v in f[2:])
    return out


def _plan(exe, shapes):
    args = [str(v) for s in shapes for v in s]
    r = subprocess.run([exe, "plan"] + args, capture_output=True, text=True, check=True, env=_clean_env())
    return _parse(r.stdout)


def _sweep(exe, ns, lo, hi, parts=16):
    """Every nx in [lo, hi] at this ns, the range split over concurrent probe processes (chirp-z plans dominate)."""
    edges = [lo + (hi + 1 - lo) * i // parts for i in range(parts + 1)]

    def run(i):
        r = subprocess.run([exe, "sweep", str(ns), str(edges[i]), str(edges[i + 1] - 1)], capture_output=True, text=True,
                           check=True, env=_clean_env())
        return _parse(r.stdout)

    out = {}
    with ThreadPoolExecutor(max_workers=min(parts, os.cpu_count() or 1)) as pool:
        for part in pool.map(run, range(parts)):
            out.update(part)
    assert len(out) == hi + 1 - lo
    return out


def route_key(r):
    """(scheme, dual, X1, ra, rb, pipe, column template) of a probe route."""
    d = dict(zip(FIELDS, r))
    single = d["scheme"] in (0, 1, 4)
    return (d["scheme"], d["dual"] if single else 0, d["x1"], d["ra"], d["rb"], d["pipe"], d["col_threads"] if single else 0)


def test_routes_table_is_the_planners(exe):
    got = _plan(exe, list(ROUTES))
    for shape, want in ROUTES.items():
        assert got[shape] == want, (shape, dict(zip(FIELDS, got[shape] or ())), dict(zip(FIELDS, want)))


def test_sweep_reaches_exactly_the_documented_routes(exe):
    seen = {}
    for ns in SWEEP_NS:
        for (nx, _), r in _sweep(exe, ns, *SWEEP_NX).items():
            if r is not None:
                seen.setdefault(route_key(r), (nx, ns))
    assert set(seen) == REACHABLE, {"new": {k: seen[k] for k in set(seen) - REACHABLE}, "gone": REACHABLE - set(seen)}
    assert {(k[3], k[4]) for k in seen if k[3]} == REACHABLE_FUSED
    assert {(k[2], k[3], k[4]) for k in seen if k[5]} == REACHABLE_PIPE


def test_routes_table_covers_every_reachable_route_but_chirp_z():
    keys = {route_key(r) for r in ROUTES.values()}
    assert keys == {k for k in REACHABLE if k[0] != 4}


def test_knob_only_lists_are_the_built_complement():
    """The fused level-B pairs and pipelined splits the launchers are built for, minus the reachable ones, are the
    knob-only lists above."""
    src = open(os.path.join(ROOT, "das4whales_b200", "csrc", "d4w_fk.cu")).read()
    fused = {tuple(int(v) for v in m) for m in re.findall(r"D4W_FUSED\((\d+), (\d+)\)", src)}
    pipes = {tuple(int(v) for v in m) for m in re.findall(r"D4W_PIPE\((\d+), (\d+), (\d+)\)", src)}
    assert fused - REACHABLE_FUSED == KNOB_ONLY_FUSED and REACHABLE_FUSED <= fused
    assert pipes - REACHABLE_PIPE == KNOB_ONLY_PIPE and REACHABLE_PIPE <= pipes
