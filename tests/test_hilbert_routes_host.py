"""CPU guard for the GPU route tables of the Hilbert rows: the host planner (tests/host_emul/row_czt_emul.cu, the same
227 KB shared-memory cap as an H100) still splits every length of test_hilbert_routes_gpu.DIRECT_ROUTES and
test_hilbert_czt_gpu.LENGTHS as the tables say, and the tables reach every split radix row_plan.hpp's with_t1 is built
for and the device code of the generic prime stages.  A radix added to with_t1 without a GPU case fails here."""
import os
import re

import pytest

from conftest import ROOT
from test_hilbert_czt_gpu import LENGTHS, SPLIT_T1
from test_hilbert_czt_host import NVCC, _compile, _plans
from test_hilbert_routes_gpu import DIRECT_ROUTES

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _compile(tmp_path_factory, "row_czt_emul")


def _with_t1_radices():
    src = open(os.path.join(ROOT, "das4whales_b200", "csrc", "row_plan.hpp")).read()
    body = re.search(r"int with_t1\(.*?\n\}", src, re.S).group(0)
    radices = {int(r) for r in re.findall(r"case (\d+):", body)}
    assert radices
    return radices


def _generic_primes(n):
    """prime factors of n that the FFT engine runs through its generic stage (7..61)"""
    out = set()
    for p in range(2, 62):
        while n % p == 0:
            n //= p
            if p >= 7:
                out.add(p)
    return out


def test_tables_are_the_planners_routes(exe):
    p = _plans(exe, [n for n, _, _ in DIRECT_ROUTES] + LENGTHS)
    for n, t1, t2 in DIRECT_ROUTES:
        assert p[n] == ("direct", f"{t1} {t2}"), (n, p[n])
    for n in LENGTHS:
        kind, rest = p[n]
        assert kind == "czt", (n, p[n])
        m, t1, t2, _ = (int(v) for v in rest.split())
        assert t1 == SPLIT_T1.get(n, 1) and t1 * t2 == m, (n, p[n])


def test_tables_cover_every_route():
    radices = _with_t1_radices()
    assert {t1 for _, t1, _ in DIRECT_ROUTES} >= radices | {1}
    # chirp-z T1 = 2 is rare: M / 2 <= 10 240 < 16 384 < M leaves only the 5-smooth M in (16 384, 20 480], e.g.
    # n = 8 439 .. 8 640 -> M = 17 280
    assert set(SPLIT_T1.values()) >= radices
    assert set(SPLIT_T1) <= set(LENGTHS)
    # the device branch of stage_generic: whole rows and split T2s with generic prime factors, two distinct ones included
    assert any(_generic_primes(n) for n, t1, _ in DIRECT_ROUTES if t1 == 1)
    assert any(_generic_primes(t2) for _, t1, t2 in DIRECT_ROUTES if t1 > 1)
    assert any(len(_generic_primes(t2)) >= 2 for _, t1, t2 in DIRECT_ROUTES if t1 > 1)
