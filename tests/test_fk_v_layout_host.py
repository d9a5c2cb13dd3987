"""CPU: the two-level column bodies with ragged last time chunks (fewer sample pairs than the chunk width) and chunk
rows whose length is not a multiple of 8 pairs, run by the host emulation of the f-k passes and checked against the
float64 filter.  Inside each 8-pair group of a chunk row the intermediate V keeps the even sample pairs in the first
half and the odd pairs in the second (pairs past the last whole group stay in place), so a level A and a level B that
disagree on a position fail here."""
import numpy as np

from oracle import dsp_oracle as O
from conftest import rel_err
from test_host_emul import DX, FS, _build, _run, pytestmark  # noqa: F401  (nvcc skip marker)

# (nx, ns, planner settings, column scheme code of the emulator: 1000 * (1 + fused radix A) + X1)
CASES = [
    (10000, 56, {"D4W_COL_CHUNK_PAIRS": "16"}, 21025),     # 28 pairs: 16 + 12, the last tile 4 of 8 pairs; fused 20 x 20
    (10000, 44, {"D4W_COL_CHUNK_PAIRS": "16", "D4W_COLB_FUSED": "0"}, 1025),   # 22 pairs: 16 + 6; smem level B
    (20000, 36, {"D4W_COL_CHUNK_PAIRS": "8"}, 1025),       # X2 = 800, 4-pair tiles: 18 pairs = 8 + 8 + 2
    (10000, 52, None, 21025),                              # one 26-pair chunk: pairs 24, 25 past the last whole group
]


def test_fk_two_level_ragged_chunks_emulation(tmp_path):
    tmp = str(tmp_path)
    exe = _build("fk_pipeline_emul", tmp)
    rng = np.random.default_rng(7)
    c = (1400., 1450., 3400., 3500.)
    for nx, ns, env, scheme in CASES:
        x32 = rng.standard_normal((nx, ns)).astype(np.float32)
        kval, fval = 1.0 / (nx * DX), 1.0 / (ns * (1 / FS))
        M = O.fk_filter_design((nx, ns), [0, nx, 1], DX, FS, *c)
        ref = O.fk_filter_filt(x32.astype(np.float64), M, tapering=True)
        y, tail = _run(exe, tmp, nx, ns, 0, True, x32, kval, fval, c, env=env)
        assert tail[4] == scheme, (nx, ns, tail)
        assert rel_err(y, ref)[0] <= 5e-6, (nx, ns, env)
