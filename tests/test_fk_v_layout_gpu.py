"""The two-level column passes with a ragged last time chunk, on the GPU.  Inside each 8-pair group of a chunk row of
the intermediate V, level A stores the even sample pairs in the first half and the odd pairs in the second; every
level-B body reads them back from there, and a last chunk shorter than the others uses the same positions."""
import numpy as np
import pytest

from conftest import rel_err

DX, FS = 2.0419046878814697, 200.0
FAN = (1400.0, 1450.0, 3400.0, 3500.0)


def _filter(monkeypatch, x, nx, ns, env, scheme):
    import das4whales_b200 as dw
    from das4whales_b200 import fk
    mask = dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS, *FAN)
    try:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        fk.free_plans()                          # the column scheme and the chunk width are fixed when the plan is made
        flt = fk.FkFilter(mask)
        assert flt.plan.col_scheme == scheme, flt.plan.col_scheme
        y = flt(x).cpu().numpy()
        del flt
    finally:
        for k in env:
            monkeypatch.delenv(k, raising=False)
        fk.free_plans()
    return y


def _reference(x, nx, ns):
    from oracle import dsp_oracle as O
    return O.fk_filter_filt(x.cpu().numpy().astype(np.float64), O.fk_filter_design((nx, ns), [0, nx, 1], DX, FS, *FAN))


@pytest.mark.gpu
def test_col_pipe_ragged_chunk_matches_separate_launches(monkeypatch):
    """10 000 channels, ns = 2 480: 1 240 sample pairs are fifteen 80-pair chunks and a 40-pair one, so the pipelined
    kernel (column scheme 3) re-uses every ring slot and ends on a ragged chunk.  The separate level-A / level-B
    launches (scheme 2, 256-pair chunks, also ragged at the end) run the same bodies with plain loads and stores: the
    two must agree bit for bit, and both with the float64 filter."""
    import torch
    nx, ns = 10000, 2480
    rng = np.random.default_rng(31)
    x = torch.from_numpy(rng.standard_normal((nx, ns)).astype(np.float32)).cuda()
    y_pipe = _filter(monkeypatch, x, nx, ns, {}, 3)
    y_sep = _filter(monkeypatch, x, nx, ns, {"D4W_COL_PIPE": "0"}, 2)
    assert np.array_equal(y_pipe, y_sep)
    mx, l2 = rel_err(y_pipe, _reference(x, nx, ns))
    assert mx <= 1e-4 and l2 <= 1e-5, (mx, l2)


@pytest.mark.gpu
def test_col_two_level_four_pair_tiles_ragged_chunk(monkeypatch):
    """20 000 channels: X2 = 800 takes 4-pair level-B tiles and the shared-memory level B in separate launches.
    ns = 2 460 is 1 230 sample pairs: four 256-pair chunks and a 206-pair one whose last tile is half full."""
    import torch
    nx, ns = 20000, 2460
    rng = np.random.default_rng(32)
    x = torch.from_numpy(rng.standard_normal((nx, ns)).astype(np.float32)).cuda()
    y = _filter(monkeypatch, x, nx, ns, {}, 2)
    mx, l2 = rel_err(y, _reference(x, nx, ns))
    assert mx <= 1e-4 and l2 <= 1e-5, (mx, l2)
