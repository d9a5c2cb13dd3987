"""The pipelined two-level column kernel (k_col2_pipe, plan column scheme 3) at 10 000 channels: its launch settings
(CTAs per SM, V-ring slots) change how fast it runs, never what it computes."""
import numpy as np
import pytest

from conftest import rel_err

DX, FS = 2.0419046878814697, 200.0
FAN = (1400.0, 1450.0, 3400.0, 3500.0)


@pytest.mark.gpu
def test_col_pipe_launch_settings_bit_identical(monkeypatch):
    """Default settings (forward at 2 CTAs/SM, three ring slots beyond the lag) against the previous ones (3 CTAs/SM, two
    slots): bit-identical outputs, and both within the float64 filter's tolerance.  1 200 sample pairs are 15 chunks,
    so every ring slot is re-used."""
    import torch
    import das4whales_b200 as dw
    from das4whales_b200 import fk
    from oracle import dsp_oracle as O
    nx, ns = 10000, 2400
    rng = np.random.default_rng(21)
    x64 = rng.standard_normal((nx, ns))
    x = torch.from_numpy(x64.astype(np.float32)).cuda()
    mask = dw.dsp.fk_filter_design((nx, ns), [0, nx, 1], DX, FS, *FAN)
    outs = []
    try:
        for env in ({}, {"D4W_PIPE_OCC": "3", "D4W_PIPE_SLACK": "2"}):
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            fk.free_plans()                      # the ring size is fixed when the plan is made
            flt = fk.FkFilter(mask)
            assert flt.plan.col_scheme == 3
            outs.append(flt(x).cpu().numpy())
            del flt
    finally:
        monkeypatch.delenv("D4W_PIPE_OCC", raising=False)
        monkeypatch.delenv("D4W_PIPE_SLACK", raising=False)
        fk.free_plans()
    assert np.array_equal(outs[0], outs[1])
    ref = O.fk_filter_filt(x.cpu().numpy().astype(np.float64), O.fk_filter_design((nx, ns), [0, nx, 1], DX, FS, *FAN))
    mx, l2 = rel_err(outs[0], ref)
    assert mx <= 1e-4 and l2 <= 1e-5, (mx, l2)
