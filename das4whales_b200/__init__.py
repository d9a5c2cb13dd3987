"""das4whales_b200 -- H100-native (sm_90a) implementation of the DAS4Whales channel-parallel
DSP hot path: f-k filter, band-pass, spectrogram, matched-filter / spectrogram correlators.

    import das4whales_b200 as dw
    mask = dw.dsp.fk_filter_design(tr.shape, selected_channels, dx, fs)
    trf  = dw.dsp.fk_filter_filt(tr, mask)

keeps the `das4whales.dsp` / `das4whales.detect` signatures (reference:
/root/reference/src/das4whales/{dsp,detect}.py).  Everything numeric runs in libd4w.so
(hand-written CUDA behind the C ABI of include/d4w.h); there is no CPU fallback.
"""
__version__ = "0.1.0"

from . import dsp, detect, fk, data_handle, improcess  # noqa: F401
from ._build import build_library  # noqa: F401
