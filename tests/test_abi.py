"""CPU: libd4w.so builds for sm_90a, loads, and exports every symbol include/d4w.h declares
(no compute calls -- there is no GPU here); the product path fails loudly without CUDA."""
import ctypes
import os

import pytest

from das4whales_b200 import _lib, _build


@pytest.fixture(scope="module")
def libpath():
    return _build.build_library()


def test_library_exports_every_declared_symbol(libpath):
    names = _lib.declared_symbols()
    assert len(names) >= 15 and "d4w_fk_apply" in names
    dll = ctypes.CDLL(libpath)
    missing = [n for n in names if not hasattr(dll, n)]
    assert not missing, f"symbols declared in include/d4w.h but not exported: {missing}"


def test_cffi_binding_parses_header_and_loads(libpath):
    L = _lib.lib()
    assert L.d4w_version() >= 100
    assert L.d4w_launch_count() >= 0
    assert isinstance(_lib.ffi.string(L.d4w_last_error()).decode(), str)


def test_no_cpu_fallback():
    """Without a CUDA device every op must raise, never silently compute on the host."""
    import numpy as np
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import das4whales_b200 as dw
    mask = dw.dsp.fk_filter_design((8, 16), [0, 8, 1], 2.0, 200.)
    with pytest.raises(RuntimeError):
        dw.dsp.fk_filter_filt(np.zeros((8, 16)), mask)
    with pytest.raises(RuntimeError):
        dw.detect.compute_cross_correlogram(np.zeros((2, 64)), np.ones(64))


def test_sass_is_sm90a(libpath):
    """The fat binary must contain sm_90a (H100) code only (no PTX-JIT or other-arch fallbacks)."""
    import shutil
    import subprocess
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([exe, "--list-elf", libpath], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert all("sm_90a" in line for line in out.splitlines() if "ELF file" in line)


def test_packaged_header_matches_canonical(libpath):
    """das4whales_b200/d4w.h (shipped with the package) must be byte-identical to include/d4w.h."""
    root = os.path.join(os.path.dirname(_lib.HERE), "include", "d4w.h")
    pkg = os.path.join(_lib.HERE, "d4w.h")
    assert os.path.exists(root) and os.path.exists(pkg)
    assert open(root, "rb").read() == open(pkg, "rb").read()
