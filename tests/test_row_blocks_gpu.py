"""GPU tests of the row blocks of libd4w.so: the row kernels put one row (or row pair) on each blockIdx.y, so a launch takes at
most 65 535 of them, and every row entry point splits a larger call into blocks itself.  Each entry point is called once
through the C ABI on rows that span more than one block, and its result must equal, bit for bit, the same entry point
called block by block; the launch counter must show one set of launches per block.  The rows at the block edges are
made distinctive (a zero row, a spike) so that a block offset by a row would show."""
import numpy as np
import pytest
import scipy.signal as sps

pytestmark = pytest.mark.gpu
BLOCK = 65535               # rows per launch (csrc/d4w_common.hpp, kMaxGridRows)


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available()
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _L():
    from das4whales_b200 import _lib
    return _lib, _lib.lib()


def _rows(nx, ns, seed, zero=BLOCK - 1, spike=BLOCK):
    """float32 CUDA [nx, ns] of noise with a zero row and a spike row at the edge of the first block"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((nx, ns), device="cuda", generator=g)
    if zero is not None:
        x[zero] = 0.0
    if spike is not None:
        x[spike] = 0.0
        x[spike, ns // 3] = 50.0
    return x


def _same_as_blocks(run, nx, launches_per_block, block=BLOCK):
    """run(r0, r1) -> a tensor whose first dimension is rows r0 .. r1 - 1: one call on every row equals the calls on each
    block, and takes launches_per_block launches per block"""
    import torch
    _, L = _L()
    n0 = L.d4w_launch_count()
    whole = run(0, nx)
    blocks = [(r0, min(nx, r0 + block)) for r0 in range(0, nx, block)]
    assert len(blocks) >= 2
    assert L.d4w_launch_count() - n0 == launches_per_block * len(blocks)
    for r0, r1 in blocks:
        assert torch.equal(whole[r0:r1], run(r0, r1)), (r0, r1)


def _tabs(plan, taps, nb):
    """conj(FFT_nb(c)) / nb of each template in the plan's table order, complex64 CUDA"""
    import torch
    t = np.stack([(np.conj(np.fft.fft(c, nb)) / nb)[plan.tab2freq] for c in taps]).astype(np.complex64)
    return torch.from_numpy(t.view(np.float32)).cuda()


def test_xcorr(dw):
    """normalised matched filter, two templates: the template stride of the output is the whole call's"""
    import torch
    lib, L = _L()
    nx, ns = 65537, 300
    x = _rows(nx, ns, 1, zero=None)
    x[BLOCK - 1] += 3.0                                              # a row far from zero mean next to the spike row
    taps = [np.hanning(40) - 0.3, np.sin(np.arange(60) / 5.0)]
    nb = dw.rows._pick_block(60, ns)
    valid = nb - 60 + 1
    plan = dw.rows.fft_plan(nb, 0)
    tabs = _tabs(plan, taps, nb)
    mu = torch.tensor([0.01, -0.02], dtype=torch.float64, device="cuda")
    stats, segpre = dw.rows.row_stats(x, seglen=valid)

    def run(r0, r1):
        out = torch.empty((2, r1 - r0, ns), dtype=torch.float32, device="cuda")
        lib.check(L.d4w_xcorr(plan.ptr, lib.ptr(x[r0:r1], "float*"), r1 - r0, ns, valid, 2, lib.ptr(tabs), lib.ptr(mu, "double*"),
                              lib.ptr(stats[r0:r1], "double*"), lib.ptr(segpre[r0:r1], "double*"), lib.ptr(out, "float*"),
                              lib.stream_ptr()), "xcorr")
        return out.transpose(0, 1)
    _same_as_blocks(run, nx, 1)


def test_xcorr_same(dw):
    import torch
    lib, L = _L()
    nx, ns = 65537, 300
    x = _rows(nx, ns, 2)
    _, lag0, nb, valid, spec = dw.rows.same_mode_layout([np.hanning(41), np.hanning(80)], ns)
    plan = dw.rows.fft_plan(nb, 0)
    tabs = torch.from_numpy(np.ascontiguousarray(spec[:, plan.tab2freq], dtype=np.complex64).view(np.float32)).cuda()
    rowmax = dw.rows.row_max(x)

    def run(r0, r1):
        out = torch.empty((2, r1 - r0, ns), dtype=torch.float32, device="cuda")
        lib.check(L.d4w_xcorr_same(plan.ptr, lib.ptr(x[r0:r1], "float*"), r1 - r0, ns, valid, lag0, 2, lib.ptr(tabs),
                                   lib.ptr(rowmax[r0:r1], "float*"), lib.ptr(out, "float*"), lib.stream_ptr()), "xcorr_same")
        return out.transpose(0, 1)
    _same_as_blocks(run, nx, 1)


# split Hilbert rows: 131 072 rows are one block of 2 x 65 535 rows (65 535 row pairs) and one of 2 rows
@pytest.mark.parametrize("ns,route,launches", [(16445, (5, 0), 3), (8193, (3, 1), 5)], ids=["direct", "chirp_z"])
def test_hilbert_split_rows(dw, ns, route, launches):
    import torch
    lib, L = _L()
    nx = 131072
    plan = dw.rows.row_plan(ns, 0)
    t1, _, m = plan.info()
    assert (t1, int(m > 0)) == route
    ws_bytes = int(L.d4w_row_workspace_bytes(plan.ptr, nx))
    assert ws_bytes == int(L.d4w_row_workspace_bytes(plan.ptr, 2 * BLOCK))
    need = 4 * nx * ns * 3 + ws_bytes                               # x, the whole call's and one block's output, workspace
    free = torch.cuda.mem_get_info()[0]
    if free < need + (1 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    x = _rows(nx, ns, 3, zero=None, spike=2 * BLOCK)
    x[2 * BLOCK - 1] *= 1e-3                                         # a quiet row paired with a loud one
    x[2 * BLOCK - 2, ns // 2] += 80.0
    stats, _ = dw.rows.row_stats(x)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    whole = torch.empty_like(x)
    part = torch.empty_like(x[:2 * BLOCK])

    def run(r0, r1):
        out = whole if (r0, r1) == (0, nx) else part[:r1 - r0]
        lib.check(L.d4w_hilbert(plan.ptr, lib.ptr(x[r0:r1], "float*"), lib.ptr(out, "float*"), r1 - r0, lib.ptr(ws),
                                3, lib.ptr(stats[r0:r1], "double*"), lib.stream_ptr()), "hilbert")
        return out
    _same_as_blocks(run, nx, launches, block=2 * BLOCK)


def test_stft(dw):
    """the sliding-DFT and the frame-by-frame STFT"""
    import torch
    lib, L = _L()
    nx, ns = 65537, 400
    x = _rows(nx, ns, 4)
    slide, frames = dw.rows.fft_plan(256, 0), dw.rows.fft_plan(64, 0)
    assert L.d4w_stft_slide_supported(256, 16, 11)
    win = torch.from_numpy(sps.get_window("hann", 64, fftbins=True).astype(np.float32)).cuda()

    def run_slide(r0, r1):
        out = torch.empty((r1 - r0, 11, 1 + ns // 16), dtype=torch.float32, device="cuda")
        lib.check(L.d4w_stft_slide(slide.ptr, lib.ptr(x[r0:r1], "float*"), lib.ptr(out, "float*"), r1 - r0, ns, 16, 10, 20,
                                   lib.stream_ptr()), "stft_slide")
        return out

    def run_frames(r0, r1):
        out = torch.empty((r1 - r0, 33, 1 + ns // 16), dtype=torch.float32, device="cuda")
        lib.check(L.d4w_stft_mag(frames.ptr, lib.ptr(x[r0:r1], "float*"), lib.ptr(out, "float*"), r1 - r0, ns, 16,
                                 lib.ptr(win, "float*"), 0, 32, lib.stream_ptr()), "stft_mag")
        return out
    _same_as_blocks(run_slide, nx, 1)
    _same_as_blocks(run_frames, nx, 1)


def test_speccorr(dw):
    """one kernel (d4w_speccorr); two tiled kernels in one pass, and a kernel too wide for the tile that goes through a
    dense copy of its band (d4w_speccorr_multi)"""
    import torch
    lib, L = _L()
    ffi = lib.ffi
    nx, nf, nt = 65537, 6, 64
    S = _rows(nx, nf * nt, 5).abs().reshape(nx, nf, nt).contiguous()
    med = torch.rand(nx, device="cuda") + 0.5
    g = np.random.default_rng(5)
    kers = [torch.from_numpy(g.standard_normal(s).astype(np.float32)).cuda() for s in ((nf, 7), (3, 5), (2, 9), (1, 14000))]

    def run_one(r0, r1):
        out = torch.empty((r1 - r0, nt), dtype=torch.float32, device="cuda")
        lib.check(L.d4w_speccorr(lib.ptr(S[r0:r1], "float*"), r1 - r0, nf, nt, lib.ptr(kers[0], "float*"), 7,
                                 lib.ptr(med[r0:r1], "float*"), lib.ptr(out, "float*"), lib.stream_ptr()), "speccorr")
        return out

    def multi(ks, f0):
        def run(r0, r1):
            outs = torch.empty((len(ks), r1 - r0, nt), dtype=torch.float32, device="cuda")
            lib.check(L.d4w_speccorr_multi(lib.ptr(S[r0:r1], "float*"), r1 - r0, nf, nt, len(ks), ffi.new("int[]", f0),
                                           ffi.new("int[]", [k.shape[0] for k in ks]),
                                           ffi.new("float*[]", [lib.ptr(k, "float*") for k in ks]),
                                           ffi.new("int[]", [k.shape[1] for k in ks]),
                                           ffi.new("float*[]", [lib.ptr(med[r0:r1], "float*")] * len(ks)),
                                           ffi.new("float*[]", [lib.ptr(o, "float*") for o in outs]), lib.stream_ptr()),
                      "speccorr_multi")
            return outs.transpose(0, 1)
        return run
    _same_as_blocks(run_one, nx, 1)
    _same_as_blocks(multi(kers[1:3], [1, 4]), nx, 1)
    _same_as_blocks(multi(kers[3:], [2]), nx, 1)


def test_find_peaks(dw):
    """the workspace holds one block of rows; flags are cleared for every row"""
    import torch
    lib, L = _L()
    nx, ns = 65537, 300
    x = _rows(nx, ns, 6)
    ws_bytes = int(L.d4w_find_peaks_workspace_bytes(nx, ns))
    assert ws_bytes == int(L.d4w_find_peaks_workspace_bytes(BLOCK, ns))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")

    def run(r0, r1):
        flags = torch.ones((r1 - r0, ns), dtype=torch.uint8, device="cuda")
        lib.check(L.d4w_find_peaks(lib.ptr(x[r0:r1], "float*"), r1 - r0, ns, 0.5, lib.ffi.cast("unsigned char*", flags.data_ptr()),
                                   lib.ptr(ws), lib.stream_ptr()), "find_peaks")
        return flags
    _same_as_blocks(run, nx, 2)


def test_detrend_linear(dw):
    """rows of a strided view (ld > n)"""
    import torch
    lib, L = _L()
    nx, n, ld = 65537, 64, 80
    X = _rows(nx, ld, 7)
    X[BLOCK - 2] += torch.arange(ld, device="cuda") * 0.5                # a pure trend next to the zero row
    x = X[:, :n]
    mom = dw.rows.row_moments(x)

    def run(r0, r1):
        out = torch.empty((r1 - r0, n), dtype=torch.float32, device="cuda")
        lib.check(L.d4w_detrend_linear(lib.ptr(x[r0:r1], "float*"), ld, r1 - r0, n, lib.ptr(mom[r0:r1], "double*"),
                                       lib.ptr(out, "float*"), lib.stream_ptr()), "detrend_linear")
        return out
    _same_as_blocks(run, nx, 1)


def test_env_stats(dw):
    """a window read in place from rows of a wider matrix: row statistics, envelope, its statistics, its median and the
    record per block"""
    import torch
    lib, L = _L()
    nx, n, ld, t0 = 65537, 64, 80, 8
    X = _rows(nx, ld, 8, zero=BLOCK - 1, spike=BLOCK)
    plan = dw.rows.row_plan(n, 0)
    ws_bytes = int(L.d4w_env_stats_workspace_bytes(plan.ptr, nx, ld))
    assert ws_bytes == int(L.d4w_env_stats_workspace_bytes(plan.ptr, BLOCK, ld))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")

    def run(r0, r1):
        out = torch.empty((r1 - r0, 5), dtype=torch.float64, device="cuda")
        lib.check(L.d4w_env_stats(plan.ptr, lib.ffi.cast("float*", X.data_ptr() + 4 * (r0 * ld + t0)), r1 - r0, ld,
                                  lib.ptr(out, "double*"), lib.ptr(ws), lib.stream_ptr()), "env_stats")
        return out
    _same_as_blocks(run, nx, 5)


def test_loc_grid(dw):
    """the grid-searched first guess of 65 537 calls"""
    import torch
    from das4whales_b200 import loc
    ncalls, nobs = 65537, 6
    g = np.random.default_rng(9)
    pos = np.zeros((ncalls * nobs, 3))
    pos[:, 0] = np.tile(np.linspace(0.0, 5000.0, nobs), ncalls)
    src = np.stack([g.uniform(0, 5000, ncalls), g.uniform(500, 3000, ncalls), np.full(ncalls, -40.0)], axis=1)
    T = np.linalg.norm(pos - np.repeat(src, nobs, axis=0), axis=1) / 1500.0 + np.repeat(g.uniform(0, 60, ncalls), nobs)
    Td, Pd = (torch.from_numpy(a).cuda() for a in (T, pos))
    off = torch.arange(0, (ncalls + 1) * nobs, nobs, dtype=torch.int64, device="cuda")
    axes = (np.linspace(0, 5000, 11), np.linspace(0, 3000, 7), np.array([-40.0]))

    def run(r0, r1):
        index, score, n0 = loc._grid(Td, Pd, off[r0:], r1 - r0, 1500.0, True, axes)
        return torch.cat([index.double()[:, None], score[:, None], n0], dim=1)
    _same_as_blocks(run, ncalls, 2)
