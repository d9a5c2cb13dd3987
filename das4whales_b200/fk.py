"""Host side of the f-k filter: mask descriptors (`FkMask`), per-shape plans and the reusable
`FkFilter` object that owns the device buffers.  dsp.fk_filter_design / hybrid_*_filter_design
return `FkMask`; dsp.fk_filter_filt / fk_filter_sparsefilt run an `FkFilter`; dsp.fk_spectrum runs an
`FkSpectrum` (the same forward transform, ending in |X|^2 over a band); dsp.fk_welch runs an `FkWelch`
(staged, detrended and windowed segments through an FkSpectrum, averaged over time).

All arithmetic happens in libd4w.so (hand-written sm_90a CUDA, see csrc/fk_kernels.cuh);
PyTorch is used for device memory and streams only.
"""
import threading
import weakref
from collections import namedtuple

import numpy as np

from . import _lib

_plan_cache = {}
_plan_lock = threading.Lock()
_plan_serial = [0]      # every _Plan gets a unique, never re-used serial (ids of freed objects can be re-used)


def _torch():
    import torch
    if not torch.cuda.is_available():
        raise _lib.D4WError("das4whales_b200 needs a CUDA device (no CPU fallback)")
    return torch


class _Plan:
    """d4w_fk_plan handle for one (nx, ns, device)."""

    def __init__(self, nx, ns, device):
        L = _lib.lib()
        out = _lib.ffi.new("d4w_fk_plan**")
        _lib.check(L.d4w_fk_plan_create(out, int(nx), int(ns), int(device)), f"fk plan {nx}x{ns}")
        self.ptr = out[0]
        # the C plan lives exactly as long as this object: device masks keep a strong reference to their plan, so a
        # d4w_fk_mask can never outlive the d4w_fk_plan it points to (free_plans() only empties the cache)
        weakref.finalize(self, L.d4w_fk_plan_destroy, self.ptr)
        with _plan_lock:
            _plan_serial[0] += 1
            self.serial = _plan_serial[0]
        self.nx, self.ns, self.device = int(nx), int(ns), int(device)
        info = _lib.ffi.new("int[8]")
        _lib.check(L.d4w_fk_plan_info(self.ptr, info), "fk plan info")
        self.t1, self.t2, self.tile, self.col_stages, self.row_stages = info[0], info[1], info[2], info[3], info[4]
        # column transform: 0 single-level, 1 single-level TMA, 2 two-level, 3 pipelined two-level, 4 chirp-z single-level
        self.col_scheme = int(info[7])
        self.col_threads = int(info[5])      # block size of the single-level column kernels
        self.workspace = None

    def get_workspace(self, nbytes):
        torch = _torch()
        if self.workspace is None or self.workspace.numel() < nbytes:
            self.workspace = None
            self.workspace = torch.empty(int(nbytes), dtype=torch.uint8, device=f"cuda:{self.device}")
        return self.workspace


def get_plan(nx, ns, device):
    key = (int(nx), int(ns), int(device))
    with _plan_lock:
        p = _plan_cache.get(key)
    if p is None:
        p = _Plan(*key)
        with _plan_lock:
            p = _plan_cache.setdefault(key, p)
    return p


def free_plans():
    """Empty the plan cache (and the dense-mask cache).  A plan (and its workspace) is destroyed when the last
    FkFilter / device mask that uses it is gone, so outstanding objects stay valid."""
    with _plan_lock:
        for p in _plan_cache.values():
            p.workspace = None
        _plan_cache.clear()
    _dense_cache.clear()


class _DeviceMask:
    """d4w_fk_mask handle + its transform-order table for one plan."""

    def __init__(self, plan, create, eps=0.0):
        torch = _torch()
        L = _lib.lib()
        self.plan = plan
        out = _lib.ffi.new("d4w_fk_mask**")
        with torch.cuda.device(plan.device):
            create(L, out, plan)
            self.ptr = out[0]
            if eps and eps > 0:
                _lib.check(L.d4w_fk_mask_prune(self.ptr, float(eps), _lib.stream_ptr()), "fk mask prune")
            self.rows = L.d4w_fk_mask_rows(self.ptr)
            nbytes = L.d4w_fk_mask_table_bytes(self.ptr)
            self.table = torch.empty(int(nbytes) // 4, dtype=torch.float32, device=f"cuda:{plan.device}")
            _lib.check(L.d4w_fk_mask_build(self.ptr, _lib.ptr(self.table, "float*"), _lib.stream_ptr()), "fk mask build")
            self.workspace_bytes = L.d4w_fk_workspace_bytes(plan.ptr, self.ptr)
        weakref.finalize(self, L.d4w_fk_mask_destroy, self.ptr)


# the masks designed on the device as a float32 plane (d4w_mask_design's kind codes); the filter takes them through the dense
# route, and todense() runs the host restatement the design function passed in
DESIGN_KINDS = {"hybrid": 0, "hybrid_gs": 1, "hybrid_ninf_gs": 2}


class FkMask:
    """Lazy f-k mask: the closed-form description of what the reference's design function
    returns.  `np.asarray(mask)` / `mask.todense()` materialise exactly the reference's
    [channel x time] float64 array (shifted layout) on demand; `fk_filter_filt` uses the
    description directly and never builds the dense matrix.  For the DESIGN_KINDS the filter's
    table comes from a plane designed on the device, and todense() runs the host design (`host`).
    """

    def __init__(self, kind, shape, params, order="C", host=None):
        self.kind = kind
        self.shape = (int(shape[0]), int(shape[1]))
        self.params = params
        self.order = order
        self.prune_eps = 0.0           # opt-in: FkFilter / fk_filter_filt drop rows whose folded mask never exceeds this
        self.ndim = 2
        self.dtype = np.dtype(np.float64)
        self._dev = {}
        self._dense = None
        self._host = host              # designed kinds: the host restatement todense() runs (and caches) on demand

    # ---- device side -------------------------------------------------------------------
    def _create(self, L, out, plan):
        p = self.params
        if self.kind == "fan":
            _lib.check(L.d4w_fk_mask_create_fan(out, plan.ptr, p["kval"], p["fval"], p["cs_min"], p["cp_min"],
                                                p["cp_max"], p["cs_max"]), "fan mask")
        elif self.kind == "hybrid_ninf":
            h = np.ascontiguousarray(p["H"], dtype=np.float64)
            _lib.check(L.d4w_fk_mask_create_hybrid_ninf(out, plan.ptr, p["kval"], p["fval"], p["cs_min"], p["cp_min"],
                                                        p["cp_max"], p["cs_max"],
                                                        _lib.ffi.cast("double*", h.ctypes.data), p["col_lo"], p["col_hi"]),
                       "hybrid_ninf mask")
        else:
            raise ValueError(f"unknown analytic mask kind {self.kind}")

    def _design_plane(self, plan):
        """float32 [nx, ns] device plane of a designed kind (d4w_mask_design), for the dense support scan and table."""
        if (plan.nx, plan.ns) != self.shape:
            raise ValueError(f"operands could not be broadcast together with shapes ({plan.nx},{plan.ns}) {self.shape}")
        torch = _torch()
        L = _lib.lib()
        p = self.params
        nx, ns = self.shape
        h = np.ascontiguousarray(p["H"], dtype=np.float64)
        with torch.cuda.device(plan.device):
            out = torch.empty((nx, ns), dtype=torch.float32, device=f"cuda:{plan.device}")
            ws = torch.empty(int(L.d4w_mask_design_workspace_bytes(nx, ns)), dtype=torch.uint8, device=f"cuda:{plan.device}")
            _lib.check(L.d4w_mask_design(DESIGN_KINDS[self.kind], _lib.ptr(out, "float*"), nx, ns, p["kval"], p["fval"],
                                         p["cs_min"], p["cp_min"], p["cp_max"], p["fmin"], p["fmax"], p["col_lo"], p["col_hi"],
                                         _lib.ffi.cast("double*", h.ctypes.data), _lib.ptr(ws), _lib.stream_ptr()),
                       f"{self.kind} mask design")
        return out

    def _new_device_mask(self, plan, eps=0.0):
        if self.kind == "dense":      # caller-supplied planes, and designs outside the device route's domain
            return _DenseMaskHolder(plan, _dense_to_device(self._dense, plan.device), eps).dm
        if self.kind in DESIGN_KINDS:  # designed into a transient plane on the device, then scanned like a dense mask
            return _DenseMaskHolder(plan, self._design_plane(plan), eps).dm
        return _DeviceMask(plan, self._create, eps)

    def on_device(self, plan, eps=0.0):
        eps = float(eps or 0.0)
        if eps:
            key = (plan.serial, eps)
            dm = self._dev.get(key)
            if dm is None:
                dm = self._new_device_mask(plan, eps)
                self._dev[key] = dm
            return dm
        dm = self._dev.get(plan.serial)
        if dm is None:
            for k in [k for k, v in self._dev.items() if _plan_cache.get((v.plan.nx, v.plan.ns, v.plan.device)) is not v.plan]:
                del self._dev[k]                      # tables of plans that were dropped by free_plans()
            if (plan.nx, plan.ns) != self.shape:
                raise ValueError(f"operands could not be broadcast together with shapes ({plan.nx},{plan.ns}) {self.shape}")
            dm = self._new_device_mask(plan)
            self._dev[plan.serial] = dm
        return dm

    @classmethod
    def from_dense(cls, array):
        """Wrap a dense [channel x time] mask (reference shifted layout) in the sparse.COO-like API."""
        a = np.asarray(array, dtype=np.float64)
        m = cls("dense", a.shape, {}, order="C")
        m._dense = a
        return m

    # ---- host side (what plots / prints see) -------------------------------------------
    def todense(self):
        if self._dense is None and self._host is not None:
            self._dense = self._host()
        if self._dense is None:
            torch = _torch()
            L = _lib.lib()
            dev = torch.cuda.current_device()
            plan = get_plan(self.shape[0], self.shape[1], dev)
            dm = self.on_device(plan)
            with torch.cuda.device(dev):
                out = torch.empty(self.shape, dtype=torch.float64, device=f"cuda:{dev}")
                _lib.check(L.d4w_fk_mask_materialize(dm.ptr, _lib.ptr(out, "double*"), _lib.stream_ptr()), "mask materialize")
                a = out.cpu().numpy()
            self._dense = np.asfortranarray(a) if self.order == "F" else a
        return self._dense

    def __array__(self, dtype=None, copy=None):
        a = self.todense()
        return a if dtype is None else a.astype(dtype, copy=False)

    def __getitem__(self, idx):
        return self.todense()[idx]

    @property
    def nnz(self):
        return int(np.count_nonzero(self.todense()))

    @property
    def data(self):
        """Non-zero values, like sparse.COO.data (the reference's tools.disp_comprate reads `.data.nbytes`, tools.py:248)."""
        d = self.todense()
        return d[d != 0]

    def __repr__(self):
        return f"<FkMask {self.kind} shape={self.shape}>"


class _DenseMaskHolder:
    """Device state for a caller-supplied dense mask (ndarray / sparse.COO / tensor)."""

    def __init__(self, plan, mask_dev, eps=0.0):
        self.mask_dev = mask_dev      # float32 [nx, ns] shifted layout, kept alive for the support scan only

        def create(L, out, plan_):
            _lib.check(L.d4w_fk_mask_create_dense(out, plan_.ptr, _lib.ptr(mask_dev, "float*"), _lib.stream_ptr()),
                       "dense mask")
        self.dm = _DeviceMask(plan, create, eps)
        _torch().cuda.current_stream().synchronize()
        self.mask_dev = None          # the transform-order table is all the filter needs


_dense_cache = {}


def _dense_to_device(mask, device):
    torch = _torch()
    if isinstance(mask, torch.Tensor):
        return mask.to(device=f"cuda:{device}", dtype=torch.float32).contiguous()
    if hasattr(mask, "todense") and not isinstance(mask, np.ndarray):
        mask = mask.todense()
    m = np.asarray(mask)
    out = torch.empty(m.shape, dtype=torch.float32, device=f"cuda:{device}")
    # row-chunked upload keeps host temporaries small for very large masks
    step = max(1, (64 << 20) // max(1, m.shape[1] * 8))
    for r0 in range(0, m.shape[0], step):
        chunk = np.ascontiguousarray(m[r0:r0 + step])
        out[r0:r0 + step] = torch.from_numpy(chunk).to(f"cuda:{device}").to(torch.float32)
    return out


def _fingerprint(mask):
    """Cheap content fingerprint of a caller-owned dense mask: the cached device table is only re-used while the
    array still holds the values it was built from (callers may refill / scale a mask array in place)."""
    torch = _torch()
    if isinstance(mask, torch.Tensor):
        flat = mask.reshape(-1)
        n = flat.numel()
        step = max(1, n // 65536) | 1
        samp = flat[::step].to(torch.float64)
        return ("t", tuple(mask.shape), str(mask.dtype), int(mask.data_ptr()), int(mask._version),
                float(samp.sum().item()), float((samp * samp).sum().item()))
    if isinstance(mask, np.ndarray):
        n = mask.size
        step = max(1, n // 65536) | 1
        samp = np.asarray(mask.reshape(-1, order="A")[::step], dtype=np.float64) if (mask.flags.c_contiguous or mask.flags.f_contiguous) \
            else np.asarray(mask[::max(1, mask.shape[0] // 64)], dtype=np.float64).ravel()
        return ("n", mask.shape, mask.dtype.str, mask.__array_interface__["data"][0], mask.strides,
                float(samp.sum()), float(np.dot(samp, samp)))
    data = getattr(mask, "data", None)           # sparse.COO: fingerprint the stored values
    if isinstance(data, np.ndarray):
        return ("s", tuple(mask.shape), data.size, float(np.sum(data[::max(1, data.size // 65536) | 1], dtype=np.float64)))
    return None


def device_mask_for(mask, plan, eps=0.0):
    """Resolve any accepted mask object to a _DeviceMask for `plan`."""
    if isinstance(mask, FkMask):
        return mask.on_device(plan, eps if eps else getattr(mask, "prune_eps", 0.0))
    if eps:
        return _DenseMaskHolder(plan, _dense_to_device(mask, plan.device), float(eps)).dm
    shape = tuple(getattr(mask, "shape", ()))
    if shape != (plan.nx, plan.ns):
        raise ValueError(f"operands could not be broadcast together with shapes ({plan.nx},{plan.ns}) {shape}")
    key = (id(mask), plan.serial)
    fp = _fingerprint(mask)
    hit = _dense_cache.get(key)
    if hit is not None and fp is not None and hit[0]() is mask and hit[2] == fp:
        return hit[1].dm
    holder = _DenseMaskHolder(plan, _dense_to_device(mask, plan.device))
    if fp is not None:
        try:
            ref = weakref.ref(mask, lambda _r, k=key: _dense_cache.pop(k, None))
            _dense_cache[key] = (ref, holder, fp)
        except TypeError:
            pass
    return holder.dm


def _misaligned(t, ns):
    """True when t does not start on the boundary d4w_fk_apply needs for rows of ns samples (16 bytes when ns % 4 == 0,
    8 when ns is even): a contiguous view that starts inside its allocation, such as buf[1:].view(nx, ns)."""
    align = 16 if ns % 4 == 0 else 8 if ns % 2 == 0 else 4
    return t.data_ptr() % align != 0


class FkFilter:
    """Reusable f-k filter for one matrix shape: plan + mask table + workspace on one GPU.

    >>> flt = FkFilter(mask, device=0)          # mask: FkMask / ndarray / sparse.COO
    >>> y = flt(x_cuda)                         # x_cuda: float32 CUDA tensor [nx, ns]
    """

    def __init__(self, mask, shape=None, device=None, eps=0.0):
        """eps > 0: opt-in approximate support pruning (d4w_fk_mask_prune): wavenumber rows whose folded mask never
        exceeds eps are dropped; l2 error <= eps * ||x||.  A mask object may also carry the setting as `mask.prune_eps`."""
        torch = _torch()
        self.device = torch.cuda.current_device() if device is None else int(device)
        shape = tuple(shape) if shape is not None else tuple(mask.shape)
        self.plan = get_plan(shape[0], shape[1], self.device)
        with torch.cuda.device(self.device):
            self.dm = device_mask_for(mask, self.plan, eps)
        self.mask = mask
        self.rows_kept = self.dm.rows

    def _ws(self):
        return self.plan.get_workspace(self.dm.workspace_bytes)

    def __call__(self, x, out=None, tapering=False):
        torch = _torch()
        if x.dtype != torch.float32 or not x.is_cuda or not x.is_contiguous():
            raise ValueError("FkFilter expects a contiguous float32 CUDA tensor")
        if tuple(x.shape) != (self.plan.nx, self.plan.ns):
            raise ValueError(f"FkFilter built for {(self.plan.nx, self.plan.ns)}, got {tuple(x.shape)}")
        ns = self.plan.ns
        xin = x.clone() if _misaligned(x, ns) else x          # a misaligned matrix goes through an aligned copy
        y = torch.empty_like(x) if out is None or _misaligned(out, ns) else out
        L = _lib.lib()
        with torch.cuda.device(self.device):
            _lib.check(L.d4w_fk_apply(self.plan.ptr, self.dm.ptr, _lib.ptr(xin, "float*"), _lib.ptr(y, "float*"),
                                      _lib.ptr(self._ws()), int(bool(tapering)), _lib.stream_ptr()), "fk_filter_filt")
        if out is not None and y is not out:
            out.copy_(y)
            return out
        return y

    def run_pass(self, i, x, out, tapering=False):
        """Launch pass i (1..5) alone -- profiling / per-kernel timing."""
        L = _lib.lib()
        torch = _torch()
        with torch.cuda.device(self.device):
            _lib.check(L.d4w_fk_apply_pass(self.plan.ptr, self.dm.ptr, _lib.ptr(x, "float*"), _lib.ptr(out, "float*"),
                                           _lib.ptr(self._ws()), int(bool(tapering)), int(i), _lib.stream_ptr()),
                       f"fk pass {i}")

    def traffic_bytes(self):
        """Actual HBM bytes each pass must move (for the per-kernel bandwidth report)."""
        return _traffic_bytes(self.plan, self.rows_kept)


def _traffic_bytes(plan, r, nmasks=1):
    nx, ns = plan.nx, plan.ns
    real, spec = nx * ns * 4, r * ns * 8
    split = 2 * spec if plan.t1 > 1 else 0
    return {"p1_col_fwd": real + spec, "p2_row_split": split, "p3_row_mid": nmasks * (2 * spec + r * ns * 4),
            "p4_row_unsplit": nmasks * split, "p5_col_inv": nmasks * (spec + real)}


def _destroy_bank(lib, ptr, dms):
    """Destroy a d4w_fk_bank; `dms` holds its masks (and their tables) until the bank is gone."""
    lib.d4w_fk_bank_destroy(ptr)


class FkFilterBank:
    """Several f-k masks over one matrix shape, sharing one forward transform (d4w_fk_bank).

    >>> bank = FkFilterBank([m1, m2, m3], device=0)   # masks: anything FkFilter accepts
    >>> y1, y2, y3 = bank(x_cuda)                       # each equal to FkFilter(m_i)(x_cuda)

    The rows filtered are the union of the masks' kept wavenumber rows (`rows_kept`); a mask is exactly zero on the
    rows it does not keep, so each output equals the single-mask filter's.  `eps` / `mask.prune_eps` prune each mask
    as FkFilter does."""

    def __init__(self, masks, shape=None, device=None, eps=0.0):
        torch = _torch()
        masks = list(masks)
        if not masks:
            raise ValueError("FkFilterBank needs at least one mask")
        self.device = torch.cuda.current_device() if device is None else int(device)
        shape = tuple(shape) if shape is not None else tuple(masks[0].shape)
        self.plan = get_plan(shape[0], shape[1], self.device)
        L = _lib.lib()
        out = _lib.ffi.new("d4w_fk_bank**")
        with torch.cuda.device(self.device):
            self.dms = [device_mask_for(m, self.plan, eps) for m in masks]
            arr = _lib.ffi.new("d4w_fk_mask*[]", [dm.ptr for dm in self.dms])
            _lib.check(L.d4w_fk_bank_create(out, self.plan.ptr, arr, len(self.dms)), "fk bank")
            self.ptr = out[0]
            weakref.finalize(self, _destroy_bank, L, self.ptr, self.dms)
            self.rows_kept = L.d4w_fk_bank_rows(self.ptr)
            nbytes = L.d4w_fk_bank_table_bytes(self.ptr)
            self.table = torch.empty(int(nbytes) // 4, dtype=torch.float32, device=f"cuda:{self.device}")
            _lib.check(L.d4w_fk_bank_build(self.ptr, _lib.ptr(self.table, "float*"), _lib.stream_ptr()), "fk bank build")
            self.workspace_bytes = L.d4w_fk_bank_workspace_bytes(self.plan.ptr, self.ptr)
        self.masks = masks

    def __len__(self):
        return len(self.dms)

    def _ws(self):
        return self.plan.get_workspace(self.workspace_bytes)

    def _outs(self, x, outs):
        torch = _torch()
        if x.dtype != torch.float32 or not x.is_cuda or not x.is_contiguous():
            raise ValueError("FkFilterBank expects a contiguous float32 CUDA tensor")
        if tuple(x.shape) != (self.plan.nx, self.plan.ns):
            raise ValueError(f"FkFilterBank built for {(self.plan.nx, self.plan.ns)}, got {tuple(x.shape)}")
        if outs is None:
            outs = [torch.empty_like(x) for _ in self.dms]
        outs = list(outs)
        if len(outs) != len(self.dms):
            raise ValueError(f"FkFilterBank has {len(self.dms)} masks, got {len(outs)} outputs")
        for o in outs:
            if o.dtype != torch.float32 or not o.is_cuda or not o.is_contiguous() or tuple(o.shape) != tuple(x.shape) \
                    or o.device != x.device:
                raise ValueError("FkFilterBank outputs must be contiguous float32 CUDA tensors of the input's shape")
        return outs, _lib.ffi.new("float*[]", [_lib.ptr(o, "float*") for o in outs])

    def __call__(self, x, outs=None, tapering=False):
        """Filter x with every mask; returns the list of outputs.  One of `outs` may be x itself; no two may overlap."""
        outs, _ = self._outs(x, outs)
        nbytes = x.numel() * 4
        for i, o in enumerate(outs):          # checked on the caller's outputs, before any is swapped for a temporary
            for j in range(i):
                a, c = o.data_ptr(), outs[j].data_ptr()
                if a < c + nbytes and c < a + nbytes:
                    raise ValueError(f"FkFilterBank outputs {j} and {i} overlap")
        ns = self.plan.ns
        xin = x.clone() if _misaligned(x, ns) else x          # misaligned matrices go through aligned copies
        run = [_torch().empty_like(o) if _misaligned(o, ns) else o for o in outs]
        ys = _lib.ffi.new("float*[]", [_lib.ptr(o, "float*") for o in run])
        L = _lib.lib()
        with _torch().cuda.device(self.device):
            _lib.check(L.d4w_fk_bank_apply(self.plan.ptr, self.ptr, _lib.ptr(xin, "float*"), ys, _lib.ptr(self._ws()),
                                           int(bool(tapering)), _lib.stream_ptr()), "fk bank")
        for o, r in zip(outs, run):
            if r is not o:
                o.copy_(r)
        return outs

    def run_pass(self, i, x, outs, tapering=False, mask=0):
        """Launch pass i (1..5) alone -- profiling / per-kernel timing.  Passes 1 and 2 serve every mask; passes 3..5
        run mask `mask`."""
        outs, ys = self._outs(x, outs)
        L = _lib.lib()
        with _torch().cuda.device(self.device):
            _lib.check(L.d4w_fk_bank_apply_pass(self.plan.ptr, self.ptr, _lib.ptr(x, "float*"), ys, _lib.ptr(self._ws()),
                                                int(bool(tapering)), int(i), int(mask), _lib.stream_ptr()),
                       f"fk bank pass {i}")

    def traffic_bytes(self):
        """HBM bytes each pass must move for the whole bank (passes 3..5 summed over the masks)."""
        return _traffic_bytes(self.plan, self.rows_kept, len(self.dms))


def _destroy_spectrum(lib, ptr, plan):
    """Destroy a d4w_fk_spectrum; `plan` is held until then, since the spectrum points to it."""
    lib.d4w_fk_spectrum_destroy(ptr)


class FkSpectrum:
    """f-k power spectrum |fftshift(fft2(x))|^2 over one band of one matrix shape (d4w_fk_spectrum): the filter's
    forward transform on the half-plane wavenumber rows that touch the band, then a forward-only power pass.

    >>> spec = FkSpectrum((nx, ns), (k0, k1), (f0, f1), device=0)   # half-open index ranges on the shifted axes
    >>> p = spec(x_cuda)             # float32 [k1 - k0, f1 - f0]
    >>> p = spec(x_long)             # x_long [nx, m >= ns]: mean over the m // ns whole blocks of ns samples

    `rows` is the number of half-plane rows k' in [0, nx/2] transformed (those with +k' or -k' inside the band)."""

    def __init__(self, shape, k_idx, f_idx, device=None):
        torch = _torch()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.plan = get_plan(int(shape[0]), int(shape[1]), self.device)
        self.k_idx = (int(k_idx[0]), int(k_idx[1]))
        self.f_idx = (int(f_idx[0]), int(f_idx[1]))
        self.shape = (self.k_idx[1] - self.k_idx[0], self.f_idx[1] - self.f_idx[0])
        L = _lib.lib()
        out = _lib.ffi.new("d4w_fk_spectrum**")
        with torch.cuda.device(self.device):
            _lib.check(L.d4w_fk_spectrum_create(out, self.plan.ptr, *self.k_idx, *self.f_idx), "fk spectrum")
        self.ptr = out[0]
        weakref.finalize(self, _destroy_spectrum, L, self.ptr, self.plan)
        self.rows = int(L.d4w_fk_spectrum_rows(self.ptr))
        self.workspace_bytes = int(L.d4w_fk_spectrum_workspace_bytes(self.plan.ptr, self.ptr))

    def _ws(self):
        return self.plan.get_workspace(self.workspace_bytes)

    def __call__(self, x, out=None, tapering=False):
        """Spectrum of x [nx, ns], or the mean of the spectra of the m // ns whole blocks x[:, b*ns:(b+1)*ns] of
        x [nx, m] (a trailing partial block is not used).  tapering=True: each block is multiplied by
        Tukey(ns, alpha=0.03) along time first; x is never modified."""
        torch = _torch()
        nx, ns = self.plan.nx, self.plan.ns
        if x.dtype != torch.float32 or not x.is_cuda or not x.is_contiguous() or x.dim() != 2:
            raise ValueError("FkSpectrum expects a contiguous 2-D float32 CUDA tensor")
        if x.shape[0] != nx or x.shape[1] < ns:
            raise ValueError(f"FkSpectrum built for blocks of {(nx, ns)}, got {tuple(x.shape)}")
        if out is None:
            out = torch.empty(self.shape, dtype=torch.float32, device=x.device)
        elif out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous() or tuple(out.shape) != self.shape \
                or out.device != x.device:
            raise ValueError(f"FkSpectrum output must be a contiguous float32 CUDA tensor of shape {self.shape}")
        nblocks = x.shape[1] // ns
        L = _lib.lib()
        with torch.cuda.device(self.device):
            # x of exactly ns samples: x itself (through an aligned copy if it starts off the column kernels' boundary);
            # otherwise each block is copied into one contiguous [nx, ns] buffer (one extra read and write of the block),
            # and the power pass accumulates P / nblocks into out
            whole = x.shape[1] == ns
            if whole:
                buf = x.clone() if _misaligned(x, ns) else x
            else:
                buf = torch.empty((nx, ns), dtype=x.dtype, device=x.device)
            for b in range(nblocks):
                if not whole:
                    buf.copy_(x[:, b * ns:(b + 1) * ns])
                _lib.check(L.d4w_fk_spectrum_apply(self.plan.ptr, self.ptr, _lib.ptr(buf, "float*"), _lib.ptr(out, "float*"),
                                                   _lib.ptr(self._ws()), int(bool(tapering)), 1.0 / nblocks, int(b > 0),
                                                   _lib.stream_ptr()), "fk_spectrum")
        return out


FkWelchLayout = namedtuple("FkWelchLayout", "nperseg noverlap step nseg starts nperseg_x noverlap_x step_x nseg_x starts_x")


def fk_welch_layout(nx, ns, nperseg, noverlap, nperseg_x, noverlap_x):
    """Segment geometry of the f-k Welch spectrum of an [nx, ns] record, pure Python (dsp.fk_welch's rules, those of
    dsp.welch_layout on each axis).  nperseg=None is 256 and noverlap=None is nperseg // 2; time segment s covers samples
    [starts[s], starts[s] + nperseg), starts[s] = s * step, step = nperseg - noverlap, nseg = (ns - nperseg) // step + 1
    (a trailing partial segment is dropped).  The channel axis follows the same rules, except that nperseg_x=None is one
    segment spanning all nx channels (noverlap_x is then ignored).  ValueError for an empty record, a segment length
    outside [1, ns] (or [1, nx]) and an overlap that is not less than its segment length."""
    nx, ns = int(nx), int(ns)
    if nx < 1 or ns < 1:
        raise ValueError(f"fk_welch: empty record of shape {(nx, ns)}")

    def axis(n, nper, nover, what, default):
        nper = default if nper is None else int(nper)
        if not 1 <= nper <= n:
            raise ValueError(f"fk_welch: {what} = {nper} must lie in [1, {n}]")
        nover = nper // 2 if nover is None else int(nover)
        if nover >= nper:
            raise ValueError(f"fk_welch: the overlap {nover} must be less than {what} = {nper}")
        step = nper - nover
        nseg = (n - nper) // step + 1
        return nper, nover, step, nseg, tuple(s * step for s in range(nseg))

    t = axis(ns, nperseg, noverlap, "nperseg", 256)
    c = axis(nx, nperseg_x, noverlap_x if nperseg_x is not None else 0, "nperseg_x", nx)
    return FkWelchLayout(*t, *c)


# staging buffer of FkWelch: as many whole segments as fit this many bytes, at least one
FK_WELCH_STAGE_BYTES = 512 << 20


class FkWelch:
    """f-k power spectral density by Welch's method over one record shape (dsp.fk_welch): segments of segment_shape
    (Lx, L) are detrended, windowed and staged as contiguous matrices (d4w_fk_segment_stage), each goes through an
    FkSpectrum of that shape, and the power pass averages the time segments of one channel segment in place.

    >>> w = FkWelch((nx, ns), (Lx, L), (k0, k1), (f0, f1), wt, wx, True, scale, device=0, noverlap=L // 2)
    >>> p = w(x_cuda)          # float32 [nseg_x, k1 - k0, f1 - f0]: scale * the mean over time segments, per channel segment

    window (L) and window_x (Lx) are float arrays; scale multiplies the mean periodogram (dsp.fk_welch passes the density
    or spectrum normalisation).  noverlap / noverlap_x follow fk_welch_layout; with Lx == nx there is one channel segment.
    `layout` is the fk_welch_layout, `batch` the number of time segments staged per launch (FK_WELCH_STAGE_BYTES)."""

    def __init__(self, shape, segment_shape, k_idx, f_idx, window, window_x, detrend, scale, device=None, noverlap=None,
                 noverlap_x=None):
        torch = _torch()
        nx, ns = int(shape[0]), int(shape[1])
        lx, l = int(segment_shape[0]), int(segment_shape[1])
        self.layout = fk_welch_layout(nx, ns, l, noverlap, lx, noverlap_x)
        wt, wx = np.asarray(window, dtype=np.float64), np.asarray(window_x, dtype=np.float64)
        if wt.shape != (l,) or wx.shape != (lx,):
            raise ValueError(f"FkWelch: windows of shapes {wt.shape} and {wx.shape} for segments of {(lx, l)} "
                             f"(time window [{l}], channel window [{lx}])")
        self.shape, self.segment_shape = (nx, ns), (lx, l)
        self.spec = FkSpectrum((lx, l), k_idx, f_idx, device=device)
        self.device, self.plan = self.spec.device, self.spec.plan
        self.detrend, self.scale = bool(detrend), float(scale)
        self.out_shape = (self.layout.nseg_x,) + self.spec.shape
        dev = f"cuda:{self.device}"
        self.wt = torch.from_numpy(wt).to(dev, torch.float32)
        self.wx = torch.from_numpy(wx).to(dev, torch.float32)
        # each staged segment starts 16 bytes aligned: the column kernels' boundary for rows of L samples
        self.seg_stride = (lx * l + 3) // 4 * 4
        self.batch = max(1, min(self.layout.nseg, FK_WELCH_STAGE_BYTES // (4 * self.seg_stride)))
        self.buf = torch.empty(self.batch * self.seg_stride, dtype=torch.float32, device=dev)

    def __call__(self, x, out=None):
        """P [nseg_x, k1 - k0, f1 - f0] of x [nx, ns] (contiguous float32 CUDA); x is never modified."""
        torch = _torch()
        if x.dtype != torch.float32 or not x.is_cuda or not x.is_contiguous() or x.dim() != 2:
            raise ValueError("FkWelch expects a contiguous 2-D float32 CUDA tensor")
        if tuple(x.shape) != self.shape:
            raise ValueError(f"FkWelch built for records of {self.shape}, got {tuple(x.shape)}")
        if out is None:
            out = torch.empty(self.out_shape, dtype=torch.float32, device=x.device)
        elif out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous() or tuple(out.shape) != self.out_shape \
                or out.device != x.device:
            raise ValueError(f"FkWelch output must be a contiguous float32 CUDA tensor of shape {self.out_shape}")
        lay, (nx, ns), (lx, l) = self.layout, self.shape, self.segment_shape
        L = _lib.lib()
        plane = self.spec.shape[0] * self.spec.shape[1]
        scale = self.scale / lay.nseg
        with torch.cuda.device(self.device):
            ws = _lib.ptr(self.spec._ws())
            stream = _lib.stream_ptr()
            for j, c0 in enumerate(lay.starts_x):
                dst = _lib.ffi.cast("float*", out.data_ptr() + 4 * j * plane)
                for s0 in range(0, lay.nseg, self.batch):
                    cnt = min(self.batch, lay.nseg - s0)
                    _lib.check(L.d4w_fk_segment_stage(_lib.ptr(x, "float*"), nx, ns, c0, lx, lay.starts[s0], l, lay.step, cnt,
                                                      _lib.ptr(self.wx, "float*"), _lib.ptr(self.wt, "float*"), int(self.detrend),
                                                      _lib.ptr(self.buf, "float*"), self.seg_stride, stream), "fk_welch stage")
                    for s in range(cnt):
                        seg = _lib.ffi.cast("float*", self.buf.data_ptr() + 4 * s * self.seg_stride)
                        _lib.check(L.d4w_fk_spectrum_apply(self.plan.ptr, self.spec.ptr, seg, dst, ws, 0, scale,
                                                           int(s0 + s > 0), stream), "fk_welch")
        return out
