"""Host side of the f-k filter: mask descriptors (`FkMask`), per-shape plans and the reusable
`FkFilter` object that owns the device buffers.  dsp.fk_filter_design / hybrid_*_filter_design
return `FkMask`; dsp.fk_filter_filt / fk_filter_sparsefilt run an `FkFilter`.

All arithmetic happens in libd4w.so (hand-written sm_90a CUDA, see csrc/fk_kernels.cuh);
PyTorch is used for device memory and streams only.
"""
import threading
import weakref

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


class FkMask:
    """Lazy f-k mask: the closed-form description of what the reference's design function
    returns.  `np.asarray(mask)` / `mask.todense()` materialise exactly the reference's
    [channel x time] float64 array (shifted layout) on demand; `fk_filter_filt` uses the
    description directly and never builds the dense matrix.
    """

    def __init__(self, kind, shape, params, order="C"):
        self.kind = kind
        self.shape = (int(shape[0]), int(shape[1]))
        self.params = params
        self.order = order
        self.prune_eps = 0.0           # opt-in: FkFilter / fk_filter_filt drop rows whose folded mask never exceeds this
        self.ndim = 2
        self.dtype = np.dtype(np.float64)
        self._dev = {}
        self._dense = None

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

    def on_device(self, plan, eps=0.0):
        eps = float(eps or 0.0)
        if eps:
            key = (plan.serial, eps)
            dm = self._dev.get(key)
            if dm is None:
                if self.kind == "dense":
                    dm = _DenseMaskHolder(plan, _dense_to_device(self._dense, plan.device), eps).dm
                else:
                    dm = _DeviceMask(plan, self._create, eps)
                self._dev[key] = dm
            return dm
        dm = self._dev.get(plan.serial)
        if dm is None:
            for k in [k for k, v in self._dev.items() if _plan_cache.get((v.plan.nx, v.plan.ns, v.plan.device)) is not v.plan]:
                del self._dev[k]                      # tables of plans that were dropped by free_plans()
            if (plan.nx, plan.ns) != self.shape:
                raise ValueError(f"operands could not be broadcast together with shapes ({plan.nx},{plan.ns}) {self.shape}")
            if self.kind == "dense":      # design functions without a closed form on the device
                dm = _DenseMaskHolder(plan, _dense_to_device(self._dense, plan.device)).dm
            else:
                dm = _DeviceMask(plan, self._create)
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
        if out is None:
            out = torch.empty_like(x)
        L = _lib.lib()
        with torch.cuda.device(self.device):
            _lib.check(L.d4w_fk_apply(self.plan.ptr, self.dm.ptr, _lib.ptr(x, "float*"), _lib.ptr(out, "float*"),
                                      _lib.ptr(self._ws()), int(bool(tapering)), _lib.stream_ptr()), "fk_filter_filt")
        return out

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
        nx, ns, r = self.plan.nx, self.plan.ns, self.rows_kept
        real, spec = nx * ns * 4, r * ns * 8
        split = 2 * spec if self.plan.t1 > 1 else 0
        return {"p1_col_fwd": real + spec, "p2_row_split": split, "p3_row_mid": 2 * spec + r * ns * 4,
                "p4_row_unsplit": split, "p5_col_inv": spec + real}
