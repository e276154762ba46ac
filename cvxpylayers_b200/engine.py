"""Python handle around the C-ABI engine: one :class:`Engine` per (structure, device).

PyTorch is plumbing here -- device memory, the current CUDA stream -- not the compute path:
every tensor is passed to libbcone.so as a raw device pointer.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .structure import Structure

STATUS = {1: "solved", 2: "inaccurate", -1: "unbounded", -2: "infeasible", -4: "failed"}

# solver_args keys accepted at the reference boundary (README "Passing arguments to the solvers",
# tests/test_torch.py:401-405; diffcp keys per SURVEY.md section 5) -> engine settings
_ARG_MAP = {
    "eps_abs": "eps_abs", "eps_rel": "eps_rel", "eps_infeas": "eps_infeas", "max_iters": "max_iters",
    "alpha": "alpha", "rho_x": "rho_x", "scale": "scale", "normalize": "normalize",
    "adaptive_scale": "adaptive_scale", "check_interval": "check_interval", "ruiz_passes": "ruiz_passes",
    "lsqr_atol": "lsqr_atol", "lsqr_btol": "lsqr_btol", "lsqr_conlim": "lsqr_conlim",
    "lsqr_iter_lim": "lsqr_iter_lim", "lsqr_precond": "lsqr_precond", "adaptive_check": "adaptive_check",
    "acceleration_lookback": "acceleration_lookback", "acceleration_interval": "acceleration_interval",
}
_IGNORED = {"verbose", "n_jobs_forward", "n_jobs_backward", "solve_method", "warm_starts", "raise_on_error", "warm_start", "reuse_setup", "shared_matrices"}   # (warm_start / reuse_setup / shared_matrices are handled by the layer)


def make_settings(args: dict | None) -> _lib.BconeSettings:
    st = _lib.default_settings()
    for k, v in (args or {}).items():
        if k == "eps":  # diffcp maps eps -> eps_abs = eps_rel for SCS >= 3 (SURVEY.md 8a F7)
            st.eps_abs = float(v)
            st.eps_rel = float(v)
        elif k == "mode":
            if v not in ("lsqr",):
                raise ValueError(f"backward mode {v!r} is not supported (only 'lsqr')")
        elif k in _ARG_MAP:
            cur = getattr(st, _ARG_MAP[k])
            setattr(st, _ARG_MAP[k], type(cur)(v))
        elif k in _IGNORED:
            continue
        else:
            raise ValueError(f"unknown solver argument {k!r}")
    return st


def _ptr(t: torch.Tensor | None) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _chk(t: torch.Tensor | None, shape, dtype, device, name: str):
    if t is None:
        return
    if t.device != device or t.dtype != dtype or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
        raise ValueError(f"{name}: expected contiguous {dtype} {tuple(shape)} on {device}, got "
                         f"{t.dtype} {tuple(t.shape)} on {t.device} (contiguous={t.is_contiguous()})")


@dataclass
class Solution:
    x: torch.Tensor
    y: torch.Tensor
    s: torch.Tensor
    status: torch.Tensor
    iters: torch.Tensor
    resid: torch.Tensor


class Engine:
    """Owns the device copy of one problem structure and launches the kernels."""

    def __init__(self, structure: Structure, device: torch.device | str | int = "cuda", max_batch: int = 0):
        self.lib = _lib.load()
        self.structure = structure
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.EngineUnavailable("the engine runs on CUDA devices only (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        st = structure
        d = _lib.BconeDesc()
        d.n, d.m, d.nnzA, d.nnzP = st.n, st.m, st.nnzA, st.nnzP
        ip = lambda a: a.ctypes.data_as(_lib._i32p)  # noqa: E731
        self._keep = [st.A_indptr, st.A_indices]
        d.A_indptr, d.A_indices = ip(st.A_indptr), ip(st.A_indices)
        if st.P_indptr is not None:
            d.P_indptr, d.P_indices = ip(st.P_indptr), ip(st.P_indices)
            self._keep += [st.P_indptr, st.P_indices]
        q = np.asarray(st.cones.q, dtype=np.int32)
        s = np.asarray(st.cones.s, dtype=np.int32)
        self._keep += [q, s]
        d.z, d.l, d.nq, d.ns, d.ep, d.ed = st.cones.z, st.cones.l, q.size, s.size, st.cones.ep, st.cones.ed
        d.q, d.s = ip(q), ip(s)
        d.device, d.max_batch = self.device.index, max_batch
        h = C.c_void_p()
        rc = self.lib.bcone_create(C.byref(d), C.byref(h))
        if rc != 0:
            raise _lib.EngineUnavailable(f"bcone_create failed ({rc}): {self.lib.bcone_last_error(None).decode()}")
        self.h = h
        self._boundary = None

    def __del__(self):
        h = getattr(self, "h", None)
        if h:
            self.lib.bcone_destroy(h)
            self.h = None

    # ------------------------------------------------------------------ helpers
    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _raise(self, rc: int, what: str):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.bcone_last_error(self.h).decode()}")

    def launch_count(self) -> int:
        return int(self.lib.bcone_launch_count(self.h))

    def fallback_count(self) -> int:
        v = C.c_int32()
        self.lib.bcone_fallback_count(self.h, C.byref(v))
        return int(v.value)

    def kernel_info(self) -> dict:
        v = [C.c_int32() for _ in range(6)]
        self.lib.bcone_kernel_info(self.h, *[C.byref(x) for x in v])
        k = ["fwd_threads", "fwd_smem", "fwd_ctas_per_sm", "bwd_threads", "bwd_smem", "bwd_ctas_per_sm"]
        return {a: int(b.value) for a, b in zip(k, v)}

    # codes 4-6 / 3: the values-off-chip tier (instances whose CSR values do not fit in shared memory; include/bcone.h)
    FWD_PATHS = ("fwd_kernel (on-chip Cholesky)", "fwd_kernel (indirect, CG)", "fwd_fast_kernel (register-tiled)",
                 "fwd_kernel (values on chip, Cholesky factor and vectors in a global slab)",
                 "fwd_kernel (values off chip: values in a global slab, Cholesky factor and vectors on chip)",
                 "fwd_kernel (values off chip: values, Cholesky factor and vectors in a global slab)",
                 "fwd_kernel (values off chip: values and vectors in a global slab, indirect, CG)")
    BWD_PATHS = ("bwd_kernel (generic LSQR)", "bwd_fast_kernel (fused single-pass LSQR)", "bwd_block_kernel (KKT-block preconditioned, bwd_fast_kernel fallback)",
                 "bwd_kernel (generic LSQR, values off chip: read in place from A_vals)")

    def small_cta_info(self) -> dict:
        """CTAs per SM of the 4-CTA/SM builds of the generic forward and adjoint (0: the structure has none)."""
        f, b = C.c_int32(), C.c_int32()
        self.lib.bcone_small_cta_info(self.h, C.byref(f), C.byref(b))
        return {"fwd": f.value, "bwd": b.value}

    def path_info(self) -> dict:
        f, b = C.c_int32(), C.c_int32()
        self.lib.bcone_path_info(self.h, C.byref(f), C.byref(b))
        return {"fwd": self.FWD_PATHS[f.value], "bwd": self.BWD_PATHS[b.value]}

    def alloc_solution(self, B: int) -> Solution:
        dev, f64, st = self.device, torch.float64, self.structure
        return Solution(torch.empty((B, st.n), dtype=f64, device=dev), torch.empty((B, st.m), dtype=f64, device=dev),
                        torch.empty((B, st.m), dtype=f64, device=dev), torch.empty(B, dtype=torch.int32, device=dev),
                        torch.empty(B, dtype=torch.int32, device=dev), torch.empty((B, 3), dtype=f64, device=dev))

    def copy2d(self, dst: torch.Tensor, src: torch.Tensor, lo: int, hi: int, to_device: bool):
        """Pitched copy of the batch slice [:, lo:hi] between a pinned host tensor [rows, B] and a
        contiguous device chunk [rows, hi-lo] on the current stream."""
        host, devt = (src, dst) if to_device else (dst, src)
        rows, Bfull = host.shape
        w = (hi - lo) * 8
        hp = host.data_ptr() + lo * 8
        args = (devt.data_ptr(), w, hp, Bfull * 8) if to_device else (hp, Bfull * 8, devt.data_ptr(), w)
        rc = self.lib.bcone_memcpy2d(C.c_void_p(args[0]), C.c_int64(args[1]), C.c_void_p(args[2]), C.c_int64(args[3]),
                                     C.c_int64(w), C.c_int64(rows), C.c_int32(1 if to_device else 0), self._stream())
        if rc != 0:
            raise RuntimeError(f"bcone_memcpy2d failed: {self.lib.bcone_last_error(None).decode()}")

    # ------------------------------------------------------------------ boundary re-packing
    def set_boundary(self, gather: np.ndarray, b_idx: np.ndarray):
        gather = np.ascontiguousarray(gather, dtype=np.int32)
        b_idx = np.ascontiguousarray(b_idx, dtype=np.int32)
        rc = self.lib.bcone_set_boundary(self.h, C.c_int32(gather.size + b_idx.size), gather.ctypes.data_as(_lib._i32p),
                                         C.c_int32(b_idx.size), b_idx.ctypes.data_as(_lib._i32p))
        self._raise(rc, "bcone_set_boundary")
        self._boundary = (gather.size + b_idx.size, b_idx.size)
        self._nnzP_b = self.structure.nnzP

    def set_boundary_P(self, nnzP_boundary: int, gatherP: np.ndarray):
        """Rows of the reference's P_eval feeding the engine's upper-triangular slots (any symmetric pattern)."""
        gatherP = np.ascontiguousarray(gatherP, dtype=np.int32)
        rc = self.lib.bcone_set_boundary_quad(self.h, C.c_int32(nnzP_boundary), gatherP.ctypes.data_as(_lib._i32p))
        self._raise(rc, "bcone_set_boundary_quad")
        self._nnzP_b = int(nnzP_boundary)

    def ingest(self, A_eval: torch.Tensor, q_eval: torch.Tensor, P_eval: torch.Tensor | None = None, out=None):
        """[nnz_aug,B] / [n+1,B] boundary tensors -> engine-layout (A_vals, P_vals, b, c).
        ``out`` = preallocated (A_vals, P_vals, b, c) views (pipelined callers)."""
        st, dev, f64 = self.structure, self.device, torch.float64
        if self._boundary is None:
            raise RuntimeError("set_boundary() has not been called")
        B = A_eval.shape[1]
        _chk(A_eval, (self._boundary[0], B), f64, dev, "A_eval")
        _chk(q_eval, (st.n + 1, B), f64, dev, "q_eval")
        _chk(P_eval, (self._nnzP_b, B), f64, dev, "P_eval")
        if out is not None:
            A_vals, P_vals, b, c = out
        else:
            A_vals = torch.empty((B, st.nnzA), dtype=f64, device=dev)
            b = torch.empty((B, st.m), dtype=f64, device=dev)
            c = torch.empty((B, st.n), dtype=f64, device=dev)
            P_vals = torch.empty((B, st.nnzP), dtype=f64, device=dev) if (P_eval is not None and st.nnzP) else None
        rc = self.lib.bcone_ingest(self.h, C.c_int32(B), _ptr(A_eval), _ptr(q_eval), _ptr(P_eval), _ptr(A_vals),
                                   _ptr(P_vals), _ptr(b), _ptr(c), self._stream())
        self._raise(rc, "bcone_ingest")
        return A_vals, P_vals, b, c

    def ingest_cols(self, A_eval, q_eval, P_eval, lo: int, hi: int, out):
        """Column slice [lo, hi) of full boundary tensors -> the engine-layout views in ``out`` (no staging copy)."""
        Bfull = A_eval.shape[1]
        A_vals, P_vals, b, c = out
        off = lo * 8
        pp = lambda t: C.c_void_p(0 if t is None else t.data_ptr() + off)  # noqa: E731
        rc = self.lib.bcone_ingest_pitched(self.h, C.c_int32(hi - lo), C.c_int64(Bfull), pp(A_eval), pp(q_eval), pp(P_eval), _ptr(A_vals),
                                           _ptr(P_vals), _ptr(b), _ptr(c), self._stream())
        self._raise(rc, "bcone_ingest_pitched")

    def emit_cols(self, dA_vals, dP_vals, db, dc, lo: int, hi: int, out):
        """Engine gradients of instances [lo, hi) -> columns [lo, hi) of the full boundary gradient tensors in ``out``."""
        dA_eval, dq_eval, dP_eval = out
        Bfull = dA_eval.shape[1]
        off = lo * 8
        pp = lambda t: C.c_void_p(0 if t is None else t.data_ptr() + off)  # noqa: E731
        rc = self.lib.bcone_emit_pitched(self.h, C.c_int32(hi - lo), C.c_int64(Bfull), _ptr(dA_vals), _ptr(dP_vals), _ptr(db), _ptr(dc),
                                         pp(dA_eval), pp(dq_eval), pp(dP_eval), self._stream())
        self._raise(rc, "bcone_emit_pitched")

    def emit(self, dA_vals, dP_vals, db, dc, out=None):
        st, dev, f64 = self.structure, self.device, torch.float64
        B = dA_vals.shape[0]
        if out is not None:
            dA_eval, dq_eval, dP_eval = out
        else:
            dA_eval = torch.empty((self._boundary[0], B), dtype=f64, device=dev)
            dq_eval = torch.empty((st.n + 1, B), dtype=f64, device=dev)
            dP_eval = torch.empty((self._nnzP_b, B), dtype=f64, device=dev) if (dP_vals is not None and st.nnzP) else None
        rc = self.lib.bcone_emit(self.h, C.c_int32(B), _ptr(dA_vals), _ptr(dP_vals), _ptr(db), _ptr(dc), _ptr(dA_eval),
                                 _ptr(dq_eval), _ptr(dP_eval), self._stream())
        self._raise(rc, "bcone_emit")
        return dA_eval, dq_eval, dP_eval

    # ------------------------------------------------------------------ fused parameter -> matrix map
    def set_param_maps(self, A_map, q_map, P_map=None):
        """SciPy CSR matrices [rows x P1] in boundary row order (the reference's ``_A_scipy`` / ``_q_scipy`` /
        ``_P_scipy``, ``torch/cvxpylayer.py:443-451``)."""
        import scipy.sparse as sp  # noqa: PLC0415

        def parts(M):
            if M is None:
                return None, None, None, []
            M = sp.csr_matrix(M)
            M.sort_indices()
            ptr = np.ascontiguousarray(M.indptr, dtype=np.int32)
            col = np.ascontiguousarray(M.indices, dtype=np.int32)
            val = np.ascontiguousarray(M.data, dtype=np.float64)
            return (ptr.ctypes.data_as(_lib._i32p), col.ctypes.data_as(_lib._i32p), val.ctypes.data_as(_lib._f64p), [ptr, col, val])

        P1 = int(A_map.shape[1])
        if self._boundary is None:
            raise RuntimeError("set_boundary() has not been called")
        if A_map.shape[0] != self._boundary[0] or q_map.shape != (self.structure.n + 1, P1):
            raise ValueError("parameter maps do not match the boundary tensors")
        if (P_map is not None) != bool(self.structure.nnzP) or (P_map is not None and P_map.shape != (self._nnzP_b, P1)):
            raise ValueError("P parameter map does not match the structure")
        a, q, p = parts(A_map), parts(q_map), parts(P_map)
        rc = self.lib.bcone_set_param_maps(self.h, C.c_int32(P1), a[0], a[1], a[2], q[0], q[1], q[2], p[0], p[1], p[2])
        self._raise(rc, "bcone_set_param_maps")
        self._P1 = P1

    def ingest_params(self, p_stack: torch.Tensor, out=None, shared: bool = False):
        """p_stack[P1, B] -> engine-layout (A_vals, P_vals, b, c) without materialising A_eval.
        ``shared=True``: A_vals[nnzA] / P_vals[nnzP] are evaluated once, from column 0 (the parameters feeding A and P are
        unbatched); b and c from every column."""
        st, dev, f64 = self.structure, self.device, torch.float64
        B = p_stack.shape[1]
        _chk(p_stack, (self._P1, B), f64, dev, "p_stack")
        if out is not None:
            A_vals, P_vals, b, c = out
        else:
            lead = () if shared else (B,)
            A_vals = torch.empty((*lead, st.nnzA), dtype=f64, device=dev)
            b = torch.empty((B, st.m), dtype=f64, device=dev)
            c = torch.empty((B, st.n), dtype=f64, device=dev)
            P_vals = torch.empty((*lead, st.nnzP), dtype=f64, device=dev) if st.nnzP else None
        fn = self.lib.bcone_ingest_params_shared if shared else self.lib.bcone_ingest_params
        rc = fn(self.h, C.c_int32(B), _ptr(p_stack), _ptr(A_vals), _ptr(P_vals), _ptr(b), _ptr(c), self._stream())
        self._raise(rc, "bcone_ingest_params_shared" if shared else "bcone_ingest_params")
        return A_vals, P_vals, b, c

    def emit_params(self, dA_vals, dP_vals, db, dc, out=None, shared: bool = False):
        """engine gradients -> dp_stack[P1, B] (transposed parameter maps; the constant's row stays 0).
        ``shared=True``: dA_vals[nnzA] / dP_vals[nnzP] are batch sums (:meth:`vjp` on shared matrices); their contribution goes
        into column 0, that of db / dc into every column."""
        B = db.shape[0]
        dp = out if out is not None else torch.empty((self._P1, B), dtype=torch.float64, device=self.device)
        fn = self.lib.bcone_emit_params_shared if shared else self.lib.bcone_emit_params
        rc = fn(self.h, C.c_int32(B), _ptr(dA_vals), _ptr(dP_vals), _ptr(db), _ptr(dc), _ptr(dp), self._stream())
        self._raise(rc, "bcone_emit_params_shared" if shared else "bcone_emit_params")
        return dp

    # ------------------------------------------------------------------ forward / backward
    def cache_bytes(self, B: int) -> int:
        """Bytes of the set-up cache of a batch of B instances; 0 = this structure has no cached set-up path."""
        return int(self.lib.bcone_cache_bytes(self.h, C.c_int32(B)))

    def new_cache(self, B: int):
        """A zero-filled set-up cache for ``solve(..., cache=)`` (``None`` when the structure has no such path)."""
        nb = self.cache_bytes(B)
        return torch.zeros(nb // 8, dtype=torch.float64, device=self.device) if nb else None

    def solve(self, A_vals, b, c, P_vals=None, settings: _lib.BconeSettings | None = None, out: "Solution | None" = None,
              warm: "tuple | Solution | None" = None, cache=None, reuse: bool = False) -> Solution:
        """``cache`` (from :meth:`new_cache`): keep the equilibration and the factorisation of every instance; ``reuse=True``
        states that ``A_vals`` / ``P_vals`` are those of the call that filled it (``b`` and ``c`` may differ) and skips them.
        1-D ``A_vals[nnzA]`` (and ``P_vals[nnzP]``): one copy shared by the batch (``bcone_solve_shared``; B from ``b``)."""
        st, dev, f64 = self.structure, self.device, torch.float64
        shared = A_vals.dim() == 1
        B = b.shape[0] if shared else A_vals.shape[0]
        lead = () if shared else (B,)
        _chk(A_vals, (*lead, st.nnzA), f64, dev, "A_vals")
        _chk(b, (B, st.m), f64, dev, "b")
        _chk(c, (B, st.n), f64, dev, "c")
        if st.nnzP:
            if P_vals is None:
                raise ValueError("structure has a quadratic term but P_vals is None")
            _chk(P_vals, (*lead, st.nnzP), f64, dev, "P_vals")
        if shared and cache is not None:
            raise ValueError("cache: a shared-matrix solve keeps its own set-up (pass cache=None)")
        settings = settings or _lib.default_settings()
        if out is not None:
            x, y, s, status, iters, resid = out.x, out.y, out.s, out.status, out.iters, out.resid
        else:
            x = torch.empty((B, st.n), dtype=f64, device=dev)
            y = torch.empty((B, st.m), dtype=f64, device=dev)
            s = torch.empty((B, st.m), dtype=f64, device=dev)
            status = torch.empty(B, dtype=torch.int32, device=dev)
            iters = torch.empty(B, dtype=torch.int32, device=dev)
            resid = torch.empty((B, 3), dtype=f64, device=dev)
        x0 = y0 = s0 = None
        if warm is not None:   # a previous solution of a nearby problem (training loops re-solve almost the same programs)
            x0, y0, s0 = (warm.x, warm.y, warm.s) if isinstance(warm, Solution) else warm
            for name, t_, shp in (("x0", x0, (B, st.n)), ("y0", y0, (B, st.m)), ("s0", s0, (B, st.m))):
                _chk(t_, shp, f64, dev, name)
        if cache is not None and (cache.dtype != f64 or cache.device != dev or cache.numel() * 8 < self.cache_bytes(B) or not cache.is_contiguous()):
            raise ValueError("cache: need a contiguous float64 tensor of cache_bytes(B) bytes on the engine's device (engine.new_cache(B))")
        if shared:
            rc = self.lib.bcone_solve_shared(self.h, C.c_int32(B), _ptr(A_vals), _ptr(P_vals if st.nnzP else None), _ptr(b), _ptr(c),
                                             _ptr(x0), _ptr(y0), _ptr(s0), _ptr(x), _ptr(y), _ptr(s), _ptr(status), _ptr(iters), _ptr(resid),
                                             C.byref(settings), self._stream())
        else:
            rc = self.lib.bcone_solve_cached(self.h, C.c_int32(B), _ptr(A_vals), _ptr(P_vals if st.nnzP else None), _ptr(b), _ptr(c),
                                             _ptr(x0), _ptr(y0), _ptr(s0), _ptr(x), _ptr(y), _ptr(s), _ptr(status), _ptr(iters), _ptr(resid),
                                             _ptr(cache), C.c_int32(1 if (cache is not None and reuse) else 0), C.byref(settings), self._stream())
        self._raise(rc, "bcone_solve_shared" if shared else "bcone_solve")
        return Solution(x, y, s, status, iters, resid)

    def vjp(self, A_vals, b, c, x, y, s, dx, dy, P_vals=None, settings: _lib.BconeSettings | None = None, out=None):
        """-> dA_vals[B,nnzA], dP_vals[B,nnzP]|None, db[B,m], dc[B,n], lsqr_iters[B]  (``out``: the same five, preallocated).
        1-D ``A_vals[nnzA]`` / ``P_vals[nnzP]`` (shared by the batch): dA_vals[nnzA] / dP_vals[nnzP] are the batch sums
        (``bcone_vjp_shared``)."""
        st, dev, f64 = self.structure, self.device, torch.float64
        shared = A_vals.dim() == 1
        B = b.shape[0] if shared else A_vals.shape[0]
        lead = () if shared else (B,)
        for name, t, shp in (("A_vals", A_vals, (*lead, st.nnzA)), ("b", b, (B, st.m)), ("c", c, (B, st.n)),
                             ("x", x, (B, st.n)), ("y", y, (B, st.m)), ("s", s, (B, st.m)),
                             ("dx", dx, (B, st.n)), ("dy", dy, (B, st.m))):
            _chk(t, shp, f64, dev, name)
        if shared and st.nnzP:
            _chk(P_vals, (st.nnzP,), f64, dev, "P_vals")
        settings = settings or _lib.default_settings()
        if out is not None:
            dA, dP, db, dc, its = out
        else:
            dA = torch.empty((*lead, st.nnzA), dtype=f64, device=dev)
            db = torch.empty((B, st.m), dtype=f64, device=dev)
            dc = torch.empty((B, st.n), dtype=f64, device=dev)
            dP = torch.empty((*lead, st.nnzP), dtype=f64, device=dev) if st.nnzP else None
            its = torch.empty(B, dtype=torch.int32, device=dev)
        fn = self.lib.bcone_vjp_shared if shared else self.lib.bcone_vjp
        rc = fn(self.h, C.c_int32(B), _ptr(A_vals), _ptr(P_vals if st.nnzP else None), _ptr(b), _ptr(c),
                _ptr(x), _ptr(y), _ptr(s), _ptr(dx), _ptr(dy), _ptr(dA), _ptr(dP), _ptr(db), _ptr(dc),
                _ptr(its), C.byref(settings), self._stream())
        self._raise(rc, "bcone_vjp_shared" if shared else "bcone_vjp")
        return dA, dP, db, dc, its

    def jvp(self, A_vals, b, c, x, y, s, dA, db, dc, P_vals=None, dP=None, settings: _lib.BconeSettings | None = None, out=None):
        """Forward-mode derivative of the solution map at (x, y, s) (diffcp's ``D``; the transpose of :meth:`vjp`): tangents of
        the data in engine layout -> dx[B,n], dy[B,m], ds[B,m], lsqr_iters[B]  (``out``: the same four, preallocated).
        ``dP`` None = no tangent on P.  1-D ``A_vals`` / ``P_vals`` with 1-D tangents ``dA`` / ``dP``: matrices and their
        tangents shared by the batch (``bcone_jvp_shared``)."""
        st, dev, f64 = self.structure, self.device, torch.float64
        shared = A_vals.dim() == 1
        B = b.shape[0] if shared else A_vals.shape[0]
        lead = () if shared else (B,)
        for name, t, shp in (("A_vals", A_vals, (*lead, st.nnzA)), ("b", b, (B, st.m)), ("c", c, (B, st.n)),
                             ("x", x, (B, st.n)), ("y", y, (B, st.m)), ("s", s, (B, st.m)),
                             ("dA", dA, (*lead, st.nnzA)), ("db", db, (B, st.m)), ("dc", dc, (B, st.n))):
            _chk(t, shp, f64, dev, name)
        if st.nnzP:
            if P_vals is None:
                raise ValueError("structure has a quadratic term but P_vals is None")
            _chk(P_vals, (*lead, st.nnzP), f64, dev, "P_vals")
            _chk(dP, (*lead, st.nnzP), f64, dev, "dP")
        settings = settings or _lib.default_settings()
        if out is not None:
            dx, dy, ds, its = out
        else:
            dx = torch.empty((B, st.n), dtype=f64, device=dev)
            dy = torch.empty((B, st.m), dtype=f64, device=dev)
            ds = torch.empty((B, st.m), dtype=f64, device=dev)
            its = torch.empty(B, dtype=torch.int32, device=dev)
        fn = self.lib.bcone_jvp_shared if shared else self.lib.bcone_jvp
        rc = fn(self.h, C.c_int32(B), _ptr(A_vals), _ptr(P_vals if st.nnzP else None), _ptr(b), _ptr(c),
                _ptr(x), _ptr(y), _ptr(s), _ptr(dA), _ptr(dP if st.nnzP else None), _ptr(db), _ptr(dc),
                _ptr(dx), _ptr(dy), _ptr(ds), _ptr(its), C.byref(settings), self._stream())
        self._raise(rc, "bcone_jvp_shared" if shared else "bcone_jvp")
        return dx, dy, ds, its
