"""Drop-in solver interface (solver name "B200"): the GPU twin of ``cvxpylayers/interfaces/diffcp_if.py``.

Mirrors, name for name and argument for argument, what the reference's torch layer expects of a
backend (SURVEY.md section 8b):

* ``B200_ctx(objective_structure, constraint_structure, dims, lower_bounds, upper_bounds, options)``
  -- same constructor as ``DIFFCP_ctx`` (``diffcp_if.py:105-120``): the CSC structure
  ``(indices, indptr, (m, n+1))`` of ``[A_cvx | b]`` and cvxpy's cone dims.
* ``_CvxpyLayer.apply(P_eval, q_eval, A_eval, cl_ctx, solver_args, needs_grad, warm_start)``
  -> ``(primal[B,n], dual[B,m], opaque, opaque)`` -- same call the layer makes at
  ``torch/cvxpylayer.py:475-483``; backward returns the 7-tuple of ``diffcp_if.py:403``.

Differences from DIFFCP, all deliberate and documented in DESIGN.md: tensors stay on the GPU
(CPU inputs are copied in and results copied back, so outputs live where the inputs live,
as ``tests/test_moreau.py:787-815`` requires of a GPU backend); a native quadratic ``P`` is accepted
(``moreau_if.py:400-426`` convention, upper triangle); the gradient covers *every* structural
entry of ``A`` (the reference's ``dA.data`` drops exact zeros, SURVEY.md 8a note).
"""
from __future__ import annotations

import os
from types import SimpleNamespace
import sys
import time
import warnings
from typing import Any

import numpy as np
import scipy.sparse as sp
import torch

from . import _lib
from .engine import STATUS, Engine, make_settings
from .structure import ConeSpec, Structure

try:  # raise the reference's own exception type when diffcp is importable (tests/test_torch.py:299-316)
    from diffcp import SolverError as _SolverErrorBase  # type: ignore
except Exception:  # noqa: BLE001
    _SolverErrorBase = Exception


_TRACE = bool(os.environ.get("B200_TRACE"))


class SolverError(_SolverErrorBase):
    """Raised when an instance is infeasible / unbounded / failed, like ``diffcp.SolverError``."""


def dims_to_solver_dict(dims: Any) -> dict:
    """cvxpy ``ConeDims`` -> {"z","l","q","s","ep","ed","p"} (the conversion the reference imports
    from cvxpy at ``diffcp_if.py:8``); plain dicts pass through."""
    if isinstance(dims, dict):
        return dims
    if isinstance(dims, ConeSpec):
        return dims.to_dict()
    out = {"z": int(getattr(dims, "zero", 0)), "l": int(getattr(dims, "nonneg", 0)),
           "q": [int(v) for v in getattr(dims, "soc", [])], "s": [int(v) for v in getattr(dims, "psd", [])],
           "ep": int(getattr(dims, "exp", 0)), "ed": 0}
    p3d = getattr(dims, "p3d", [])
    if len(p3d):
        out["p"] = list(p3d)
    return out


def _detect_batch_size(con_values: torch.Tensor) -> tuple[int, bool]:
    """Same rule as ``diffcp_if.py:34-43``: 1-D values = one unbatched instance."""
    if con_values.dim() == 1:
        return 1, True
    return con_values.shape[1], False


class B200_ctx:
    """Per-layer solver context (twin of ``DIFFCP_ctx``, ``diffcp_if.py:99-120``)."""

    def __init__(self, objective_structure, constraint_structure, dims, lower_bounds=None, upper_bounds=None,
                 options=None, device: str | torch.device | None = None):
        con_indices, con_ptr, (m, np1) = constraint_structure
        con_indices = np.asarray(con_indices)
        con_ptr = np.asarray(con_ptr)
        n = np1 - 1
        self.A_structure = (con_indices, con_ptr)
        self.A_shape = (m, np1)
        self.b_idx = con_indices[con_ptr[-2]: con_ptr[-1]]
        self.dims = dims
        self.options = options or {}
        self.device = device
        nnzA = int(con_ptr[-2])
        # CSC (boundary order) -> CSR (engine order): gather[k] = boundary row feeding CSR slot k
        csc = sp.csc_matrix((np.arange(1, nnzA + 1), con_indices[:nnzA], con_ptr[:-1]), shape=(m, n))
        csr = csc.tocsr()
        csr.sort_indices()
        self.gather = (csr.data - 1).astype(np.int32)
        P_indptr = P_indices = None
        self.nnzP = 0          # engine slots (upper triangle)
        self.nnzP_boundary = 0  # rows of P_eval
        self.gatherP = None
        if objective_structure is not None:
            # cvxpy's CSC structure (indices = rows, indptr over columns) of a symmetric P, exactly what DIFFCP_ctx is
            # handed (reduced_P.problem_data_index, interfaces/__init__.py:27-34).  Any symmetric pattern is accepted:
            # upper, lower or full.  The engine stores the upper triangle in CSR order; slot (i, j), i <= j, is fed by
            # the boundary row of entry (i, j) if present, else by its mirror (j, i).  (The CSR upper triangle, which the
            # CSR-route backends get, is the CSC lower triangle of the same matrix and lands on the identity map.)
            p_indices, p_ptr, _ = objective_structure
            p_indices, p_ptr = np.asarray(p_indices), np.asarray(p_ptr)
            nb_ = int(p_indices.size)
            cols = np.repeat(np.arange(n), np.diff(p_ptr))
            rows = p_indices.astype(np.int64)
            lo, hi = np.minimum(rows, cols), np.maximum(rows, cols)
            order = np.lexsort((rows > cols, hi, lo))   # by slot (lo, hi); the true upper entry first when both exist
            key = lo[order] * n + hi[order]
            first = np.ones(nb_, dtype=bool)
            first[1:] = key[1:] != key[:-1]
            sel = order[first]
            P_indices = hi[sel].astype(np.int32)
            P_indptr = np.concatenate([[0], np.cumsum(np.bincount(lo[sel], minlength=n))]).astype(np.int32)
            self.gatherP = sel.astype(np.int32)
            self.nnzP = int(sel.size)
            self.nnzP_boundary = nb_
        cones = ConeSpec.from_dict(dims_to_solver_dict(dims))
        self.structure = Structure(n, m, csr.indptr.astype(np.int32), csr.indices.astype(np.int32), cones,
                                   P_indptr, P_indices)
        self._engines: dict[torch.device, Engine] = {}

    def engine(self, device: torch.device) -> Engine:
        eng = self._engines.get(device)
        if eng is None:
            eng = Engine(self.structure, device)
            eng.set_boundary(self.gather, np.asarray(self.b_idx, dtype=np.int32))
            if self.nnzP:
                eng.set_boundary_P(self.nnzP_boundary, self.gatherP)
            if getattr(self, "_param_maps", None) is not None:
                eng.set_param_maps(*self._param_maps)
            self._engines[device] = eng
        return eng

    def set_param_maps(self, A_map, q_map, P_map=None):
        """Register the layer's parameter -> matrix maps (SciPy CSR [rows x P1], boundary row order: the reference's
        ``_A_scipy`` / ``_q_scipy`` / ``_P_scipy``, ``torch/cvxpylayer.py:443-451``) so that
        :class:`_CvxpyLayerFused` can take ``p_stack`` instead of the evaluated matrices."""
        self._param_maps = (A_map, q_map, P_map if self.nnzP else None)
        # The reference's `PA_is_constant` (interfaces/moreau_if.py:233-241): no entry of A or P depends on a parameter (only the
        # constant column of their rows is populated), so the equilibration and the factorisation of a call stay valid for
        # the next one.  (The trailing rows of A_map feed b and may depend on parameters.)
        try:
            nA = A_map.shape[0] - len(self.b_idx)
            self.PA_is_constant = bool(A_map.tocsr()[:nA, :-1].nnz == 0 and (P_map is None or not self.nnzP or P_map.tocsr()[:, :-1].nnz == 0))
        except Exception:  # noqa: BLE001  (a map that is not a SciPy matrix: no claim)
            self.PA_is_constant = False
        for eng in self._engines.values():
            eng.set_param_maps(*self._param_maps)

    # ---- warm starts (SURVEY.md 8f.2): the previous call's solution seeds the next one ({"warm_start": True}) ----
    def warm_for(self, dev: torch.device, B: int, warm_start, merged: dict):
        """What to start from: an explicit (x0, y0, s0) / Solution passed as ``warm_start``, else -- when the option
        ``warm_start`` is on -- the cached solution of the previous call with the same batch size on this device (the
        reference's rule for its one warm-startable backend, ``torch/cvxpylayer.py:464-473``)."""
        if warm_start is not None and not isinstance(warm_start, bool):
            ws = (warm_start.x, warm_start.y, warm_start.s) if hasattr(warm_start, "x") else tuple(warm_start)
            return tuple(t.detach().to(device=dev, dtype=torch.float64).contiguous() for t in ws)
        if warm_start is True or merged.get("warm_start"):
            return getattr(self, "_last_solution", {}).get((dev, B))
        return None

    def remember(self, dev: torch.device, B: int, sol, merged: dict, warm_start) -> None:
        if warm_start is True or merged.get("warm_start"):
            if not hasattr(self, "_last_solution"):
                self._last_solution = {}
            self._last_solution[(dev, B)] = (sol.x.detach(), sol.y.detach(), sol.s.detach())

    # ---- cached set-up (SURVEY.md 8f.2): equilibration + factorisation kept across calls while A and P do not change ----
    def setup_cache(self, eng: Engine, dev: torch.device, B: int, merged: dict):
        """The set-up cache of (device, batch size) when the option ``reuse_setup`` is on -- explicitly (the caller states that
        A and P are the same on every call), or by default when the parameter maps show it (``PA_is_constant``) -- else None.
        The engine validates every record itself, so a fresh (zero-filled) cache is simply filled by its first solve."""
        if merged.get("shared_matrices"):
            if merged.get("reuse_setup"):
                raise ValueError("shared_matrices and reuse_setup exclude each other: a shared-matrix solve builds one set-up per call")
            return None   # (nor the automatic PA_is_constant cache: the batch shares one set-up per call instead)
        if not merged.get("reuse_setup", getattr(self, "PA_is_constant", False)):
            return None
        if not hasattr(self, "_setup_cache"):
            self._setup_cache = {}
        key = (dev, B)
        if key not in self._setup_cache:
            self._setup_cache[key] = eng.new_cache(B)   # None: this structure has no cached path
        return self._setup_cache[key]

    def check_shared_matrices(self, sizes, batched, col_order) -> None:
        """With ``shared_matrices`` every parameter whose p_stack rows feed A (the first nnzA rows of the A map) or P must be
        unbatched: the layer evaluates A and P from the first instance only.  Per user parameter i: ``sizes[i]`` entries,
        ``batched[i]``, ``col_order[i]`` (the reference's ``user_order_to_col_order``); p_stack holds the parameters' rows in
        column order (``_flatten_and_batch_params``).  Raises ValueError naming the first batched one."""
        maps = getattr(self, "_param_maps", None)
        if maps is None:
            return
        A_map, _, P_map = maps
        nA = A_map.shape[0] - len(self.b_idx)
        used = set(sp.csr_matrix(A_map)[:nA, :-1].indices.tolist())
        if P_map is not None:
            used |= set(sp.csr_matrix(P_map)[:, :-1].indices.tolist())
        acc = 0
        for i in sorted(range(len(sizes)), key=lambda i: col_order[i]):
            rows = range(acc, acc + sizes[i])
            acc += sizes[i]
            if batched[i] and any(r in used for r in rows):
                raise ValueError(f"shared_matrices: parameter {i} feeds A or P but is batched; the matrices must come from "
                                 "unbatched parameters")

    def compute_device(self, t: torch.Tensor) -> torch.device:
        if t.is_cuda:
            return t.device
        if self.device is not None:
            return torch.device(self.device)
        if not torch.cuda.is_available():
            raise _lib.EngineUnavailable("no CUDA device: the B200 backend has no CPU fallback")
        return torch.device("cuda", torch.cuda.current_device())


class _Saved:
    """Opaque carrier for the tensors the backward needs (kept out of autograd's sight)."""

    def __init__(self, *items):
        self.items = items


def _forward_ad_active() -> bool:
    """Inside ``torch.autograd.forward_ad.dual_level()``: a Function's ``jvp`` may run for dual inputs that do not require
    grad, so what it needs is kept whatever ``needs_grad`` says (the reference computes that from ``requires_grad`` only)."""
    from torch.autograd import forward_ad  # noqa: PLC0415

    return forward_ad._current_level >= 0


def _tangent(t: torch.Tensor | None, rows: int, B: int, unbatched: bool, dev: torch.device) -> torch.Tensor:
    """A boundary-layout input tangent [rows, B] on the engine's device; None (no tangent) is zero."""
    if t is None:
        return torch.zeros((rows, B), dtype=torch.float64, device=dev)
    return _to_dev(t.unsqueeze(1) if unbatched else t, dev)


def _to_dev(t: torch.Tensor | None, dev: torch.device) -> torch.Tensor | None:
    """Host -> device (asynchronous DMA when the caller's tensor is pinned)."""
    if t is None:
        return None
    return t.detach().to(device=dev, dtype=torch.float64, non_blocking=True).contiguous()


def _to_host_like(t: torch.Tensor | None, device: torch.device, dtype: torch.dtype) -> torch.Tensor | None:
    """Device -> the caller's device.  CPU results land in pinned memory (torch's caching host
    allocator recycles the blocks) so the copy is one asynchronous DMA instead of a staged
    pageable copy; the stream is synchronised before the tensor is handed out."""
    if t is None:
        return None
    if device.type != "cpu":
        return t.to(device=device, dtype=dtype)
    out = torch.empty(t.shape, dtype=dtype, pin_memory=True)
    out.copy_(t if t.dtype == dtype else t.to(dtype), non_blocking=True)
    return out


PIPE_CHUNK = int(os.environ.get("B200_PIPE_CHUNK", "1024"))   # instances per pipeline stage (host-resident inputs)


def _chunks(B: int):
    n = max(1, B // max(PIPE_CHUNK, 1))
    base, extra = divmod(B, n)
    lo = 0
    for k in range(n):
        hi = lo + base + (1 if k < extra else 0)
        yield lo, hi
        lo = hi


def _pipe_ok(eng: Engine, B: int, *tensors) -> bool:
    """Host-resident, pinned, contiguous fp64 inputs and a batch worth splitting: overlap the PCIe copies
    with the solve by running batch slices on two streams."""
    if B < 2 * PIPE_CHUNK or PIPE_CHUNK <= 0:
        return False
    info = eng.kernel_info()
    for t in tensors:
        if t is None:
            continue
        if t.device.type != "cpu" or t.dtype != torch.float64 or not t.is_contiguous() or not t.is_pinned():
            return False
    return info["fwd_smem"] > 0


def _stage_ok(B: int, *tensors) -> bool:
    """Host-resident but NOT pinned inputs (what the reference's own CPU path hands over: ``torch.from_numpy`` results of its sparse
    products, ``torch/cvxpylayer.py:21-24``) and a batch worth splitting: batch slices are gathered into a small ring of pinned
    staging buffers by a background thread while the previous slice is copied and solved."""
    if B < 2 * PIPE_CHUNK or PIPE_CHUNK <= 0 or os.environ.get("B200_NO_STAGING"):
        return False
    return all(t is None or (t.device.type == "cpu" and t.dim() == 2 and t.dtype == torch.float64) for t in tensors)


_STAGE_SLOTS = 3


def _stager(eng: Engine):
    """The staging state of one engine (ring buffers + two thread pools), created on first use.  Like the engine itself it serves one
    forward call at a time: concurrent calls on the SAME engine from several Python threads would share the ring (one engine per
    thread, or a lock around the call, as for every other per-engine resource -- INTEGRATION.md)."""
    sg = getattr(eng, "_stager", None)
    if sg is None:
        from concurrent.futures import ThreadPoolExecutor  # noqa: PLC0415

        nthr = int(os.environ.get("B200_STAGE_THREADS", "8"))
        sg = SimpleNamespace(pool=ThreadPoolExecutor(max_workers=1, thread_name_prefix="b200-stage"),          # one slice at a time, in order
                             copiers=ThreadPoolExecutor(max_workers=nthr, thread_name_prefix="b200-copy"),   # ... gathered by row blocks
                             nthr=nthr, bufs={})
        eng._stager = sg
    return sg


def _side_streams(eng: Engine, dev):
    """The two pipeline streams of an engine, created once: torch's device allocator keeps one block pool per
    stream, so fresh streams per call would cudaMalloc every chunk buffer again (tens of ms per step)."""
    ss = getattr(eng, "_pipe_streams", None)
    if ss is None:
        ss = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
        eng._pipe_streams = ss
    return ss


def _post_options(eng: Engine, merged: dict) -> tuple[bool, int]:
    """The layer options ``polish`` and ``refine`` -> (polish, refinement steps; 0 = off), refused (ValueError) before anything
    is staged or solved: both at once, a ``refine`` other than a bool or an int in 1 ... 10 (True = 3 steps), or a structure
    without the plan the option needs."""
    polish, refine = bool(merged.get("polish")), merged.get("refine", False)
    if refine is None or refine is False:
        refine = 0
    elif refine is True:
        refine = 3
    elif not isinstance(refine, (int, np.integer)) or not 1 <= int(refine) <= 10:
        raise ValueError(f"refine: expected True or an int in 1 ... 10, got {refine!r}")
    refine = int(refine)
    if polish and refine:
        raise ValueError("the layer options polish and refine exclude each other")
    if polish:
        eng.require_polish()
    if refine:
        eng.require_refine()
    return polish, refine


def _forward_pipelined(eng: Engine, dev, A_eval, q_eval, P_eval, settings, use_P, warm=None, cache=None, staged: bool = False,
                       polish: bool = False, refine: int = 0):
    st = eng.structure
    B = A_eval.shape[1]
    cstride = (cache.numel() // B) if cache is not None else 0
    f64 = torch.float64
    A_vals = torch.empty((B, st.nnzA), dtype=f64, device=dev)
    b = torch.empty((B, st.m), dtype=f64, device=dev)
    c = torch.empty((B, st.n), dtype=f64, device=dev)
    P_vals = torch.empty((B, st.nnzP), dtype=f64, device=dev) if use_P else None
    sol = eng.alloc_solution(B)
    primal = torch.empty((B, st.n), dtype=f64, pin_memory=True)
    dual = torch.empty((B, st.m), dtype=f64, pin_memory=True)
    cur = torch.cuda.current_stream(dev)
    streams = _side_streams(eng, dev)
    for s_ in streams:
        s_.wait_stream(cur)
    chunks = list(_chunks(B))
    futs = enq = cev = None
    if staged:
        # Pageable (or non-fp64) host inputs: a background thread gathers slice k into pinned staging buffers (the gather is
        # split over a few copy threads) while slice k-1 is on its way; a slot of the ring is rewritten only after the device copy that read
        # it has completed (per-call handshake: the main thread publishes the event, the stager waits for it).
        import threading  # noqa: PLC0415

        sg = _stager(eng)
        enq = [threading.Event() for _ in chunks]
        cev = [None] * len(chunks)
        abort = threading.Event()   # set when the main thread leaves early (an exception): the stager must not wait for it
        srcs = (("A", A_eval), ("q", q_eval), ("P", P_eval if use_P else None))

        def stage(k, lo, hi):
            if k >= _STAGE_SLOTS:
                while not enq[k - _STAGE_SLOTS].wait(0.05):
                    if abort.is_set():
                        return None
                cev[k - _STAGE_SLOTS].synchronize()
            out = []
            for name, src in srcs:
                if src is None:
                    out.append(None)
                    continue
                key = (k % _STAGE_SLOTS, name, src.shape[0], hi - lo)
                buf = sg.bufs.get(key)
                if buf is None:
                    buf = torch.empty((src.shape[0], hi - lo), dtype=f64, pin_memory=True)
                    sg.bufs[key] = buf
                rows = src.shape[0]
                step = max(256, -(-rows // sg.nthr))   # a strided gather is one core's memcpy: split it by row blocks
                if rows <= step:
                    buf.copy_(src[:, lo:hi])
                else:
                    list(sg.copiers.map(lambda r0, buf=buf, src=src: buf[r0:r0 + step].copy_(src[r0:r0 + step, lo:hi]), range(0, rows, step)))
                out.append(buf)
            return out

        futs = [sg.pool.submit(stage, k, lo, hi) for k, (lo, hi) in enumerate(chunks)]
    try:   # any exception leaving the chunk loop (a failed copy, solve, polish or refinement) releases the stager
        for k, (lo, hi) in enumerate(chunks):
            with torch.cuda.stream(streams[k % 2]):
                Bc = hi - lo
                A_c = torch.empty((A_eval.shape[0], Bc), dtype=f64, device=dev)
                q_c = torch.empty((q_eval.shape[0], Bc), dtype=f64, device=dev)
                P_c = torch.empty((P_eval.shape[0], Bc), dtype=f64, device=dev) if use_P else None
                if staged:
                    hA_, hq_, hP_ = futs[k].result()
                    A_c.copy_(hA_, non_blocking=True)
                    q_c.copy_(hq_, non_blocking=True)
                    if use_P:
                        P_c.copy_(hP_, non_blocking=True)
                    cev[k] = torch.cuda.Event()
                    cev[k].record(streams[k % 2])
                    enq[k].set()
                else:
                    eng.copy2d(A_c, A_eval, lo, hi, True)
                    eng.copy2d(q_c, q_eval, lo, hi, True)
                    if use_P:
                        eng.copy2d(P_c, P_eval, lo, hi, True)
                eng.ingest(A_c, q_c, P_c, out=(A_vals[lo:hi], P_vals[lo:hi] if use_P else None, b[lo:hi], c[lo:hi]))
                from .engine import Solution  # noqa: PLC0415
                sol_c = Solution(sol.x[lo:hi], sol.y[lo:hi], sol.s[lo:hi], sol.status[lo:hi], sol.iters[lo:hi], sol.resid[lo:hi])
                eng.solve(A_vals[lo:hi], b[lo:hi], c[lo:hi], P_vals[lo:hi] if use_P else None, settings, out=sol_c,
                          warm=None if warm is None else tuple(w_[lo:hi] for w_ in warm),
                          cache=None if cache is None else cache[lo * cstride:hi * cstride], reuse=True)
                if polish:
                    eng.polish(A_vals[lo:hi], b[lo:hi], c[lo:hi], sol_c, P_vals[lo:hi] if use_P else None, settings)
                if refine:
                    eng.refine(A_vals[lo:hi], b[lo:hi], c[lo:hi], sol_c, P_vals[lo:hi] if use_P else None, settings, refine)
                primal[lo:hi].copy_(sol.x[lo:hi], non_blocking=True)
                dual[lo:hi].copy_(sol.y[lo:hi], non_blocking=True)
    except BaseException:
        if staged:
            abort.set()   # (the stager must not wait for a slice that will never be copied)
        raise
    for s_ in streams:
        cur.wait_stream(s_)
    return A_vals, P_vals, b, c, sol, primal, dual


def _backward_pipelined(eng: Engine, dev, settings, A_vals, P_vals, b, c, x, y, s, dprimal, ddual, use_P, nnz_aug):
    st = eng.structure
    B = A_vals.shape[0]
    f64 = torch.float64
    _t0 = time.perf_counter()
    dA_eval = torch.empty((nnz_aug, B), dtype=f64, pin_memory=True)
    dq_eval = torch.empty((st.n + 1, B), dtype=f64, pin_memory=True)
    dP_eval = torch.empty((st.nnzP, B), dtype=f64, pin_memory=True) if use_P else None
    _t1 = time.perf_counter()
    _evs = []
    dx = dprimal.detach().to(device=dev, dtype=f64, non_blocking=True).reshape(B, -1).contiguous()
    dy = ddual.detach().to(device=dev, dtype=f64, non_blocking=True).reshape(B, -1).contiguous()
    cur = torch.cuda.current_stream(dev)
    streams = _side_streams(eng, dev)
    for s_ in streams:
        s_.wait_stream(cur)
    for k, (lo, hi) in enumerate(_chunks(B)):
        with torch.cuda.stream(streams[k % 2]):
            if _TRACE:
                _e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                _e[0].record()
            gA, gP, gb, gc, _ = eng.vjp(A_vals[lo:hi], b[lo:hi], c[lo:hi], x[lo:hi], y[lo:hi], s[lo:hi], dx[lo:hi], dy[lo:hi],
                                        P_vals[lo:hi] if P_vals is not None else None, settings)
            gA_e, gq_e, gP_e = eng.emit(gA, gP if use_P else None, gb, gc)
            if _TRACE:
                _e[1].record()
            eng.copy2d(dA_eval, gA_e, lo, hi, False)
            eng.copy2d(dq_eval, gq_e, lo, hi, False)
            if use_P:
                eng.copy2d(dP_eval, gP_e, lo, hi, False)
            if _TRACE:
                _e[2].record()
                _evs.append(_e)
    for s_ in streams:
        cur.wait_stream(s_)
    _t2 = time.perf_counter()
    cur.synchronize()
    if _TRACE:
        _t3 = time.perf_counter()
        print(f"[b200] bwd: pinned alloc {1e3 * (_t1 - _t0):.1f} ms, enqueue {1e3 * (_t2 - _t1):.1f} ms, drain {1e3 * (_t3 - _t2):.1f} ms; chunks (compute, d2h) "
              + ", ".join(f"({e[0].elapsed_time(e[1]):.1f}, {e[1].elapsed_time(e[2]):.1f})" for e in _evs), file=sys.stderr)
    return dA_eval, dq_eval, dP_eval


class _CvxpyLayer(torch.autograd.Function):
    """Twin of ``diffcp_if._CvxpyLayer`` (``diffcp_if.py:327-403``)."""

    @staticmethod
    def forward(P_eval, q_eval, A_eval, cl_ctx, solver_args, needs_grad=True, warm_start=None):
        ctx: B200_ctx = cl_ctx.solver_ctx
        batch_size, originally_unbatched = _detect_batch_size(A_eval)
        if originally_unbatched:
            A_eval = A_eval.unsqueeze(1)
            q_eval = q_eval.unsqueeze(1)
            P_eval = P_eval.unsqueeze(1) if P_eval is not None else None
        in_device, in_dtype = A_eval.device, A_eval.dtype
        dev = ctx.compute_device(A_eval)
        eng = ctx.engine(dev)
        merged = {**ctx.options}
        if solver_args:
            merged.update(solver_args)
        settings = make_settings(merged)
        use_P = P_eval is not None and ctx.nnzP > 0
        warm = ctx.warm_for(dev, batch_size, warm_start, merged)
        cache = ctx.setup_cache(eng, dev, batch_size, merged)
        piped = _pipe_ok(eng, batch_size, A_eval.detach(), q_eval.detach(), P_eval.detach() if use_P else None)
        staged = (not piped) and eng.kernel_info()["fwd_smem"] > 0 and _stage_ok(batch_size, A_eval, q_eval, P_eval if use_P else None)
        piped = piped or staged
        # polish / refine: the solution is polished or refined right after the solve, so the backward, the forward mode and the
        # next warm start all see that point
        polish, refine = _post_options(eng, merged)   # (before any chunk is staged or solved)
        with torch.cuda.device(dev):
            if piped:
                A_vals, P_vals, b, c, sol, primal, dual = _forward_pipelined(
                    eng, dev, A_eval.detach(), q_eval.detach(), P_eval.detach() if use_P else None, settings, use_P, warm, cache, staged,
                    polish, refine)
            else:
                A_vals, P_vals, b, c = eng.ingest(_to_dev(A_eval, dev), _to_dev(q_eval, dev),
                                                  _to_dev(P_eval, dev) if use_P else None)
                sol = eng.solve(A_vals, b, c, P_vals, settings, warm=warm, cache=cache, reuse=True)
                if polish:
                    eng.polish(A_vals, b, c, sol, P_vals, settings)
                if refine:
                    eng.refine(A_vals, b, c, sol, P_vals, settings, refine)
            status = sol.status.cpu()  # the one host sync of the forward: per-instance status
        ctx.remember(dev, batch_size, sol, merged, warm_start)
        bad = (status != 1) & (status != 2)
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0])
            raise SolverError(f"instance {i}: solver returned status {STATUS.get(int(status[i]), int(status[i]))}")
        if bool((status == 2).any()):
            warnings.warn("Solved/Inaccurate.", stacklevel=2)
        if not piped:
            with torch.cuda.device(dev):
                primal = _to_host_like(sol.x, in_device, in_dtype)
                dual = _to_host_like(sol.y, in_device, in_dtype)
                if in_device.type == "cpu":
                    torch.cuda.current_stream(dev).synchronize()
        keep = needs_grad or _forward_ad_active()
        saved = _Saved(eng, settings, A_vals, P_vals, b, c, sol.x, sol.y, sol.s, piped, A_eval.shape[0]) if keep else None
        return primal, dual, saved, (batch_size, originally_unbatched, in_device, in_dtype, use_P)

    @staticmethod
    def setup_context(ctx: Any, inputs: tuple, outputs: tuple) -> None:
        _, _, saved, backward_data = outputs
        ctx.saved = saved
        ctx.backward_data = backward_data

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx: Any, dprimal, ddual, _saved, _data):
        batch_size, originally_unbatched, in_device, in_dtype, use_P = ctx.backward_data
        if ctx.saved is None:
            raise RuntimeError("backward called on a forward pass run with needs_grad=False")
        eng, settings, A_vals, P_vals, b, c, x, y, s, piped, nnz_aug = ctx.saved.items
        dev = eng.device
        _tb = time.perf_counter() if _TRACE else 0.0
        if piped and in_dtype == torch.float64:
            with torch.cuda.device(dev):
                dA_eval, dq_eval, dP_eval = _backward_pipelined(eng, dev, settings, A_vals, P_vals, b, c, x, y, s, dprimal, ddual,
                                                                use_P, nnz_aug)
            if _TRACE:
                print(f"[b200] backward body (pipelined) {1e3 * (time.perf_counter() - _tb):.1f} ms", file=sys.stderr)
            return dP_eval, dq_eval, dA_eval, None, None, None, None
        with torch.cuda.device(dev):
            dx = _to_dev(dprimal, dev).reshape(batch_size, -1)
            dy = _to_dev(ddual, dev).reshape(batch_size, -1)
            dA_vals, dP_vals, db, dc, _ = eng.vjp(A_vals, b, c, x, y, s, dx, dy, P_vals, settings)
            dA_eval, dq_eval, dP_eval = eng.emit(dA_vals, dP_vals if use_P else None, db, dc)
            dA_eval = _to_host_like(dA_eval, in_device, in_dtype)
            dq_eval = _to_host_like(dq_eval, in_device, in_dtype)
            dP_eval = _to_host_like(dP_eval, in_device, in_dtype)
            if in_device.type == "cpu":
                torch.cuda.current_stream(dev).synchronize()
        if _TRACE:
            print(f"[b200] backward body {1e3 * (time.perf_counter() - _tb):.1f} ms", file=sys.stderr)
        if originally_unbatched:
            dq_eval = dq_eval.squeeze(1)
            dA_eval = dA_eval.squeeze(1)
            dP_eval = dP_eval.squeeze(1) if dP_eval is not None else None
        return dP_eval, dq_eval, dA_eval, None, None, None, None

    @staticmethod
    def jvp(ctx: Any, tP, tq, tA, *_):
        """Forward mode (diffcp's ``D``): the boundary tangents go through the same ingest maps as the data (they are linear),
        then ``bcone_jvp``.  Tangents come back where the outputs live; absent ones are zero."""
        batch_size, originally_unbatched, in_device, in_dtype, use_P = ctx.backward_data
        if ctx.saved is None:
            raise RuntimeError("forward-mode AD on a forward pass that kept nothing for it")
        eng, settings, A_vals, P_vals, b, c, x, y, s, _piped, nnz_aug = ctx.saved.items
        dev = eng.device
        with torch.cuda.device(dev):
            tA_e = _tangent(tA, nnz_aug, batch_size, originally_unbatched, dev)
            tq_e = _tangent(tq, eng.structure.n + 1, batch_size, originally_unbatched, dev)
            tP_e = _tangent(tP, eng._nnzP_b, batch_size, originally_unbatched, dev) if (use_P and tP is not None) else None
            dA, dP, db, dc = eng.ingest(tA_e, tq_e, tP_e)
            dx, dy, _, _ = eng.jvp(A_vals, b, c, x, y, s, dA, db, dc, P_vals, dP, settings)
            dprimal = _to_host_like(dx, in_device, in_dtype)
            ddual = _to_host_like(dy, in_device, in_dtype)
            if in_device.type == "cpu":
                torch.cuda.current_stream(dev).synchronize()
        return dprimal, ddual, None, None


def get_solver_ctx(solver, param_prob, cone_dims, data, kwargs, verbose=False):
    """Twin of ``cvxpylayers.interfaces.get_solver_ctx`` (``interfaces/__init__.py:13-69``) for the solver name
    "B200".  Like DIFFCP it takes cvxpy's CSC structures as they are (``reduced_P/A.problem_data_index``): the CSC -> CSR
    re-ordering and the upper-triangle selection of P happen inside the engine's ingest kernels, so the parametrisation
    matrices need no row permutation (what ``convert_to_csr`` does for the other CSR backends)."""
    if solver != "B200":
        raise RuntimeError("Unknown solver. Check if your solver is supported by CVXPYlayers")
    options = dict(kwargs) if kwargs else {}
    if verbose:
        options["verbose"] = True
    red_P = getattr(param_prob, "reduced_P", None)
    p_struct = getattr(red_P, "problem_data_index", None) if red_P is not None else None
    ctx = B200_ctx(p_struct, param_prob.reduced_A.problem_data_index, cone_dims,
                   data.get("lower_bound"), data.get("upper_bound"), options)
    # the fused path needs the parametrisation matrices themselves (rows in boundary order, last column = constant)
    A_mat = getattr(param_prob.reduced_A, "reduced_mat", None)
    q_mat = getattr(param_prob, "q", getattr(param_prob, "c", None))
    P_mat = getattr(red_P, "reduced_mat", None) if (red_P is not None and p_struct is not None) else None
    if A_mat is not None and q_mat is not None:
        ctx.set_param_maps(A_mat, q_mat, P_mat)
    return ctx


def get_torch_cvxpylayer(solver):
    """Twin of ``cvxpylayers.interfaces.get_torch_cvxpylayer`` (``interfaces/__init__.py:72-101``)."""
    if solver != "B200":
        raise RuntimeError("Unknown solver. Check if your solver is supported by CVXPYlayers")
    return _CvxpyLayer


class _CvxpyLayerFused(torch.autograd.Function):
    """``p_stack -> (primal, dual)`` with the parameter -> matrix affine map fused into the engine's load stage and its
    transpose into the gradient write-back (SURVEY.md 8f.1): replaces the three sparse products at
    ``torch/cvxpylayer.py:443-451`` + ``_CvxpyLayer.apply`` + their transposes (``:33-37``).  ``p_stack[P1, B]`` is what
    ``_flatten_and_batch_params`` builds (last row = 1).  Only parameters and parameter gradients cross PCIe."""

    @staticmethod
    def forward(p_stack, cl_ctx, solver_args, needs_grad=True, warm_start=None):
        ctx: B200_ctx = cl_ctx.solver_ctx
        unb = p_stack.dim() == 1
        ps = p_stack.unsqueeze(1) if unb else p_stack
        in_device, in_dtype = ps.device, ps.dtype
        dev = ctx.compute_device(ps)
        eng = ctx.engine(dev)
        merged = {**ctx.options, **(solver_args or {})}
        settings = make_settings(merged)
        B = ps.shape[1]
        # shared_matrices: the caller states that A and P are the same for every instance (their parameters are unbatched);
        # they are evaluated once and the batch shares them through solve, adjoint and forward mode
        shared = bool(merged.get("shared_matrices"))
        polish, refine = _post_options(eng, merged)
        with torch.cuda.device(dev):
            cache = ctx.setup_cache(eng, dev, B, merged)
            A_vals, P_vals, b, c = eng.ingest_params(_to_dev(ps, dev), shared=shared)
            sol = eng.solve(A_vals, b, c, P_vals, settings, warm=ctx.warm_for(dev, B, warm_start, merged), cache=cache, reuse=True)
            # (before the solution is kept for the backward, the forward mode and the next warm start)
            if polish:
                eng.polish(A_vals, b, c, sol, P_vals, settings)
            if refine:
                eng.refine(A_vals, b, c, sol, P_vals, settings, refine)
            status = sol.status.cpu()
        ctx.remember(dev, B, sol, merged, warm_start)
        bad = (status != 1) & (status != 2)
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0])
            raise SolverError(f"instance {i}: solver returned status {STATUS.get(int(status[i]), int(status[i]))}")
        if bool((status == 2).any()):
            warnings.warn("Solved/Inaccurate.", stacklevel=2)
        with torch.cuda.device(dev):
            primal = _to_host_like(sol.x, in_device, in_dtype)
            dual = _to_host_like(sol.y, in_device, in_dtype)
            if in_device.type == "cpu":
                torch.cuda.current_stream(dev).synchronize()
        saved = _Saved(eng, settings, A_vals, P_vals, b, c, sol.x, sol.y, sol.s) if (needs_grad or _forward_ad_active()) else None
        return primal, dual, saved, (unb, in_device, in_dtype)

    @staticmethod
    def setup_context(ctx: Any, inputs: tuple, outputs: tuple) -> None:
        ctx.saved, ctx.backward_data = outputs[2], outputs[3]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx: Any, dprimal, ddual, _saved, _data):
        unb, in_device, in_dtype = ctx.backward_data
        if ctx.saved is None:
            raise RuntimeError("backward called on a forward pass run with needs_grad=False")
        eng, settings, A_vals, P_vals, b, c, x, y, s = ctx.saved.items
        dev = eng.device
        B = b.shape[0]
        with torch.cuda.device(dev):
            dA, dP, db, dc, _ = eng.vjp(A_vals, b, c, x, y, s, _to_dev(dprimal, dev).reshape(B, -1), _to_dev(ddual, dev).reshape(B, -1), P_vals, settings)
            dp = _to_host_like(eng.emit_params(dA, dP, db, dc, shared=A_vals.dim() == 1), in_device, in_dtype)
            if in_device.type == "cpu":
                torch.cuda.current_stream(dev).synchronize()
        return (dp.squeeze(1) if unb else dp), None, None, None, None

    @staticmethod
    def jvp(ctx: Any, tp, *_):
        """Forward mode: the tangent of ``p_stack`` through the parameter maps (linear in ``p_stack``), then ``bcone_jvp``."""
        unb, in_device, in_dtype = ctx.backward_data
        if ctx.saved is None:
            raise RuntimeError("forward-mode AD on a forward pass that kept nothing for it")
        eng, settings, A_vals, P_vals, b, c, x, y, s = ctx.saved.items
        dev = eng.device
        B = b.shape[0]
        with torch.cuda.device(dev):
            dA, dP, db, dc = eng.ingest_params(_tangent(tp, eng._P1, B, unb, dev), shared=A_vals.dim() == 1)
            dx, dy, _, _ = eng.jvp(A_vals, b, c, x, y, s, dA, db, dc, P_vals, dP, settings)
            dprimal = _to_host_like(dx, in_device, in_dtype)
            ddual = _to_host_like(dy, in_device, in_dtype)
            if in_device.type == "cpu":
                torch.cuda.current_stream(dev).synchronize()
        return dprimal, ddual, None, None


_REGISTERED = False
_FORCE_B200 = False


def register(canon_solver: str = "DIFFCP", fuse: bool = True) -> None:
    """Patch an importable ``cvxpylayers`` so that ``CvxpyLayer(problem, ..., solver="B200")`` works unmodified
    (SURVEY.md 8f.4; INTEGRATION.md shows the same change as a source patch):

    * ``utils.parse_args.parse_args`` is wrapped: cvxpy does not know a solver called "B200", so the problem is
      canonicalised for ``canon_solver`` (default "DIFFCP": quad_form -> SOC, ``_quad_form_dpp.py:29-32``; pass the name of
      a cvxpy solver with a quadratic objective, e.g. "CLARABEL", together with a cvxpylayers whose
      ``SUPPORTS_QUAD_OBJ`` lists it to keep ``P``), while the context that comes back carries ``solver = "B200"`` and a
      :class:`B200_ctx` (``parse_args.py:447-462`` is where the name reaches cvxpy);
    * ``interfaces.get_solver_ctx`` / ``get_torch_cvxpylayer`` dispatch the new name (the reference's dispatch is a closed
      ``match``, ``interfaces/__init__.py:44-69,81-101``);
    * with ``fuse=True`` the torch layer's ``forward`` hands ``p_stack`` to :class:`_CvxpyLayerFused` instead of evaluating
      ``A_eval``/``q_eval``/``P_eval`` first (``torch/cvxpylayer.py:434-487``)."""
    global _REGISTERED
    import dataclasses  # noqa: PLC0415
    import importlib  # noqa: PLC0415

    ifs = importlib.import_module("cvxpylayers.interfaces")
    pa = importlib.import_module("cvxpylayers.utils.parse_args")
    if _REGISTERED and getattr(ifs.get_solver_ctx, "_b200", False):
        return
    orig_ctx, orig_layer, orig_parse = ifs.get_solver_ctx, ifs.get_torch_cvxpylayer, pa.parse_args

    def _ctx(solver, param_prob, cone_dims, data, kwargs, verbose=False):
        if solver == "B200" or _FORCE_B200:
            return get_solver_ctx("B200", param_prob, cone_dims, data, kwargs, verbose)
        return orig_ctx(solver, param_prob, cone_dims, data, kwargs, verbose)

    def _layer(solver):
        return _CvxpyLayer if solver == "B200" else orig_layer(solver)

    def _parse(problem, variables, parameters, solver, *args, **kwargs):
        global _FORCE_B200
        if solver != "B200":
            return orig_parse(problem, variables, parameters, solver, *args, **kwargs)
        _FORCE_B200 = True
        try:
            ctx = orig_parse(problem, variables, parameters, canon_solver, *args, **kwargs)
        finally:
            _FORCE_B200 = False
        try:
            return dataclasses.replace(ctx, solver="B200")
        except TypeError:   # not a dataclass (stubs): plain attribute
            ctx.solver = "B200"
            return ctx

    _ctx._b200 = True
    ifs.get_solver_ctx, ifs.get_torch_cvxpylayer, pa.parse_args = _ctx, _layer, _parse
    if fuse:
        try:
            tl = importlib.import_module("cvxpylayers.torch.cvxpylayer")
        except Exception:  # noqa: BLE001
            tl = None
        if tl is not None and hasattr(tl, "CvxpyLayer"):
            orig_forward = tl.CvxpyLayer.forward

            def _forward(self, *params, solver_args=None, warm_start=False, **kw):
                sctx = getattr(self.ctx, "solver_ctx", None)
                if getattr(self.ctx, "solver", None) != "B200" or getattr(sctx, "_param_maps", None) is None:
                    return orig_forward(self, *params, solver_args=solver_args, warm_start=warm_start, **kw)
                batch = self.ctx.validate_params(list(params))
                if {**sctx.options, **(solver_args or {})}.get("shared_matrices") and hasattr(self.ctx, "batch_sizes"):
                    bs = self.ctx.batch_sizes
                    sizes = [int(np.prod(p.shape[1:] if bs[i] else p.shape, dtype=np.int64)) for i, p in enumerate(params)]
                    sctx.check_shared_matrices(sizes, [bool(v) for v in bs], self.ctx.user_order_to_col_order)
                on_dev = all(p.is_cuda and p.dtype == torch.float64 for p in params) and hasattr(self.ctx, "batch_sizes")
                if on_dev:   # prologue as index-map launches (layer_io.py, SURVEY.md 8f.3), GP log folded in
                    from . import layer_io  # noqa: PLC0415
                    p_stack = layer_io.flatten_and_batch_params(tuple(params), self.ctx, batch)
                else:
                    params_ = tl._apply_gp_log_transform(params, self.ctx)
                    p_stack = tl._flatten_and_batch_params(params_, self.ctx, batch)
                needs_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
                # (the reference refuses warm_start for every backend but one, torch/cvxpylayer.py:416-420; this one takes it)
                primal, dual, _, _ = _CvxpyLayerFused.apply(p_stack, self.ctx, solver_args or {}, needs_grad, True if warm_start else None)
                if on_dev and hasattr(self.ctx, "var_recover"):
                    return layer_io.recover_results(primal, dual, self.ctx, batch)
                return tl._recover_results(primal, dual, self.ctx, batch)

            tl.CvxpyLayer.forward = _forward
    _REGISTERED = True
