"""Layer prologue / epilogue on the device (SURVEY.md 8f.3).

Twins of the reference's ``_flatten_and_batch_params`` (``src/cvxpylayers/torch/cvxpylayer.py:84-141``) and
``_recover_results`` (``:225-282``), same arguments, same results -- but each parameter / variable is ONE kernel launch
driven by a pre-computed index map (``include/bcone.h``: ``bcone_rows_from_param``, ``bcone_gather_cols`` and their
adjoints) instead of a chain of expand / permute / reshape / cat / transpose (resp. slice / scatter / reshape) tensor ops,
so the whole ``forward()`` of a layer is a fixed sequence of launches with no intermediate tensors.  CUDA float64 tensors only;
anything else should go through the reference's own functions.
"""
from __future__ import annotations

import ctypes as C
from typing import Any

import numpy as np
import torch

from . import _lib

OP_NONE, OP_EXP, OP_LOG = 0, 1, 2


def _stream(dev) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _p(t) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _chk(rc: int, what: str):
    if rc != 0:
        raise RuntimeError(f"{what} failed ({rc}): {_lib.load().bcone_last_error(None).decode()}")


_MAP_CACHE: dict = {}


def _dev_i32(key, build, dev):
    k = (key, dev)
    t = _MAP_CACHE.get(k)
    if t is None:
        t = torch.as_tensor(np.ascontiguousarray(build(), dtype=np.int32), device=dev)
        _MAP_CACHE[k] = t
    return t


def _dev_f64(key, build, dev):
    k = (key, dev)
    t = _MAP_CACHE.get(k)
    if t is None:
        t = torch.as_tensor(np.ascontiguousarray(build(), dtype=np.float64), device=dev)
        _MAP_CACHE[k] = t
    return t


def fortran_map(shape: tuple[int, ...]) -> np.ndarray:
    """map[k] = offset (C order) of the element that has Fortran-order linear index k -- what ``_reshape_fortran(x, (-1,))``
    computes with permutes (``torch/cvxpylayer.py:40-56``)."""
    if len(shape) <= 1:
        return np.arange(int(np.prod(shape, dtype=np.int64)) if shape else 1, dtype=np.int32)
    return np.arange(int(np.prod(shape)), dtype=np.int64).reshape(shape).reshape(-1, order="F").astype(np.int32)


class _FlattenParams(torch.autograd.Function):
    """(params...) -> p_stack[P1, B]; ``spec`` = per parameter (row0, size, batched, shape, op)."""

    @staticmethod
    def forward(ctx: Any, spec, B: int, *params):
        lib = _lib.load()
        dev = params[0].device
        P1 = sum(s[1] for s in spec) + 1
        p_stack = torch.empty((P1, B), dtype=torch.float64, device=dev)
        p_stack[P1 - 1].fill_(1.0)   # the constant column of the canonical form
        keep = []
        for (row0, size, batched, shape, op), p in zip(spec, params):
            pc = p.detach().contiguous()
            keep.append(pc)
            fmap = _dev_i32(("F", shape), lambda shape=shape: fortran_map(shape), dev)
            _chk(lib.bcone_rows_from_param(_p(pc), C.c_int64(size if batched else 0), _p(fmap), C.c_int32(size), C.c_int32(B), C.c_int32(op),
                                           C.c_void_p(p_stack.data_ptr() + row0 * B * 8), _stream(dev)), "bcone_rows_from_param")
        ctx.spec, ctx.B, ctx.keep = spec, B, keep
        return p_stack

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx: Any, g):
        lib = _lib.load()
        g = g.contiguous()
        dev = g.device
        outs = []
        for (row0, size, batched, shape, op), pc in zip(ctx.spec, ctx.keep):
            gp = torch.zeros_like(pc)
            fmap = _dev_i32(("F", shape), lambda shape=shape: fortran_map(shape), dev)
            _chk(lib.bcone_param_from_rows(C.c_void_p(g.data_ptr() + row0 * ctx.B * 8), _p(pc), C.c_int64(size if batched else 0), _p(fmap),
                                           C.c_int32(size), C.c_int32(ctx.B), C.c_int32(op), _p(gp), _stream(dev)), "bcone_param_from_rows")
            outs.append(gp)
        return (None, None, *outs)

    @staticmethod
    def jvp(ctx: Any, _spec, _B, *tangents):
        """Forward mode: the same index maps on the tangents (d log p = dp / p for GP-log parameters); the constant row's
        tangent is 0, as is the rows' of a parameter without one."""
        lib = _lib.load()
        dev = ctx.keep[0].device
        P1 = sum(s[1] for s in ctx.spec) + 1
        tp = torch.zeros((P1, ctx.B), dtype=torch.float64, device=dev)
        for (row0, size, batched, shape, op), pc, t in zip(ctx.spec, ctx.keep, tangents):
            if t is None:
                continue
            tc = t.detach().to(dtype=torch.float64)
            tc = (tc / pc if op == OP_LOG else tc).contiguous()
            fmap = _dev_i32(("F", shape), lambda shape=shape: fortran_map(shape), dev)
            _chk(lib.bcone_rows_from_param(_p(tc), C.c_int64(size if batched else 0), _p(fmap), C.c_int32(size), C.c_int32(ctx.B), C.c_int32(OP_NONE),
                                           C.c_void_p(tp.data_ptr() + row0 * ctx.B * 8), _stream(dev)), "bcone_rows_from_param")
        return tp


def flatten_and_batch_params(params: tuple[torch.Tensor, ...], ctx, batch: tuple) -> torch.Tensor:
    """Device twin of ``_flatten_and_batch_params(params, ctx, batch)`` (+ the GP log of ``_apply_gp_log_transform``,
    ``torch/cvxpylayer.py:58-81``, folded into the same launch).  ``ctx`` needs ``batch_sizes``, ``user_order_to_col_order`` and
    optionally ``gp`` / ``gp_log_mask`` like the reference's ``LayersContext``."""
    B = batch[0] if batch else 1
    order = ctx.user_order_to_col_order
    sizes = []
    for i, p in enumerate(params):
        shape = tuple(p.shape[1:]) if ctx.batch_sizes[i] else tuple(p.shape)
        sizes.append(int(np.prod(shape, dtype=np.int64)) if shape else 1)
    by_col = sorted(range(len(params)), key=lambda i: order[i])
    row0, acc = {}, 0
    for i in by_col:
        row0[i] = acc
        acc += sizes[i]
    log_mask = getattr(ctx, "gp_log_mask", None) if getattr(ctx, "gp", False) else None
    spec = tuple((row0[i], sizes[i], bool(ctx.batch_sizes[i]), tuple(p.shape[1:]) if ctx.batch_sizes[i] else tuple(p.shape),
                  OP_LOG if (log_mask is not None and log_mask[i]) else OP_NONE) for i, p in enumerate(params))
    p_stack = _FlattenParams.apply(spec, B, *params)
    return p_stack if batch else p_stack.reshape(p_stack.shape[0])


class _GatherCols(torch.autograd.Function):
    @staticmethod
    def forward(ctx: Any, src, imap, scale, op: int):
        lib = _lib.load()
        s = src.detach().contiguous()
        B, ld = s.shape
        K = imap.numel()
        out = torch.empty((B, K), dtype=torch.float64, device=s.device)
        _chk(lib.bcone_gather_cols(_p(s), C.c_int64(ld), _p(imap), _p(scale), C.c_int32(K), C.c_int32(B), C.c_int32(op), _p(out), _stream(s.device)),
             "bcone_gather_cols")
        ctx.meta = (imap, scale, op, ld, out if op == OP_EXP else None)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx: Any, g):
        lib = _lib.load()
        imap, scale, op, ld, out = ctx.meta
        g = g.contiguous()
        B, K = g.shape
        gin = torch.zeros((B, ld), dtype=torch.float64, device=g.device)
        _chk(lib.bcone_scatter_cols(_p(g), _p(out), C.c_int64(ld), _p(imap), _p(scale), C.c_int32(K), C.c_int32(B), C.c_int32(op), _p(gin),
                                    _stream(g.device)), "bcone_scatter_cols")
        return gin, None, None, None

    @staticmethod
    def jvp(ctx: Any, tsrc, *_):
        """Forward mode: the same gather on the tangent (times ``out`` for GP-exp variables: d exp(u) = exp(u) du)."""
        lib = _lib.load()
        imap, scale, op, ld, out = ctx.meta
        K = imap.numel()
        if tsrc is None:
            return None
        ts = tsrc.detach().contiguous()
        B = ts.shape[0]
        tout = torch.empty((B, K), dtype=torch.float64, device=ts.device)
        _chk(lib.bcone_gather_cols(_p(ts), C.c_int64(ld), _p(imap), _p(scale), C.c_int32(K), C.c_int32(B), C.c_int32(OP_NONE), _p(tout),
                                   _stream(ts.device)), "bcone_gather_cols")
        return tout * out if op == OP_EXP else tout


def _var_map(var) -> tuple[np.ndarray, np.ndarray | None]:
    """(index map, scale) of one requested variable: out_flat[k] (C order over ``var.shape``) = scale[k] * data[start + map[k]]
    -- the composition of the slice, the svec unpacking (``torch/cvxpylayer.py:143-222``) and the Fortran reshape (``:270``)."""
    sl = var.primal if var.source == "primal" else var.dual
    start = sl.start or 0
    shape = tuple(var.shape)
    if var.unpack_fn == "reshape":
        size = int(np.prod(shape, dtype=np.int64)) if shape else 1
        if len(shape) <= 1:
            return start + np.arange(size), None
        # out[i0, i1, ...] = data[Fortran index of (i0, i1, ...)]
        f_of_c = np.arange(size).reshape(shape, order="F").reshape(-1)
        return start + f_of_c, None
    n = shape[0]
    idx = np.zeros((n, n), dtype=np.int64)
    sc = np.ones((n, n))
    if var.unpack_fn == "svec_primal":       # upper triangle, row-major, unscaled
        rows, cols = np.triu_indices(n)
        idx[rows, cols] = np.arange(rows.size)
        idx[cols, rows] = np.arange(rows.size)
        return start + idx.reshape(-1), None
    if var.unpack_fn == "svec_dual":         # lower triangle, column-major, off-diagonals * 1/sqrt2
        rows_rm, cols_rm = np.tril_indices(n)
        order = np.lexsort((rows_rm, cols_rm))
        rows, cols = rows_rm[order], cols_rm[order]
        idx[rows, cols] = np.arange(rows.size)
        idx[cols, rows] = np.arange(rows.size)
        sc[rows, cols] = np.where(rows == cols, 1.0, 1.0 / np.sqrt(2.0))
        sc[cols, rows] = sc[rows, cols]
        return start + idx.reshape(-1), sc.reshape(-1)
    raise ValueError(f"Unknown variable recovery type: {var.unpack_fn}")


def recover_results(primal: torch.Tensor, dual: torch.Tensor, ctx, batch: tuple) -> tuple[torch.Tensor, ...]:
    """Device twin of ``_recover_results(primal, dual, ctx, batch)``: one gather launch per requested variable (slice, symmetric
    unpacking with its scaling, Fortran reshape and the GP ``exp`` fused)."""
    dev = primal.device
    results = []
    for vi, var in enumerate(ctx.var_recover):
        src = primal if var.source == "primal" else dual
        key = ("V", id(ctx), vi)
        imap = _dev_i32(key, lambda var=var: _var_map(var)[0], dev)
        sc_np = _var_map(var)[1]
        scale = _dev_f64(key + ("s",), lambda sc_np=sc_np: sc_np, dev) if sc_np is not None else None
        op = OP_EXP if (getattr(ctx, "gp", False) and var.source == "primal") else OP_NONE
        out = _GatherCols.apply(src, imap, scale, op)
        results.append(out.reshape(tuple(batch) + tuple(var.shape)))
    return tuple(results)
