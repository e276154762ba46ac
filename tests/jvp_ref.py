"""Dense restatement of the forward-mode derivative of the solution map (diffcp's ``D``) -- TEST INFRASTRUCTURE.

The twin of ``oracle.np_ref.vjp_dense`` in the other direction, defined as its exact transpose: with ``M`` the matrix of
``vjp_dense`` (native ``P`` included) and ``D`` the cone Jacobian taken column by column from the C oracle (so exponential
cones are covered),

    g  = [-dA' pi - dc - dP x ;  dA x - db ;  pi'db + x'dc + x'dP x]
    z  = M^-1 g                 (numpy.linalg.lstsq, or scipy.sparse.linalg.lsqr like the engine's lsqr_precond = 0)
    dx = z_x - x z_tau,   dy = D z_y - y z_tau,   ds = D z_y - z_y - s z_tau

``dP`` is the full symmetric tangent of ``P``.
"""
from __future__ import annotations

import numpy as np
from scipy.sparse.linalg import lsqr

from cvxpylayers_b200.problems import Batch
from oracle import oracle as orc


def dense_M(st, A, P, b, c, x, y, s):
    """-> M (N x N), D (m x m), pi_y"""
    m, n = A.shape
    N = n + m + 1
    v = y - s
    D = np.stack([orc.dproj_dual_cone(st, v, e) for e in np.eye(m)], axis=1)
    piy = orc.proj_dual_cone(st, v)
    Pm = np.zeros((n, n)) if P is None else P
    Px = Pm @ x
    DQ = np.zeros((N, N))
    DQ[:n, :n] = Pm
    DQ[:n, n:n + m] = A.T
    DQ[:n, -1] = c
    DQ[n:n + m, :n] = -A
    DQ[n:n + m, -1] = b
    DQ[-1, :n] = -(2 * Px + c)
    DQ[-1, n:n + m] = -b
    DQ[-1, -1] = x @ Px
    Dpi = np.eye(N)
    Dpi[n:n + m, n:n + m] = D
    return (DQ - np.eye(N)) @ Dpi + np.eye(N), D, piy


def jvp_rhs(A, x, piy, dA, dP, db, dc):
    dPx = np.zeros_like(x) if dP is None else dP @ x
    return np.concatenate([-dA.T @ piy - dc - dPx, dA @ x - db, [piy @ db + x @ dc + x @ dPx]])


def jvp_dense(st, A, P, b, c, x, y, s, dA, dP, db, dc, exact=True, atol=1e-8, btol=1e-8, conlim=1e8, iter_lim=None):
    """-> dx, dy, ds, z"""
    m, n = A.shape
    M, D, piy = dense_M(st, A, P, b, c, x, y, s)
    g = jvp_rhs(A, x, piy, dA, dP, db, dc)
    if np.abs(g).max() <= 1e-8:
        z = np.zeros(n + m + 1)
    elif exact:
        z = np.linalg.lstsq(M, g, rcond=None)[0]
    else:
        z = lsqr(M, g, atol=atol, btol=btol, conlim=conlim, iter_lim=iter_lim or 2 * (n + m + 1))[0]
    zx, zy, zt = z[:n], z[n:n + m], z[-1]
    Dzy = D @ zy
    return zx - x * zt, Dzy - y * zt, Dzy - zy - s * zt, z


def random_tangents(bt: Batch, rng: np.random.Generator) -> Batch:
    """Engine-layout tangents of every datum of ``bt`` (A and P values on their structural entries, b, c) scaled like the data."""
    sc = lambda a: np.abs(a).max(axis=1, keepdims=True)  # noqa: E731
    dP = None if bt.P_vals is None else rng.standard_normal(bt.P_vals.shape) * sc(bt.P_vals)
    return Batch(bt.structure, rng.standard_normal(bt.A_vals.shape) * sc(bt.A_vals), rng.standard_normal(bt.b.shape) * np.maximum(sc(bt.b), 1.0),
                 rng.standard_normal(bt.c.shape) * sc(bt.c), dP)


def shifted(bt: Batch, t: Batch, h: float) -> Batch:
    """bt + h t (every instance)."""
    return Batch(bt.structure, bt.A_vals + h * t.A_vals, bt.b + h * t.b, bt.c + h * t.c,
                 None if bt.P_vals is None else bt.P_vals + h * t.P_vals)
