"""NumPy restatement of solution refinement (csrc/refine.cu, include/bcone.h bcone_refine) -- TEST INFRASTRUCTURE.

At w = (x, v), v = y - s, pi = Pi_{K*}(v) (the C oracle's projection and Jacobian, the device's algorithms):

    R(x, v) = [P x + A' pi + c ;  b - A x - (pi - v) ;  -(x'P x + c'x + b'pi)]

and its Jacobian in (x, v) is the first n + m columns of the forward mode's M (``jvp_ref.dense_M``).  A step is the kernel's:
LSQR (SciPy's, the same Paige-Saunders iteration and stopping rules) on diag(Rsc) M diag(Lsc) with the tau column masked
(Lsc_tau = 0); with ``precond`` = 1 the scalings are the kernel's Ruiz equilibration of the 0/1 skeleton of M' (bwd.cu
``equilibrate``) and an inactive nonneg row's unknown is recovered from its own equation.  Then the line search alpha = 1, 1/2,
..., 1/32 on ||R||_2, at most ``steps`` steps, and polishing's acceptance rule (``polish_ref.metrics``).
"""
from __future__ import annotations

import numpy as np
from scipy.sparse.linalg import lsqr

from oracle import oracle as orc
from tests.jvp_ref import dense_M
from tests.polish_ref import metrics


def residual(st, A, P, b, c, x, v):
    """-> R (n + m + 1), pi"""
    pi = orc.proj_dual_cone(st, v)
    Px = P @ x if P is not None else np.zeros_like(x)
    return np.concatenate([Px + A.T @ pi + c, b - A @ x - (pi - v), [-(x @ Px + c @ x + b @ pi)]]), pi


def scalings(st, A, P, b, c, x, piy, passes=10):
    """The kernel's equilibration (bwd.cu ``equilibrate``) -> Lsc, Rsc: row / column scalings of M', so M is scaled
    diag(Rsc) M diag(Lsc)."""
    m, n = A.shape
    N = n + m + 1
    lo, hi = st.cones.z, st.cones.z + st.cones.l
    Pm = np.zeros((n, n)) if P is None else P
    px2c = 2 * Pm @ x + c
    G2 = np.zeros((N, N))
    G2[:n, :n] = Pm ** 2
    G2[:n, n:n + m] = (A ** 2).T
    G2[n:n + m, :n] = A ** 2
    G2[:n, -1] = px2c ** 2
    G2[-1, :n] = c ** 2
    G2[n:n + m, -1] = b ** 2
    G2[-1, n:n + m] = b ** 2
    G2[-1, -1] = (x @ Pm @ x) ** 2
    idx = np.arange(hi, m)
    G2[n + idx, n + idx] = 1.0
    L, R = np.ones(N), np.ones(N)
    inactive = n + lo + np.flatnonzero(~(piy[lo:hi] > 0))
    L[inactive] = R[inactive] = 0.0
    for _ in range(passes):
        rs = L ** 2 * (G2 @ R ** 2)
        cs = R ** 2 * (G2.T @ L ** 2)
        L = np.where((L > 0) & (rs > 1e-300), L / np.sqrt(np.sqrt(np.where(rs > 0, rs, 1.0))), L)
        R = np.where((R > 0) & (cs > 1e-300), R / np.sqrt(np.sqrt(np.where(cs > 0, cs, 1.0))), R)
    return L, R


def newton_dir(st, A, P, b, c, x, v, R, precond=0, atol=1e-8, btol=1e-8, conlim=1e8, iter_lim=-1, passes=10):
    """z = argmin ||M[:, :n+m] z + R|| as the kernel solves it (z_tau = 0)."""
    m, n = A.shape
    N = n + m + 1
    M, _, piy = dense_M(st, A, P, b, c, x, v, np.zeros(m))
    if precond:
        Lsc, Rsc = scalings(st, A, P, b, c, x, piy, passes)
    else:
        Lsc, Rsc = np.ones(N), np.ones(N)
    Lsc[-1] = 0.0
    B = Rsc[:, None] * M * Lsc[None, :]
    u = Rsc * -R
    zs = lsqr(B, u, atol=atol, btol=btol, conlim=conlim, iter_lim=2 * N if iter_lim < 0 else iter_lim)[0] if np.any(u) else np.zeros(N)
    z = Lsc * zs
    if precond:
        lo, hi = st.cones.z, st.cones.z + st.cones.l
        inactive = lo + np.flatnonzero(~(piy[lo:hi] > 0))
        z[n + inactive] = (A @ z[:n])[inactive] - R[n + inactive]
    return z


def refine_one(st, A, P, b, c, x, y, s, status=1, steps=3, precond=0, **lsqr_kw):
    """One instance (dense A, full symmetric P or None) -> (flag, x, y, s, resid): flag 1 accepted, 0 rejected / -1 not
    attempted (the input returned unchanged, resid None)."""
    m, n = A.shape
    if status not in (1, 2) or not (np.isfinite(x).all() and np.isfinite(y).all() and np.isfinite(s).all()):
        return -1, x, y, s, None
    r0 = metrics(A, P, b, c, x, y, s)
    xw, vw = x.copy(), y - s
    z = np.zeros(n + m + 1)
    alpha, k, rn_w, yw = 0.0, 0, None, None
    while True:
        xt, vt = xw + alpha * z[:n], vw + alpha * z[n:n + m]
        R, pi = residual(st, A, P, b, c, xt, vt)
        rn = R @ R
        if rn_w is None or rn < rn_w:
            xw, vw, yw, Rw, rn_w = xt, vt, pi, R, rn
            if k == steps or not rn > 0:
                break
            k += 1
        else:
            alpha *= 0.5
            if alpha < 1.0 / 32:
                break
            continue
        z = newton_dir(st, A, P, b, c, xw, vw, Rw, precond, **lsqr_kw)
        alpha = 1.0
    sw = yw - vw
    r1 = metrics(A, P, b, c, xw, yw, sw)
    if np.all(r1 <= r0):
        return 1, xw, yw, sw, r1
    return 0, x, y, s, None


def refine_batch(bt, x, y, s, status=None, steps=3, precond=0, **lsqr_kw):
    """Every instance of a problems.Batch -> flags[B], x, y, s (copies)"""
    flags = np.zeros(bt.B, dtype=np.int32)
    X, Y, S = x.copy(), y.copy(), s.copy()
    for i in range(bt.B):
        P = bt.P_dense(i) if bt.P_vals is not None else None
        st = 1 if status is None else int(status[i])
        flags[i], X[i], Y[i], S[i], _ = refine_one(bt.structure, bt.A_dense(i), P, bt.b[i], bt.c[i], x[i], y[i], s[i], st, steps, precond,
                                                   **lsqr_kw)
    return flags, X, Y, S
