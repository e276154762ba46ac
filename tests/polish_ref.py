"""NumPy restatement of solution polishing (csrc/polish.cu, include/bcone.h bcone_polish) -- TEST INFRASTRUCTURE.

Same active-set rule (zero rows + nonneg rows with y_i > s_i), the same regularisation d = DELTA x the largest absolute entry
of P and A_L, the same REFINE steps of iterative refinement against the unregularised KKT matrix, the same completion and the
same acceptance test.  The regularised system is solved directly (the kernel goes through the Schur complement), so the two
agree to rounding.
"""
from __future__ import annotations

import numpy as np

DELTA, REFINE = 1e-6, 3


def metrics(A, P, b, c, x, y, s):
    """rp = |Ax + s - b|_inf, rd = |Px + A'y + c|_inf, gap = |x'Px + c'x + b'y|"""
    Px = P @ x if P is not None else np.zeros_like(x)
    return np.array([np.abs(A @ x + s - b).max(initial=0.0), np.abs(Px + A.T @ y + c).max(initial=0.0), abs(x @ Px + c @ x + b @ y)])


def polish_one(A, P, b, c, x, y, s, z, status=1):
    """One instance: dense A (m x n), symmetric P (n x n) or None, z zero rows then nonneg rows.
    -> (flag, x, y, s, resid): flag 1 accepted, 0 rejected / -1 not attempted (the input returned unchanged, resid None)."""
    m, n = A.shape
    if status not in (1, 2) or not (np.isfinite(x).all() and np.isfinite(y).all() and np.isfinite(s).all()):
        return -1, x, y, s, None
    live = np.flatnonzero((np.arange(m) < z) | (y > s))
    nl = live.size
    if nl > n:
        return -1, x, y, s, None
    AL = A[live]
    Pm = P if P is not None else np.zeros((n, n))
    scale = max(np.abs(Pm).max(initial=0.0), np.abs(AL).max(initial=0.0))
    d = DELTA * (scale if scale > 0 else 1.0)
    K = np.block([[Pm, AL.T], [AL, np.zeros((nl, nl))]])
    Kd = K + np.diag(np.r_[np.full(n, d), np.full(nl, -d)])
    rhs = np.r_[-c, b[live]]
    try:
        np.linalg.cholesky(Pm + d * np.eye(n))
        w = np.linalg.solve(Kd, rhs)
        for _ in range(REFINE):
            w = w + np.linalg.solve(Kd, rhs - K @ w)
    except np.linalg.LinAlgError:
        return 0, x, y, s, None
    xp = w[:n]
    yp = np.zeros(m)
    yp[live] = w[n:]
    yp[z:] = np.maximum(yp[z:], 0.0)
    sp_ = b - A @ xp
    sp_[:z] = 0.0
    sp_[z:] = np.maximum(sp_[z:], 0.0)
    sp_[live] = 0.0
    r0, r1 = metrics(A, P, b, c, x, y, s), metrics(A, P, b, c, xp, yp, sp_)
    if np.all(r1 <= r0):
        return 1, xp, yp, sp_, r1
    return 0, x, y, s, None


def polish_batch(bt, x, y, s, status=None):
    """Every instance of a problems.Batch (zero + nonneg cones) -> flags[B], x, y, s (copies)"""
    z = bt.structure.cones.z
    flags = np.zeros(bt.B, dtype=np.int32)
    X, Y, S = x.copy(), y.copy(), s.copy()
    for i in range(bt.B):
        P = bt.P_dense(i) if bt.P_vals is not None else None
        st = 1 if status is None else int(status[i])
        flags[i], X[i], Y[i], S[i], _ = polish_one(bt.A_dense(i), P, bt.b[i], bt.c[i], x[i], y[i], s[i], z, st)
    return flags, X, Y, S
