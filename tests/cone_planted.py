"""Planted mixed-cone batches -- TEST INFRASTRUCTURE.

Per cone block a strictly complementary pair (s, y) is drawn (the states are listed in ``planted``), P is positive definite
(x unique) and A is a generic CSR pattern whose dual faces have total dimension <= n - 2 (y unique); then b = A x + s and
c = -A'y - P x.  The solution map is differentiable at every instance, so solves, adjoints and forward-mode derivatives
have one well-defined answer.  Exponential blocks are placed in each case of the device projection ``proj_exp``
(0 inside, 1 polar, 2 r < 0 and s < 0, 3 iterative) with ``s`` and ``y`` from the reference projection ``cone_ref``.
"""
from __future__ import annotations

import numpy as np

from cvxpylayers_b200.problems import Batch, mat_to_svec
from cvxpylayers_b200.structure import ConeSpec, Structure
from tests import cone_ref as cr

# dimension of the face of the dual cone that holds y, per exponential case: ep rows have y = -(w - Pi_K(w)), ed rows y = Pi_K(w)
_EXP_FACE = {"ep": (0, 3, 1, 1), "ed": (3, 0, 2, 1)}


def exp_point(case: int, rng: np.random.Generator) -> np.ndarray:
    """A point w whose projection onto K_exp takes ``case``; the iterative case spreads rho = x / y over -15..20,
    including the region r > 0 small, s < 0, t > 0 of large rho."""
    a, b = rng.uniform(0.5, 2.0, 2)
    if case == 0:
        rho = rng.uniform(-3, 3)
        return a * np.array([rho, 1.0, np.exp(rho) * (1 + b)])
    if case == 1:
        u, v = -a, rng.uniform(-2, 2)
        return -np.array([u, v, -u * np.exp(v / u) / np.e * (1 + b)])
    if case == 2:
        return np.array([-a, -b, rng.uniform(0.5, 2.0)])
    rho = rng.uniform(-15, 20)
    E = np.exp(rho)
    y, mu = a / max(1.0, E) / (max(1.0, abs(rho)) if rng.random() < 0.5 else 1.0), b / max(1.0, E)
    return y * np.array([rho, 1.0, E]) + mu * np.array([E, (1 - rho) * E, -1.0])


def _block(kind, size, rng, state):
    """-> s, y, dual face dimension of one block."""
    if kind == "z":
        return np.zeros(1), rng.standard_normal(1), 1
    if kind == "l":
        a = rng.uniform(0.5, 2.0, 1)
        return (np.zeros(1), a, 1) if state % 2 else (a, np.zeros(1), 0)
    if kind == "q":
        u = rng.standard_normal(size - 1)
        nu = np.linalg.norm(u)
        a, b = rng.uniform(0.5, 2.0, 2)
        st = state % (3 if size <= 8 else 2)   # y interior costs a face of dimension q: only on small cones
        if size == 1:
            return (np.array([a]), np.zeros(1), 0) if st != 2 else (np.zeros(1), np.array([a]), 1)
        if st == 0:
            return np.concatenate([[nu + a], u]), np.zeros(size), 0
        if st == 1:
            return a * np.concatenate([[nu], u]), b * np.concatenate([[nu], -u]), 1
        return np.zeros(size), np.concatenate([[nu + a], u]), size
    if kind == "s":
        k = size
        Q = np.linalg.qr(rng.standard_normal((k, k)))[0]
        ry = min(k, state % 3)
        lam = rng.uniform(0.5, 2.0, k)
        if k - ry >= 2:
            lam[1] = lam[0]   # repeated eigenvalues in s ...
        if ry >= 2:
            lam[-1] = lam[-2]   # ... and in y
        ls, ly = np.where(np.arange(k) < k - ry, lam, 0.0), np.where(np.arange(k) >= k - ry, lam, 0.0)
        return mat_to_svec((Q * ls) @ Q.T), mat_to_svec((Q * ly) @ Q.T), ry * (ry + 1) // 2
    case = state % 4
    w = exp_point(case, rng)
    p = cr.proj_exp(w)
    if kind == "ep":   # s in K_exp, y in K_exp*: w = s - y
        return p, p - w, _EXP_FACE["ep"][case]
    return p - w, p, _EXP_FACE["ed"][case]   # ed: y in K_exp, s in K_exp*: w = y - s


def _blocks(cones: ConeSpec):
    out = [("z", 1)] * cones.z + [("l", 1)] * cones.l + [("q", q) for q in cones.q] + [("s", k) for k in cones.s]
    return out + [("ep", 3)] * cones.ep + [("ed", 3)] * cones.ed


def planted(cones: ConeSpec, B: int, seed: int, row_nnz: int | None = None, exp_state=None, block_scale=None) -> Batch:
    """B instances (seeds seed, seed + 1, ...) of one structure.  ``row_nnz``: entries per row of A (default: dense rows);
    ``exp_state(e, i)``: the case of exponential cone e in instance i (default: all four cases in turn); ``block_scale`` =
    (lo, hi): every block's (s, y) multiplied by its own log-uniform factor in [lo, hi]."""
    blocks = _blocks(cones)
    insts = []
    for i in range(B):
        rng = np.random.default_rng(seed + i)
        ss, ys, face, ne = [], [], 0, 0
        for j, (kind, size) in enumerate(blocks):
            state = j + i
            if kind in ("ep", "ed"):
                state = exp_state(ne, i) if exp_state else ne + i
                ne += 1
            s, y, f = _block(kind, size, rng, state)
            if block_scale:
                sc = np.exp(rng.uniform(np.log(block_scale[0]), np.log(block_scale[1])))
                s, y = s * sc, y * sc
            ss.append(s); ys.append(y); face += f
        insts.append((np.concatenate(ss), np.concatenate(ys), face))
    m = cones.m
    n = max(f for _, _, f in insts) + 4
    prng = np.random.default_rng(seed + 10_000)
    k = n if row_nnz is None else min(n, row_nnz)
    cols = [np.sort(prng.choice(n, k, replace=False)) for _ in range(m)]
    indptr = np.concatenate([[0], np.cumsum([len(c) for c in cols])])
    indices = np.concatenate(cols)
    pptr = np.concatenate([[0], np.cumsum(np.arange(n, 0, -1))])
    pidx = np.concatenate([np.arange(r, n) for r in range(n)])
    st = Structure(n, m, indptr, indices, cones, pptr, pidx)
    A_vals, P_vals, b, c, X, Y, S = [], [], [], [], [], [], []
    rows = np.repeat(np.arange(m), np.diff(indptr))
    iu = np.triu_indices(n)
    for i, (s, y, _) in enumerate(insts):
        rng = np.random.default_rng(seed + 20_000 + i)
        av = rng.standard_normal(indices.size) / np.sqrt(k)
        A = np.zeros((m, n)); A[rows, indices] = av
        G = rng.standard_normal((n, n)) / np.sqrt(n)
        P = G @ G.T + 0.5 * np.eye(n)
        x = rng.standard_normal(n)
        A_vals.append(av); P_vals.append(P[iu]); X.append(x); Y.append(y); S.append(s)
        b.append(A @ x + s); c.append(-A.T @ y - P @ x)
    arr = lambda a: np.ascontiguousarray(np.stack(a))  # noqa: E731
    return Batch(st, arr(A_vals), arr(b), arr(c), arr(P_vals), arr(X), arr(Y), arr(S), "planted",
                 aux={"faces": [f for _, _, f in insts]})


def structures() -> dict:
    """The structures the cone tests run (name -> (ConeSpec, planted keyword arguments))."""
    return {
        "soc_sizes": (ConeSpec(z=3, l=6, q=[1, 2, 3, 31, 32, 33, 64, 65]), {}),
        "psd_warm": (ConeSpec(z=2, l=2, s=[1, 2, 3, 7, 8, 9, 15, 16]), {"row_nnz": 12}),
        "psd_serial": (ConeSpec(z=2, s=[17, 20]), {"row_nnz": 12}),
        "exp": (ConeSpec(l=4, ep=10, ed=10), {}),
        # more SOC + PSD blocks than warps and more exponential cones than threads; most exponential cones sit in a case
        # whose y is 0 (ep inside, ed polar) so that the dual faces stay smaller than n
        "many_blocks": (ConeSpec(z=2, q=[3] * 24, s=[2] * 12, ep=300, ed=300),
                        {"row_nnz": 6, "exp_state": lambda e, i: (e + i) % 4 if e % 50 == 0 else (0 if e < 300 else 1)}),
        "mixed": (ConeSpec(z=2, l=4, q=[1, 4, 33], s=[3, 17], ep=4, ed=4), {"row_nnz": 16}),
    }


# the mixed structure with blocks of magnitudes 1e-6 ... 1e3 within each instance (the scale-covariance test)
MIXED_SCALES = (ConeSpec(z=2, l=4, q=[1, 4, 33], s=[3, 17], ep=4, ed=4), {"row_nnz": 16, "block_scale": (1e-6, 1e3)})


def make(name: str, B: int = 4) -> Batch:
    """The batch the cone tests run for ``name`` (a key of ``structures()`` or "mixed_scales"); one seed per name."""
    names = list(structures()) + ["mixed_scales"]
    cones, kw = MIXED_SCALES if name == "mixed_scales" else structures()[name]
    return planted(cones, B, 100 * (1 + names.index(name)), **kw)
