"""Batches with a planted outcome per instance: primal infeasible, unbounded or solved -- TEST INFRASTRUCTURE.

Every instance starts from an instance of a planted batch (``tests/cone_planted.py`` for the generic structures,
``tests/tiled_shapes.py`` for the dense zero + nonneg shapes) and keeps its structure's sparsity pattern; only values change.

* ``infeasible``: a certificate y in the interior of K* (no zero entry; an SOC block (|u| + a, u), a PSD block the svec of a
  positive-definite matrix, an exponential block an interior point of K_exp* on ``ep`` rows and of K_exp on ``ed`` rows).  A
  is changed within its pattern so that A'y = 0 (the least change per column: a multiple of y on the column's structural
  rows), then b <- b - y (y'b + 1) / |y|^2, so that b'y = -1.
* ``unbounded``: a ray x_d with no zero entry, A x_d = -s_d with s_d in the interior of K (0 on zero-cone rows; A changed
  within its pattern, the least change per row), P replaced by (I - x^ x^') P (I - x^ x^') so that P x_d = 0, c'x_d = -1;
  b = A x_f + s_f with s_f in the interior of K keeps the instance primal feasible.
* ``unbounded_zero_col``: the degenerate ray x_d = e_j of a variable that appears in no row of A and not in P (a zero
  column through Ruiz equilibration), c_j = -1, s_d = 0.
* ``control``: the planted instance unchanged, SOLVED at its planted point.
* ``control_near``: an ``infeasible`` instance's A with a planted optimum (x*, y*, t s*) whose slack along the certificate
  is small: s'y_cert = NEAR |b| |y_cert|.

Scales: the whole instance's (A, b) times ``scale``; ``block_scale = (lo, hi)``: each cone block's rows of (A, b) times its
own log-uniform factor D in [lo, hi].  Certificates, rays and planted points are transformed with the data (y -> y / D,
s -> D s), so every status is unchanged; ``aux`` holds them normalised to b'y = -1 and c'x_d = -1 (``control_near``: its
y_cert, with b'y_cert = NEAR |b| |y_cert| > 0).

``shared``: one A and P for the batch (instance 0's, with a zero column j and A'y_cert = 0 on the others); the outcome of each
instance is chosen through b and c alone.  There the controls' x_j is free (c_j = 0, no row or P term): it stays at the
start, 0, which the planted x* holds.
"""
from __future__ import annotations

import numpy as np

from cvxpylayers_b200.problems import Batch, mat_to_svec
from cvxpylayers_b200.structure import ConeSpec
from tests import cone_planted as cp

STATUS = {"control": 1, "control_near": 1, "infeasible": -2, "unbounded": -1, "unbounded_zero_col": -1}
NEAR = 1e-3
MIX = ("control", "infeasible", "control", "unbounded", "control_near", "unbounded_zero_col", "control")
MIX_NO_SLACK = tuple(k for k in MIX if k != "control_near")   # (every row an equality: no slack to make small)
SHARED_MIX = ("control", "infeasible", "control", "unbounded_zero_col", "control", "infeasible", "unbounded_zero_col", "control")


def blocks(cones: ConeSpec) -> list:
    """(kind, first row, rows, order) of every cone block in row order (order: of an SOC or PSD block)."""
    out, r = [], 0
    for kind, k in cp._blocks(cones):
        rows = k * (k + 1) // 2 if kind == "s" else k
        out.append((kind, r, rows, k))
        r += rows
    return out


def interior(cones: ConeSpec, dual: bool, rng: np.random.Generator) -> np.ndarray:
    """A point in the interior of K* (``dual``) or of K (zero-cone rows: 0, K's only point there)."""
    out = []
    for kind, _, size, k in blocks(cones):
        a = rng.uniform(0.5, 2.0)
        if kind == "z":
            out.append([rng.choice([-1.0, 1.0]) * a] if dual else [0.0])
        elif kind == "l":
            out.append([a])
        elif kind == "q":
            u = rng.standard_normal(size - 1)
            out.append(np.concatenate([[np.linalg.norm(u) + a], u]))
        elif kind == "s":
            G = rng.standard_normal((k, k))
            out.append(mat_to_svec(G @ G.T / k + a * np.eye(k)))
        else:   # ep rows: s in K_exp, y in K_exp*; ed rows: s in K_exp*, y in K_exp
            in_exp = (kind == "ep") != dual
            out.append(a * (np.array([0.2, 1.0, 2.0]) if in_exp else np.array([-1.0, 0.3, 1.5])))
    return np.concatenate([np.asarray(o, dtype=float) for o in out])


def _mask(st) -> np.ndarray:
    M = np.zeros((st.m, st.n), dtype=bool)
    M[np.repeat(np.arange(st.m), np.diff(st.A_indptr)), st.A_indices] = True
    return M


def _cols_orthogonal(A, M, y):
    """A'y = 0 by the least change of each column within the pattern (a multiple of y on its structural rows)."""
    for _ in range(2):   # (the second pass removes the first one's rounding)
        r = A.T @ y
        d = (M * y[:, None] ** 2).sum(0)
        A = A - M * np.outer(y, np.divide(r, d, out=np.zeros_like(r), where=d > 0))
    return A


def _rows_to(A, M, x, target):
    """A x = target by the least change of each row within the pattern."""
    for _ in range(2):
        r = A @ x - target
        d = (M * x[None, :] ** 2).sum(1)
        assert (d > 0).all(), "every row needs a structural entry"
        A = A - M * np.outer(r / d, x)
    return A


def _no_zero(n, rng):
    return rng.choice([-1.0, 1.0], n) * rng.uniform(0.5, 2.0, n)


def _near_control(A, P, x, y, s, yc):
    """(b, c, s) of the planted optimum (x, y, t s) with t s'yc = NEAR |b| |yc|."""
    a = s @ yc
    assert a > 0, "the planted slack is 0"
    t = 1.0
    for _ in range(20):
        t = NEAR * np.linalg.norm(A @ x + t * s) * np.linalg.norm(yc) / a
    return A @ x + t * s, -A.T @ y - P @ x, t * s


def _zero_col(A, P, j):
    A = A.copy(); A[:, j] = 0.0
    P = P.copy(); P[j, :] = 0.0; P[:, j] = 0.0
    return A, P


def _pack(st, A, P):
    iu = np.triu_indices(st.n)
    Pv = None
    if st.P_indptr is not None:
        rows = np.repeat(np.arange(st.n), np.diff(st.P_indptr))
        assert np.array_equal(np.stack([rows, st.P_indices]), np.stack(iu)), "P needs the full upper-triangular pattern"
        Pv = P[iu]
    return A[_mask(st)], Pv   # (boolean indexing runs row-major: CSR order for sorted indices)


def mixed(base: Batch, kinds=MIX, seed: int = 0, scale: float = 1.0, block_scale=None) -> Batch:
    """Instance i of the result is instance i of ``base`` turned into ``kinds[i]`` (see the module docstring)."""
    st = base.structure
    n, m, M = st.n, st.m, _mask(st)
    assert len(kinds) <= base.B
    rng, srng = np.random.default_rng(seed), np.random.default_rng(seed + 1)   # (the scales do not move the other draws)
    D = np.ones(m)
    if block_scale:
        for _, r, size, _ in blocks(st.cones):
            D[r:r + size] = np.exp(srng.uniform(np.log(block_scale[0]), np.log(block_scale[1])))
    D = D * scale
    out = {k: [] for k in ("A", "P", "b", "c", "x", "y", "s", "yc", "xd", "sd")}
    nan_n, nan_m = np.full(n, np.nan), np.full(m, np.nan)
    for i, kind in enumerate(kinds):
        A, P, b, c = base.A_dense(i), base.P_dense(i), base.b[i].copy(), base.c[i].copy()
        x, y, s = base.x_star[i], base.y_star[i], base.s_star[i]
        yc, xd, sd = nan_m, nan_n, nan_m
        if kind in ("infeasible", "control_near"):
            yc = interior(st.cones, True, rng)
            A = _cols_orthogonal(A, M, yc)
            if kind == "infeasible":
                b = b - yc * (yc @ b + 1.0) / (yc @ yc)
                x, y, s = nan_n, nan_m, nan_m
            else:
                b, c, s = _near_control(A, P, x, y, s, yc)
        elif kind == "unbounded":
            xd, sd = _no_zero(n, rng), interior(st.cones, False, rng)
            A = _rows_to(A, M, xd, -sd)
            Pi = np.eye(n) - np.outer(xd, xd) / (xd @ xd)
            P = Pi @ P @ Pi
            P = 0.5 * (P + P.T)
            c = c - xd * (xd @ c + 1.0) / (xd @ xd)
            b = A @ rng.standard_normal(n) + interior(st.cones, False, rng)
            x, y, s = nan_n, nan_m, nan_m
        elif kind == "unbounded_zero_col":
            j = int(rng.integers(n))
            A, P = _zero_col(A, P, j)
            xd, sd = np.eye(n)[j], np.zeros(m)
            c[j] = -1.0
            b = A @ rng.standard_normal(n) + interior(st.cones, False, rng)
            x, y, s = nan_n, nan_m, nan_m
        else:
            assert kind == "control", kind
        # the scales: A, b -> D A, D b; y -> y / D, s -> D s
        for k, v in (("A", D[:, None] * A), ("P", P), ("b", D * b), ("c", c), ("x", x), ("y", y / D), ("s", D * s),
                     ("yc", yc / D), ("xd", xd), ("sd", D * sd)):
            out[k].append(v)
    bt = _batch(st, base.name, kinds, out, shared=False)
    bt.aux["block_scale"] = block_scale
    return bt


def shared(base: Batch, kinds=SHARED_MIX, seed: int = 0) -> Batch:
    """One A and P for the whole batch: instance 0's with a zero column j and A'y_cert = 0; per instance only b and c."""
    st = base.structure
    n, m, M = st.n, st.m, _mask(st)
    rng = np.random.default_rng(seed)
    j = int(rng.integers(n))
    A, P = _zero_col(base.A_dense(0), base.P_dense(0), j)
    yc = interior(st.cones, True, rng)
    A = _cols_orthogonal(A, M, yc)
    xd = np.eye(n)[j]
    out = {k: [] for k in ("A", "P", "b", "c", "x", "y", "s", "yc", "xd", "sd")}
    nan_n, nan_m = np.full(n, np.nan), np.full(m, np.nan)
    assert len(kinds) <= base.B
    for i, kind in enumerate(kinds):
        x, y, s = base.x_star[i].copy(), base.y_star[i], base.s_star[i]
        x[j] = 0.0
        b, c = A @ x + s, -A.T @ y - P @ x
        cert = (nan_m, nan_n, nan_m)
        if kind == "infeasible":
            b = b - yc * (yc @ b + 1.0) / (yc @ yc)
            cert, (x, y, s) = (yc, nan_n, nan_m), (nan_n, nan_m, nan_m)
        elif kind == "unbounded_zero_col":
            c[j] = -1.0
            b = A @ rng.standard_normal(n) + interior(st.cones, False, rng)
            cert, (x, y, s) = (nan_m, xd, np.zeros(m)), (nan_n, nan_m, nan_m)
        else:
            assert kind == "control", kind
        for k, v in zip(("A", "P", "b", "c", "x", "y", "s", "yc", "xd", "sd"), (A, P, b, c, x, y, s, *cert)):
            out[k].append(v)
    bt = _batch(st, base.name, kinds, out, shared=True)
    bt.aux["block_scale"] = None
    return bt


def _batch(st, name, kinds, out, shared):
    packed = [_pack(st, A, P) for A, P in zip(out["A"], out["P"])]
    arr = lambda a: np.ascontiguousarray(np.stack(a))  # noqa: E731
    A_vals = arr([p[0] for p in packed])
    P_vals = arr([p[1] for p in packed]) if st.P_indptr is not None else None
    aux = {"kinds": tuple(kinds), "status": np.array([STATUS[k] for k in kinds], dtype=np.int32),
           "y_cert": arr(out["yc"]), "x_ray": arr(out["xd"]), "s_ray": arr(out["sd"]), "shared": shared}
    return Batch(st, A_vals, arr(out["b"]), arr(out["c"]), P_vals, arr(out["x"]), arr(out["y"]), arr(out["s"]),
                 f"{name}_outcomes", aux=aux)


def controls(bt: Batch) -> np.ndarray:
    return np.nonzero(bt.aux["status"] == 1)[0]
