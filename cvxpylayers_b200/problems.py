"""Synthetic workloads for the BASELINE.json configs (C1..C5, SURVEY.md section 8d).

cvxpy is not installable in this image, so the canonical tensors the reference's
layer would hand to its solver interface are fabricated directly: per instance the
solver data ``(A, b, c[, P])`` of ``min 1/2 x'Px + c'x  s.t. Ax + s = b, s in K`` in a
fixed sparsity pattern, and -- for boundary tests -- the same data re-packed as the
``(q_eval, A_eval)`` pair of ``diffcp_if.py:46-70`` (CSC values of ``[-A | b]``).

Instances with a *planted* primal-dual optimum follow SURVEY.md Appendix A.6:
draw x, z; y = Pi_{K*}(z), s = y - z, b = Ax + s, c = -A'y - Px.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp

from .structure import ConeSpec, Structure

SQRT2 = np.sqrt(2.0)


# ----------------------------------------------------------------------------- numpy cone helpers
def svec_to_mat(v: np.ndarray, k: int) -> np.ndarray:
    """svec (lower-triangle column-major, off-diagonals * sqrt2) -> symmetric matrix.
    Layout per reference ``src/cvxpylayers/torch/cvxpylayer.py:201-222``."""
    X = np.zeros(v.shape[:-1] + (k, k))
    ii, jj = np.tril_indices(k)
    order = np.lexsort((ii, jj))  # column-major walk of the lower triangle
    ii, jj = ii[order], jj[order]
    scale = np.where(ii == jj, 1.0, 1.0 / SQRT2)
    X[..., ii, jj] = v * scale
    X[..., jj, ii] = v * scale
    return X


def mat_to_svec(X: np.ndarray) -> np.ndarray:
    k = X.shape[-1]
    ii, jj = np.tril_indices(k)
    order = np.lexsort((ii, jj))
    ii, jj = ii[order], jj[order]
    scale = np.where(ii == jj, 1.0, SQRT2)
    return 0.5 * (X[..., ii, jj] + X[..., jj, ii]) * scale


def proj_dual_cone(v: np.ndarray, cones: ConeSpec) -> np.ndarray:
    """Pi_{K*}(v) along the last axis (zero cone -> free, others self-dual)."""
    out = np.array(v, dtype=np.float64, copy=True)
    off = cones.z
    out[..., off : off + cones.l] = np.maximum(out[..., off : off + cones.l], 0.0)
    off += cones.l
    for q in cones.q:
        blk = out[..., off : off + q]
        t = blk[..., 0].copy()
        nx = np.linalg.norm(blk[..., 1:], axis=-1)
        inside = nx <= t
        polar = nx <= -t
        a = 0.5 * (1.0 + t / np.where(nx > 0, nx, 1.0))
        new = np.concatenate([(a * nx)[..., None], blk[..., 1:] * a[..., None]], axis=-1)
        new = np.where(polar[..., None], 0.0, new)
        new = np.where(inside[..., None], blk, new)
        out[..., off : off + q] = new
        off += q
    for k in cones.s:
        sz = k * (k + 1) // 2
        X = svec_to_mat(out[..., off : off + sz], k)
        lam, V = np.linalg.eigh(X)
        Xp = (V * np.maximum(lam, 0.0)[..., None, :]) @ np.swapaxes(V, -1, -2)
        out[..., off : off + sz] = mat_to_svec(Xp)
        off += sz
    if cones.ep or cones.ed:
        raise NotImplementedError("exponential cones are not generated")
    return out


# ----------------------------------------------------------------------------- batch container
@dataclass
class Batch:
    """Instance-contiguous ("batch-major") solver data for one structure."""

    structure: Structure
    A_vals: np.ndarray  # [B, nnzA] CSR order
    b: np.ndarray  # [B, m]
    c: np.ndarray  # [B, n]
    P_vals: np.ndarray | None = None  # [B, nnzP] upper-tri CSR order
    x_star: np.ndarray | None = None
    y_star: np.ndarray | None = None
    s_star: np.ndarray | None = None
    name: str = ""
    aux: dict | None = None

    @property
    def B(self) -> int:
        return int(self.A_vals.shape[0])

    def A_dense(self, i: int) -> np.ndarray:
        st = self.structure
        return sp.csr_matrix((self.A_vals[i], st.A_indices, st.A_indptr), shape=(st.m, st.n)).toarray()

    def P_dense(self, i: int) -> np.ndarray:
        st = self.structure
        if st.P_indptr is None:
            return np.zeros((st.n, st.n))
        U = sp.csr_matrix((self.P_vals[i], st.P_indices, st.P_indptr), shape=(st.n, st.n)).toarray()
        return U + U.T - np.diag(np.diag(U))

    def select(self, idx) -> "Batch":
        pick = lambda a: None if a is None else np.ascontiguousarray(a[idx])  # noqa: E731
        return Batch(self.structure, pick(self.A_vals), pick(self.b), pick(self.c), pick(self.P_vals),
                     pick(self.x_star), pick(self.y_star), pick(self.s_star), self.name)


def _apply_A(st: Structure, A_vals: np.ndarray, x: np.ndarray) -> np.ndarray:
    """Batched A @ x for a shared CSR pattern."""
    rows = np.repeat(np.arange(st.m), np.diff(st.A_indptr))
    out = np.zeros((A_vals.shape[0], st.m))
    np.add.at(out, (slice(None), rows), A_vals * x[:, st.A_indices])
    return out


def _apply_AT(st: Structure, A_vals: np.ndarray, y: np.ndarray) -> np.ndarray:
    rows = np.repeat(np.arange(st.m), np.diff(st.A_indptr))
    out = np.zeros((A_vals.shape[0], st.n))
    np.add.at(out, (slice(None), st.A_indices), A_vals * y[:, rows])
    return out


def _apply_P(st: Structure, P_vals: np.ndarray, x: np.ndarray) -> np.ndarray:
    rows = np.repeat(np.arange(st.n), np.diff(st.P_indptr))
    cols = st.P_indices
    out = np.zeros((P_vals.shape[0], st.n))
    np.add.at(out, (slice(None), rows), P_vals * x[:, cols])
    offd = rows != cols
    np.add.at(out, (slice(None), cols[offd]), P_vals[:, offd] * x[:, rows[offd]])
    return out


def plant(st: Structure, A_vals: np.ndarray, P_vals: np.ndarray | None, rng: np.random.Generator, name: str = "",
          active_frac: float | None = None) -> Batch:
    """Attach a planted optimum (SURVEY.md Appendix A.6) to given A (and P) values.

    ``active_frac`` sets the probability that a nonneg row is active (y_i > 0) at the optimum.
    SURVEY.md's plain z ~ N(0,1) activates half of the inequality rows; with m > n that plants
    *more* active constraints than variables -- a primal-degenerate vertex where the dual is not
    unique and the solution map is not differentiable (diffcp's M is then rank deficient beyond
    the homogeneity direction and its LSQR stalls at the 2N cap).  The headline workload keeps
    z + (active nonneg rows) < n so every instance has a well-defined gradient."""
    B = A_vals.shape[0]
    x = rng.standard_normal((B, st.n))
    z = rng.standard_normal((B, st.m))
    if active_frac is not None and st.cones.l:
        lo, hi = st.cones.z, st.cones.z + st.cones.l
        sign = np.where(rng.random((B, st.cones.l)) < active_frac, 1.0, -1.0)
        z[:, lo:hi] = np.abs(z[:, lo:hi]) * sign
    y = proj_dual_cone(z, st.cones)
    s = y - z
    b = _apply_A(st, A_vals, x) + s
    c = -_apply_AT(st, A_vals, y)
    if P_vals is not None:
        c -= _apply_P(st, P_vals, x)
    return Batch(st, np.ascontiguousarray(A_vals), b, c, P_vals, x, y, s, name)


# ----------------------------------------------------------------------------- the five configs
def dense_qp(B: int, n: int, m: int, z: int, seed: int = 0, with_P: bool = True, active_frac: float | None = 0.2) -> Batch:
    """C1 / C2: dense QP, zero + nonneg cones.  A ~ N(0,1)/sqrt(n), P = LL'/n + 0.1 I."""
    rng = np.random.default_rng(seed)
    st = Structure.dense(n, m, ConeSpec(z=z, l=m - z), with_P=with_P)
    A = (rng.standard_normal((B, m * n)) / np.sqrt(n))
    P_vals = None
    if with_P:
        L = rng.standard_normal((B, n, n))
        P = L @ np.swapaxes(L, 1, 2) / n
        P[:, np.arange(n), np.arange(n)] += 0.1
        iu = np.triu_indices(n)
        P_vals = np.ascontiguousarray(P[:, iu[0], iu[1]])
    return plant(st, A, P_vals, rng, name=f"dense_qp_n{n}_m{m}_z{z}", active_frac=active_frac)


def dense_lp(B: int, n: int, m: int, seed: int = 0) -> Batch:
    """Dense LP with a planted NON-DEGENERATE vertex: exactly n of the m nonneg rows are active
    (strict complementarity), so the optimum is unique and the solution map differentiable."""
    rng = np.random.default_rng(seed)
    st = Structure.dense(n, m, ConeSpec(l=m))
    A = rng.standard_normal((B, m * n)) / np.sqrt(n)
    x = rng.standard_normal((B, n))
    z = -np.abs(rng.standard_normal((B, m))) - 0.1
    for i in range(B):
        act = rng.choice(m, size=n, replace=False)
        z[i, act] = np.abs(z[i, act])
    y = np.maximum(z, 0.0)
    s = y - z
    b = _apply_A(st, A, x) + s
    c = -_apply_AT(st, A, y)
    return Batch(st, A, b, c, None, x, y, s, f"dense_lp_n{n}_m{m}")


def qp_as_socp(bt: Batch, factor: str = "cholesky") -> Batch:
    """The same QPs in the form the reference's DIFFCP path hands over: DIFFCP cannot take a quadratic objective
    (``src/cvxpylayers/_quad_form_dpp.py:29-32``: "DIFFCP decomposes quad_form to SOC"), so cvxpy
    canonicalises ``1/2 x'Px`` with ``P = R'R`` through an epigraph variable and one second-order cone of size n + 2,

        min c'x + t   s.t.  (original rows),   (t + 1, t - 1, sqrt2 R x) in SOC     [<=> x'Px <= 2t],

    variables (x, t).  ``factor``:

    * ``"cholesky"`` (default): ``R`` is the upper-triangular Cholesky factor, n (n + 1) / 2 values (25,052 values per instance
      at n = 100 / m = 200: they fit in a CTA's shared memory);
    * ``"eigen"``: cvxpy's own factor, ``decomp_quad``'s eigendecomposition ``P = V diag(lam) V'``, ``R = diag(sqrt(lam)) V'`` --
      a dense n x n block (30,002 values at n = 100 / m = 200, more than a CTA holds: the engine's values-off-chip tier).

    Planted optimum carried over (both factors: the formulas only use R'R = P): t* = 1/2 x*'Px*, cone dual from the KKT
    conditions."""
    st = bt.structure
    n, m, B = st.n, st.m, bt.B
    assert st.P_indptr is not None and not st.cones.q and not st.cones.s
    Pd = np.stack([bt.P_dense(i) for i in range(B)])
    if factor == "cholesky":
        R = np.swapaxes(np.linalg.cholesky(Pd), 1, 2)            # upper triangular, P = R'R
        iu = np.triu_indices(n)
    elif factor == "eigen":
        lam, V = np.linalg.eigh(Pd)
        R = np.sqrt(np.maximum(lam, 0.0))[:, :, None] * np.swapaxes(V, 1, 2)   # dense, P = R'R
        iu = tuple(np.indices((n, n)).reshape(2, -1))
    else:
        raise ValueError(f"factor must be 'cholesky' or 'eigen', got {factor!r}")
    # rows: original m rows (columns 0..n-1), then SOC rows: [t+1], [t-1], sqrt2 R x
    rows, cols = [], []
    for i in range(m):
        lo, hi = st.A_indptr[i], st.A_indptr[i + 1]
        rows += [i] * (hi - lo)
        cols += list(st.A_indices[lo:hi])
    rows += [m, m + 1]
    cols += [n, n]
    for r_, c_ in zip(*iu):
        rows.append(m + 2 + r_)
        cols.append(c_)
    pat = sp.csr_matrix((np.arange(1, len(rows) + 1), (rows, cols)), shape=(m + n + 2, n + 1))
    pat.sort_indices()
    order = pat.data - 1                                     # CSR slot -> position in the construction order above
    st2 = Structure(n + 1, m + n + 2, pat.indptr, pat.indices, ConeSpec(z=st.cones.z, l=st.cones.l, q=[n + 2]))
    vals = np.concatenate([bt.A_vals, -np.ones((B, 2)), -SQRT2 * R[:, iu[0], iu[1]]], axis=1)   # A x + s = b with s = (t+1, t-1, sqrt2 R x)
    A_vals = np.ascontiguousarray(vals[:, order])
    b = np.concatenate([bt.b, np.ones((B, 1)), -np.ones((B, 1)), np.zeros((B, n))], axis=1)
    c = np.concatenate([bt.c, np.ones((B, 1))], axis=1)
    out = Batch(st2, A_vals, b, c, None, name=bt.name + ("_as_socp" if factor == "cholesky" else "_as_socp_eigen"))
    if bt.x_star is not None:
        x = bt.x_star
        Rx = np.einsum("bij,bj->bi", R, x)
        t = 0.5 * (Rx * Rx).sum(1)
        s_soc = np.concatenate([(t + 1)[:, None], (t - 1)[:, None], SQRT2 * Rx], axis=1)
        # dual of the cone from stationarity: the x-columns need -sqrt2 R'y_rest = Px = R'Rx, the t-column 1 - y0 - y1 = 0:
        # y = 1/2 (s0, -s1, -s_rest), on the cone boundary and orthogonal to s
        y_soc = 0.5 * np.concatenate([s_soc[:, :1], -s_soc[:, 1:]], axis=1)
        out.x_star = np.concatenate([x, t[:, None]], axis=1)
        out.y_star = np.concatenate([bt.y_star, y_soc], axis=1)
        out.s_star = np.concatenate([bt.s_star, s_soc], axis=1)
    return out


def config_c1(seed: int = 0) -> Batch:
    return dense_qp(1, 10, 20, 0, seed)


def config_c2(B: int = 4096, seed: int = 0) -> Batch:
    return dense_qp(B, 100, 200, 50, seed)


def socp_portfolio(B: int = 2048, n_assets: int = 50, n_soc: int = 5, k: int = 10, seed: int = 0) -> Batch:
    """C3: min -mu'w  s.t. 1'w = 1, w >= 0, ||F_k' w|| <= sigma_k (SURVEY.md 8d)."""
    rng = np.random.default_rng(seed)
    n = n_assets
    m = 1 + n + n_soc * (k + 1)
    rows, cols = [], []
    rows += [0] * n
    cols += list(range(n))
    for j in range(n):
        rows.append(1 + j)
        cols.append(j)
    base = 1 + n
    for c_ in range(n_soc):
        for r in range(k):
            rows += [base + c_ * (k + 1) + 1 + r] * n
            cols += list(range(n))
    pat = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(m, n))
    pat.sort_indices()
    st = Structure(n, m, pat.indptr, pat.indices, ConeSpec(z=1, l=n, q=[k + 1] * n_soc))
    mu = 0.05 + 0.02 * rng.standard_normal((B, n))
    F = rng.standard_normal((B, n_soc, n, k)) / np.sqrt(k)
    A_vals = np.zeros((B, st.nnzA))
    b = np.zeros((B, m))
    pos = 0
    A_vals[:, pos : pos + n] = 1.0
    pos += n
    b[:, 0] = 1.0
    A_vals[:, pos : pos + n] = -1.0
    pos += n
    for c_ in range(n_soc):
        b[:, base + c_ * (k + 1)] = 0.5
        for r in range(k):
            A_vals[:, pos : pos + n] = -F[:, c_, :, r]
            pos += n
    return Batch(st, A_vals, b, -mu, None, name=f"socp_portfolio_n{n}_q{n_soc}x{k + 1}")


def sparse_lp(B: int = 512, n: int = 1000, m: int = 2000, density: float = 0.01, seed: int = 0) -> Batch:
    """C4: sparse LP, one pattern for the whole batch, fresh values per instance; planted
    non-degenerate vertex (exactly n active rows, strict complementarity)."""
    rng = np.random.default_rng(seed)
    pat = sp.random(m, n, density=density, random_state=np.random.RandomState(seed), format="csr")
    pat.sort_indices()
    st = Structure(n, m, pat.indptr, pat.indices, ConeSpec(l=m))
    A_vals = rng.standard_normal((B, st.nnzA))
    x = rng.standard_normal((B, n))
    z = -np.abs(rng.standard_normal((B, m))) - 0.1
    for i in range(B):
        act = rng.choice(m, size=n, replace=False)
        z[i, act] = np.abs(z[i, act])
    y = np.maximum(z, 0.0)
    s = y - z
    b = _apply_A(st, A_vals, x) + s
    c = -_apply_AT(st, A_vals, y)
    return Batch(st, A_vals, b, c, None, x, y, s, f"sparse_lp_n{n}_m{m}")


def sparse_qp(B: int = 8, n: int = 300, m: int = 600, density: float = 0.03, seed: int = 0) -> Batch:
    """Sparse strongly convex QP (diagonal P) too large for the on-chip Cholesky: exercises the
    CG (indirect) forward path and the L2-resident-vector backward path with a well-defined gradient."""
    rng = np.random.default_rng(seed)
    pat = sp.random(m, n, density=density, random_state=np.random.RandomState(seed), format="csr")
    pat.sort_indices()
    st = Structure(n, m, pat.indptr, pat.indices, ConeSpec(l=m), np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32))
    A_vals = rng.standard_normal((B, st.nnzA))
    P_vals = 0.5 + rng.random((B, n))
    return plant(st, A_vals, P_vals, rng, name=f"sparse_qp_n{n}_m{m}", active_frac=0.2)


def sdp(B: int = 256, k: int = 10, n_eq: int = 10, seed: int = 0, rank: int | None = None) -> Batch:
    """C5: min <C,X> s.t. <A_i,X> = b_i, X >= 0 with x = svec(X); planted optimum.

    ``rank=None`` plants z ~ N(0,1) as SURVEY.md 8d says: the primal optimum then has a random rank r around k/2
    and, with only ``n_eq = 10`` equalities, is NOT unique (the optimal face has r(r+1)/2 > n_eq dimensions), so
    the solution map has no derivative and two correct adjoints only agree up to the choice of a min-norm solution.
    ``rank=r`` plants exactly r positive eigenvalues in the primal slack; with r(r+1)/2 <= n_eq <=
    k(k+1)/2 - (k-r)(k-r+1)/2 the optimum is generically unique, strictly complementary and nondegenerate."""
    rng = np.random.default_rng(seed)
    n = k * (k + 1) // 2
    m = n_eq + n
    rows = np.concatenate([np.repeat(np.arange(n_eq), n), n_eq + np.arange(n)])
    cols = np.concatenate([np.tile(np.arange(n), n_eq), np.arange(n)])
    pat = sp.csr_matrix((np.ones(rows.size), (rows, cols)), shape=(m, n))
    pat.sort_indices()
    st = Structure(n, m, pat.indptr, pat.indices, ConeSpec(z=n_eq, s=[k]))
    G = rng.standard_normal((B, n_eq, k, k))
    Asym = 0.5 * (G + np.swapaxes(G, 2, 3))
    A_vals = np.concatenate([mat_to_svec(Asym).reshape(B, n_eq * n), -np.ones((B, n))], axis=1)
    if rank is None:
        return plant(st, A_vals, None, rng, name=f"sdp_k{k}_eq{n_eq}")
    # planted pair with prescribed inertia: v = y - s, y = Pi(v) has k - rank positive eigenvalues, s = y - v has `rank`
    x = rng.standard_normal((B, n))
    z = rng.standard_normal((B, m))
    Q = np.linalg.qr(rng.standard_normal((B, k, k)))[0]
    lam = np.abs(rng.standard_normal((B, k))) + 0.2
    lam[:, :rank] *= -1.0   # negative eigenvalues of v = positive eigenvalues of the primal slack s
    V = (Q * lam[:, None, :]) @ np.swapaxes(Q, 1, 2)
    z[:, n_eq:] = mat_to_svec(V)
    y = proj_dual_cone(z, st.cones)
    s = y - z
    b = _apply_A(st, A_vals, x) + s
    c = -_apply_AT(st, A_vals, y)
    return Batch(st, np.ascontiguousarray(A_vals), b, c, None, x, y, s, f"sdp_k{k}_eq{n_eq}_rank{rank}")


def exp_sum(B: int = 64, p: int = 6, k: int = 12, lam: float = 1.0, seed: int = 0) -> Batch:
    """Exponential-cone workload:  min  sum_i exp(a_i'x + d_i) + c'x + lam/2 ||x||^2  written with
    k exponential cones (a_i'x + d_i, 1, t_i) in K_exp and the quadratic term as a (diagonal, sparse) P.
    Variables (x in R^p, t in R^k); the reference's exp-cone tests are the logistic-regression / LML
    layers of tests/test_torch.py:158-187,219-230."""
    rng = np.random.default_rng(seed)
    n, m = p + k, 3 * k
    rows, cols = [], []
    for i in range(k):
        rows += [3 * i] * p
        cols += list(range(p))
        rows.append(3 * i + 2)
        cols.append(p + i)
    pat = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(m, n))
    pat.sort_indices()
    pptr = np.concatenate([np.arange(p + 1), np.full(k, p)]).astype(np.int32)
    st = Structure(n, m, pat.indptr, pat.indices, ConeSpec(ep=k), pptr, np.arange(p, dtype=np.int32))
    a = rng.standard_normal((B, k, p)) / np.sqrt(p)
    d = 0.3 * rng.standard_normal((B, k))
    A_vals = np.zeros((B, st.nnzA))
    b = np.zeros((B, m))
    pos = 0
    for i in range(k):
        A_vals[:, pos : pos + p] = -a[:, i, :]
        pos += p
        A_vals[:, pos] = -1.0
        pos += 1
        b[:, 3 * i] = d[:, i]
        b[:, 3 * i + 1] = 1.0
    c = np.concatenate([0.5 * rng.standard_normal((B, p)), np.ones((B, k))], axis=1)
    bt = Batch(st, A_vals, b, c, np.full((B, p), lam), name=f"exp_sum_p{p}_k{k}")
    bt.aux = {"a": a, "d": d, "lam": lam, "p": p, "k": k}
    return bt


CONFIGS = {
    "C1": lambda B=1, seed=0: dense_qp(B, 10, 20, 0, seed),
    "C2": lambda B=4096, seed=0: dense_qp(B, 100, 200, 50, seed),
    # C2 in the form the reference's DIFFCP canonicalisation emits (quad_form -> one SOC of size n + 2)
    "C2SOC": lambda B=4096, seed=0: qp_as_socp(dense_qp(B, 100, 200, 50, seed)),
    "C3": lambda B=2048, seed=0: socp_portfolio(B, seed=seed),
    "C4": lambda B=512, seed=0: sparse_lp(B, seed=seed),
    # C5: 20 equalities and a rank-5 planted optimum (unique, differentiable); C5S is SURVEY.md 8d's literal default
    # (10 equalities, random rank: the optimum is not unique and the solution map has no derivative)
    "C5": lambda B=256, seed=0: sdp(B, n_eq=20, seed=seed, rank=5),
    "C5S": lambda B=256, seed=0: sdp(B, seed=seed),
    "EXP": lambda B=64, seed=0: exp_sum(B, seed=seed),
}


# ----------------------------------------------------------------------------- boundary re-packing
@dataclass
class BoundaryTensors:
    """What ``CvxpyLayer.forward`` hands to ``_CvxpyLayer.apply`` for the DIFFCP backend
    (``torch/cvxpylayer.py:434-451,475``): CSC structure of the m x (n+1) matrix ``[A_cvx | b]``
    plus the per-call value matrices with the batch axis contiguous."""

    con_indices: np.ndarray
    con_ptr: np.ndarray
    shape: tuple[int, int]
    q_eval: np.ndarray  # [n+1, B]
    A_eval: np.ndarray  # [nnz_aug, B]
    P_eval: np.ndarray | None  # [nnzP, B] (upper-tri CSR order) or None
    dims: dict


def to_boundary(batch: Batch, dense_b: bool = True) -> BoundaryTensors:
    """Solver data -> the reference's boundary layout (inverse of ``diffcp_if.py:57-68``:
    there ``A = -A_aug[:, :-1]`` and ``b = A_aug[:, -1]``)."""
    st = batch.structure
    B = batch.B
    pat = sp.csr_matrix((np.arange(1, st.nnzA + 1), st.A_indices, st.A_indptr), shape=(st.m, st.n)).tocsc()
    pat.sort_indices()
    perm = pat.data.astype(np.int64) - 1  # CSC position -> CSR position
    if dense_b:
        b_idx = np.arange(st.m)
    else:
        b_idx = np.nonzero(np.any(batch.b != 0, axis=0))[0]
    con_indices = np.concatenate([pat.indices, b_idx]).astype(np.int64)
    con_ptr = np.concatenate([pat.indptr, [pat.indptr[-1] + b_idx.size]]).astype(np.int64)
    A_eval = np.empty((st.nnzA + b_idx.size, B))
    A_eval[: st.nnzA] = -batch.A_vals[:, perm].T
    A_eval[st.nnzA :] = batch.b[:, b_idx].T
    q_eval = np.zeros((st.n + 1, B))
    q_eval[: st.n] = batch.c.T
    P_eval = None if batch.P_vals is None else np.ascontiguousarray(batch.P_vals.T)
    return BoundaryTensors(con_indices, con_ptr, (st.m, st.n + 1), q_eval, np.ascontiguousarray(A_eval), P_eval,
                           st.cones.to_dict())
