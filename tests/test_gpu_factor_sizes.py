"""The packed Cholesky + inverse (common.cuh: chol_inv_packed) advances eight columns per step; these dense QPs put n on
every residue mod 8, so every shape of the last, partial block is factored:

* n = 9..16 and 96..103 (m = 2n): the forward factors K at every size (on chip, register-tiled, or in the global slab
  at n = 102, 103); the block-preconditioned backward, where the shape selects it, factors P and S;
* a P with an exactly zero row and column: the backward's factorisation of P must report "not positive definite" and hand
  the instance to the fallback solver, whose gradient still matches the oracle.

All through the C ABI against the CPU oracle, at the tolerances of test_gpu_parity / test_gpu_fullsize.
"""
import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from oracle import np_ref
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

EPS = 1e-8
FWD = {"eps": EPS, "max_iters": 100000}
BWD_GPU = {"lsqr_precond": 2}
BWD_ORACLE = {"lsqr_precond": 1, "lsqr_iter_lim": 20000}
BLOCK_BWD = "bwd_block_kernel (KKT-block preconditioned, bwd_fast_kernel fallback)"


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _rel(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _check_against_oracle(bt, dev, expect_fallbacks):
    st, B = bt.structure, bt.B
    eng = Engine(st, dev)
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    sol = eng.solve(A, b, c, P, make_settings(FWD))
    torch.cuda.synchronize()
    paths = eng.path_info()
    block = paths["bwd"] == BLOCK_BWD
    assert "Cholesky" in paths["fwd"] or "register-tiled" in paths["fwd"], paths   # a factoring forward, on chip or in the slab
    assert block or not expect_fallbacks, paths
    assert (sol.status.cpu().numpy() == 1).all(), sol.status
    x, y, s = sol.x.cpu().numpy(), sol.y.cpu().numpy(), sol.s.cpu().numpy()
    for i in range(B):
        r = np_ref.kkt_residuals(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], x[i], y[i], s[i])
        assert np_ref.is_converged(r, EPS, EPS, 1.001), (i, r)
    xo, yo, so, sto, _ = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, bt.P_vals, **FWD)
    assert (sto == 1).all()
    assert np.abs(x - xo).max() <= 20 * EPS * max(1.0, np.abs(xo).max())
    # the adjoint at the oracle's solution: both sides differentiate the same point
    rng = np.random.default_rng(st.n)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    gA, gP, gb, gc, _ = eng.vjp(A, b, c, _t(xo, dev), _t(yo, dev), _t(so, dev), _t(dx, dev), _t(dy, dev), P, make_settings(BWD_GPU))
    torch.cuda.synchronize()
    assert eng.fallback_count() == (expect_fallbacks if block else -1)   # (-1: the block solver is not in use for this shape)
    rA, rP, rb, rc, _ = orc.vjp_batch(st, bt.A_vals, bt.b, bt.c, xo, yo, so, dx, dy, bt.P_vals, **BWD_ORACLE)
    for name, g_, r_ in (("dA", gA, rA), ("dP", gP, rP), ("db", gb, rb), ("dc", gc, rc)):
        assert _rel(g_, r_) < 1e-4, (name, _rel(g_, r_))


@pytest.mark.parametrize("n", list(range(9, 17)) + list(range(96, 104)))
def test_every_residue_mod_8(n, cuda_device):
    bt = pr.dense_qp(4, n, 2 * n, n // 4, seed=n)
    _check_against_oracle(bt, cuda_device, expect_fallbacks=0)


def test_singular_P_goes_to_the_fallback(cuda_device):
    n, m = 100, 200
    bt = pr.dense_qp(3, n, m, 50, seed=11)
    # instance 1: row and column 45 of P are zero (a PSD P whose Cholesky meets an exact zero pivot inside an
    # 8-column block); the planted optimum is re-attached so that it stays the solution of the new data
    Pd = np.stack([bt.P_dense(i) for i in range(bt.B)])
    Pd[1, 45, :] = 0.0
    Pd[1, :, 45] = 0.0
    iu = np.triu_indices(n)
    P_vals = np.ascontiguousarray(Pd[:, iu[0], iu[1]])
    bt = pr.plant(bt.structure, bt.A_vals, P_vals, np.random.default_rng(12), name="dense_qp_singular_P", active_frac=0.2)
    _check_against_oracle(bt, cuda_device, expect_fallbacks=1)
