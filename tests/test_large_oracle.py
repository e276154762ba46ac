"""CPU checks of the instances that need the engine's values-off-chip tier: cvxpy's own (eigen) factor in the SOC form of a QP.

* The eigen-factor batch of ``problems.qp_as_socp`` carries a certified planted optimum.
* The oracle's adjoint of the triangular and the eigen form agree on ``dc`` (the first n entries) and ``db`` (the original rows)
  when the cotangents sit only on x and on the duals of the original rows: both forms are then the same function of (b, c).
  tests/test_gpu_large.py relies on that identity to compare the new tier against the on-chip kernels on the same QPs.
"""
import numpy as np
import pytest

from cvxpylayers_b200 import problems as pr
from oracle import np_ref
from oracle import oracle as orc
from tests.util import rel_err

TIGHT = dict(lsqr_precond=1, lsqr_iter_lim=50000, lsqr_atol=1e-12, lsqr_btol=1e-12)


def _soc_ok(v, tol):
    return v[0] >= np.linalg.norm(v[1:]) - tol


@pytest.mark.parametrize("n,m,z,B", [(100, 200, 50, 3), (20, 40, 10, 4)])
def test_eigen_factor_batch_has_a_certified_planted_optimum(n, m, z, B):
    bq = pr.dense_qp(B, n, m, z, seed=1)
    bt = pr.qp_as_socp(bq, factor="eigen")
    st = bt.structure
    assert (st.n, st.m, st.nnzA) == (n + 1, m + n + 2, m * n + 2 + n * n)   # the dense n x n factor block
    assert st.cones.q == [n + 2]
    for i in range(B):   # R'R = P, as in the triangular form
        R = -bt.A_dense(i)[m + 2:, :n] / pr.SQRT2
        assert np.abs(R.T @ R - bq.P_dense(i)).max() < 1e-10
    for i in range(B):
        r = np_ref.kkt_residuals(bt.A_dense(i), None, bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i])
        assert max(r["rp"], r["rd"], r["gap"]) < 1e-9 * max(1.0, r["tp"], r["td"], r["tg"]), r
        s, y = bt.s_star[i], bt.y_star[i]
        assert np.abs(s[:z]).max() == 0.0 and (s[z:m] >= 0).all() and (y[z:m] >= 0).all()
        assert _soc_ok(s[m:], 1e-9) and _soc_ok(y[m:], 1e-9)
        assert abs(s @ y) < 1e-9 * max(1.0, np.abs(s).max() * np.abs(y).max())
    x, y, s, status, _ = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, None, eps=1e-10, max_iters=400000)
    assert (status == 1).all()
    assert np.abs(x - bt.x_star).max() < 1e-6 * max(1.0, np.abs(bt.x_star).max())


def test_eigen_form_keeps_the_qp_data_of_the_triangular_form():
    bq = pr.dense_qp(2, 12, 24, 4, seed=3)
    bc, be = pr.qp_as_socp(bq), pr.qp_as_socp(bq, factor="eigen")
    m = bq.structure.m
    assert np.array_equal(bc.b, be.b) and np.array_equal(bc.c, be.c)
    for i in range(bq.B):
        assert np.array_equal(bc.A_dense(i)[: m + 2], be.A_dense(i)[: m + 2])
    n = bq.structure.n
    assert np.array_equal(bc.x_star[:, :n], be.x_star[:, :n]) and np.array_equal(bc.y_star[:, :m], be.y_star[:, :m])
    assert rel_err(be.x_star[:, n], bc.x_star[:, n]) < 1e-12   # t* = 1/2 |Rx|^2, rounded differently
    with pytest.raises(ValueError):
        pr.qp_as_socp(bq, factor="ldl")


@pytest.mark.parametrize("n,m,z,B", [(100, 200, 50, 2), (20, 40, 10, 4)])
def test_oracle_adjoint_agrees_between_triangular_and_eigen_forms(n, m, z, B):
    bq = pr.dense_qp(B, n, m, z, seed=2)
    forms = [pr.qp_as_socp(bq), pr.qp_as_socp(bq, factor="eigen")]
    rng = np.random.default_rng(7)
    dx = np.concatenate([rng.standard_normal((B, n)), np.zeros((B, 1))], axis=1)          # nothing on the epigraph variable
    dy = np.concatenate([rng.standard_normal((B, m)), np.zeros((B, n + 2))], axis=1)      # nothing on the SOC rows
    grads = []
    for bt in forms:
        st = bt.structure
        x, y, s, status, _ = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, None, eps=1e-11, max_iters=400000)
        assert (status == 1).all()
        _, _, db, dc, its = orc.vjp_batch(st, bt.A_vals, bt.b, bt.c, x, y, s, dx, dy, None, **TIGHT)
        assert (its > 0).all()
        grads.append((db[:, :m], dc[:, :n]))
    (db1, dc1), (db2, dc2) = grads
    assert rel_err(db2, db1) < 1e-6 and rel_err(dc2, dc1) < 1e-6, (rel_err(db2, db1), rel_err(dc2, dc1))
