"""Solution polishing on the CPU: the NumPy restatement (tests/polish_ref.py) recovers planted optima from C-oracle solves at
eps 1e-3 -- dense QPs, LPs at a vertex, every row an equality, a CSR pattern, whole instances scaled by 1e-4 and 1e3 (which
pins the regularisation relative to the data) -- rejects a wrong active set without touching the input, never returns larger
residuals than its input's, and ``polish`` is a layer option the solver settings accept."""
from __future__ import annotations

import numpy as np
import pytest

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import make_settings
from cvxpylayers_b200.structure import ConeSpec, Structure
from oracle import oracle as orc
from tests import polish_ref as pref
from tests import tiled_shapes as ts


def _scaled(bt, a):
    return pr.Batch(bt.structure, bt.A_vals * a, bt.b * a, bt.c * a, None if bt.P_vals is None else bt.P_vals * a,
                    bt.x_star, bt.y_star, None if bt.s_star is None else bt.s_star * a, bt.name + f"_x{a:g}")


def _csr_qp(B, n, m, z, seed):
    """A random CSR pattern (about a third of the entries, every row non-empty) and a diagonal P, planted by problems.plant."""
    rng = np.random.default_rng(seed)
    mask = rng.random((m, n)) < 0.35
    mask[np.arange(m), rng.integers(0, n, m)] = True
    indptr = np.r_[0, np.cumsum(mask.sum(1))].astype(np.int32)
    indices = np.nonzero(mask)[1].astype(np.int32)
    st = Structure(n, m, indptr, indices, ConeSpec(z=z, l=m - z), np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32))
    A = rng.standard_normal((B, indices.size)) / np.sqrt(n * 0.35)
    P = rng.uniform(0.5, 2.0, (B, n))
    return pr.plant(st, A, P, rng, name="csr_qp", active_frac=0.2)


def _batches():
    """name -> (batch, oracle settings); a scaled instance keeps eps_abs relative to its data (at 1e-4 an absolute 1e-3 would
    accept the first iterate)"""
    e = {"eps": 1e-3, "max_iters": 100000}
    return {
        "dense_qp": (pr.dense_qp(4, 20, 30, 5, seed=11), e),
        "lp_vertex": (ts.planted(ts.Case(12, 30, 4, 8, False, 1), 4, seed=3), e),
        "all_equality": (pr.dense_qp(4, 20, 12, 12, seed=5), e),
        "csr_qp": (_csr_qp(4, 16, 24, 3, seed=7), e),
        "scale_1e-4": (_scaled(pr.dense_qp(4, 20, 30, 5, seed=13), 1e-4), {**e, "eps_abs": 1e-7, "eps_rel": 1e-3}),
        "scale_1e3": (_scaled(pr.dense_qp(4, 20, 30, 5, seed=13), 1e3), {**e, "eps_abs": 1.0, "eps_rel": 1e-3}),
    }


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.mark.parametrize("key", list(_batches()))
def test_polish_recovers_the_planted_optimum(key):
    bt, args = _batches()[key]
    x, y, s, status, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, **args)
    assert (status == 1).all(), (key, status)
    far = max(_rel(x, bt.x_star), _rel(y, bt.y_star))
    flags, X, Y, S = pref.polish_batch(bt, x, y, s, status)
    assert (flags == 1).all(), (key, flags)
    err = max(_rel(X, bt.x_star), _rel(Y, bt.y_star), _rel(S, bt.s_star))
    assert err < 1e-10, (key, err, far)
    assert far > 1e3 * err, (key, far, err)   # (the unpolished point really was inexact)


def test_wrong_active_set_is_rejected_and_the_input_kept():
    bt = pr.dense_qp(4, 20, 30, 5, seed=11)
    x, y, s, status, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-3, max_iters=5)
    z = bt.structure.cones.z
    wrong = [i for i in range(bt.B) if not np.array_equal(y[i, z:] > s[i, z:], bt.y_star[i, z:] > 0)]
    assert wrong, "every 5-iteration iterate already has the planted active set"
    flags, X, Y, S = pref.polish_batch(bt, x, y, s, np.ones(bt.B, dtype=np.int32))
    rejected = [i for i in wrong if flags[i] == 0]
    assert rejected, (flags, wrong)
    for i in rejected:
        assert np.array_equal(X[i], x[i]) and np.array_equal(Y[i], y[i]) and np.array_equal(S[i], s[i])


@pytest.mark.parametrize("iters", [5, 50, 100000])
def test_residuals_never_grow(iters):
    bt = pr.dense_qp(6, 20, 30, 5, seed=17)
    x, y, s, status, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-3, max_iters=iters)
    flags, X, Y, S = pref.polish_batch(bt, x, y, s, np.ones(bt.B, dtype=np.int32))
    for i in range(bt.B):
        A, P = bt.A_dense(i), bt.P_dense(i)
        r_in = pref.metrics(A, P, bt.b[i], bt.c[i], x[i], y[i], s[i])
        r_out = pref.metrics(A, P, bt.b[i], bt.c[i], X[i], Y[i], S[i])
        assert np.all(r_out <= r_in), (i, flags[i], r_in, r_out)


def test_not_attempted_for_other_status_or_non_finite_input():
    bt = pr.dense_qp(1, 6, 9, 2, seed=1)
    x, y, s = bt.x_star[0], bt.y_star[0], bt.s_star[0]
    A, P = bt.A_dense(0), bt.P_dense(0)
    assert pref.polish_one(A, P, bt.b[0], bt.c[0], x, y, s, 2, status=-4)[0] == -1
    assert pref.polish_one(A, P, bt.b[0], bt.c[0], np.full_like(x, np.nan), y, s, 2)[0] == -1


def test_polish_is_a_layer_option_not_a_solver_setting():
    st = make_settings({"polish": True, "eps": 1e-5})
    assert st.eps_abs == 1e-5
