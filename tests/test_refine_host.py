"""Solution refinement on the CPU: the NumPy restatement (tests/refine_ref.py) takes C-oracle solves at eps 1e-3 and 1e-4 and
perturbed planted optima to the planted optimum on every cone_planted structure small enough for dense least squares, on dense
QPs and on LPs; structures with exponential cones reach the bounds of EXP_BOUND and always improve on their input.  No residual
of polishing's acceptance rule ever grows, an instance scaled by 1e-4 or 1e3 refines to the scaled result, and non-solved and
non-finite rows are not attempted.  ``refine`` is a layer option the solver settings accept."""
from __future__ import annotations

import numpy as np
import pytest

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import make_settings
from oracle import oracle as orc
from tests import cone_planted as cp
from tests import refine_ref as rref
from tests import tiled_shapes as ts
from tests.polish_ref import metrics

# (many_blocks -- 600 exponential cones -- is left to the GPU tests: its dense twin takes minutes)
STRUCTS = ["soc_sizes", "psd_warm", "psd_serial", "exp", "mixed", "dense_qp", "lp_vertex"]
# error to the planted optimum the restatement reaches with lsqr_precond = 1 where the structure has exponential cones (LSQR
# hits its iteration limit there, DESIGN.md section 9); 1e-9 everywhere else
EXP_BOUND = {"exp": 1e-3, "mixed": 1e-5}
STARTS = ["eps1e-3", "eps1e-4", "pert1e-4", "pert1e-2"]


def _batch(name, B=2):
    if name == "dense_qp":
        return pr.dense_qp(B, 20, 30, 5, seed=11)
    if name == "lp_vertex":   # (an LP whose planted optimum is its only one: problems.dense_lp's need not be)
        return ts.planted(ts.Case(12, 30, 4, 8, False, 1), B, seed=3)
    return cp.make(name, B)


def _start(bt, start):
    if start.startswith("eps"):
        x, y, s, status, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=float(start[3:]), max_iters=100000)
        return x, y, s, status
    h = float(start[4:])
    rng = np.random.default_rng(1)
    x = bt.x_star + h * rng.standard_normal(bt.x_star.shape)
    return x, bt.y_star + h * rng.standard_normal(bt.y_star.shape), bt.s_star + h * rng.standard_normal(bt.s_star.shape), np.ones(bt.B, np.int32)


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _err(bt, x, y):
    return max(_rel(x, bt.x_star), _rel(y, bt.y_star))


def _metrics(bt, i, x, y, s):
    return metrics(bt.A_dense(i), bt.P_dense(i) if bt.P_vals is not None else None, bt.b[i], bt.c[i], x, y, s)


@pytest.mark.parametrize("start", STARTS)
@pytest.mark.parametrize("name", STRUCTS)
def test_refinement_reaches_the_planted_optimum(name, start):
    bt = _batch(name)
    x, y, s, status = _start(bt, start)
    assert (status == 1).all(), (name, status)
    steps = 4 if start == "pert1e-2" else 3   # (the far start takes one step more)
    flags, X, Y, S = rref.refine_batch(bt, x, y, s, status, steps=steps, precond=1)
    e_in, e_out = _err(bt, x, y), _err(bt, X, Y)
    bound = EXP_BOUND.get(name, 1e-9)
    assert (flags == 1).all(), (name, start, flags)
    assert e_out <= bound and e_out < e_in, (name, start, e_in, e_out)
    for i in range(bt.B):   # (the candidate is (x, pi, pi - v): exactly complementary)
        assert abs(Y[i] @ S[i]) <= 1e-12 * max(1.0, np.abs(Y[i]).max() * np.abs(S[i]).max() * S.shape[1]), (name, i)
    if name not in EXP_BOUND:
        _, X0, Y0, _ = rref.refine_batch(bt, x, y, s, status, steps=steps, precond=0)
        assert _err(bt, X0, Y0) <= 1e-9, (name, start, _err(bt, X0, Y0))


@pytest.mark.parametrize("iters", [5, 50, 100000])
@pytest.mark.parametrize("name", ["dense_qp", "mixed"])
def test_residuals_never_grow(name, iters):
    bt = _batch(name, 3)
    x, y, s, _, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-3, max_iters=iters)
    flags, X, Y, S = rref.refine_batch(bt, x, y, s, np.ones(bt.B, dtype=np.int32), steps=2, precond=1)
    for i in range(bt.B):
        r_in, r_out = _metrics(bt, i, x[i], y[i], s[i]), _metrics(bt, i, X[i], Y[i], S[i])
        assert np.all(r_out <= r_in), (name, iters, i, flags[i], r_in, r_out)
        if flags[i] != 1:
            assert np.array_equal(X[i], x[i]) and np.array_equal(Y[i], y[i]) and np.array_equal(S[i], s[i])


def _scaled(bt, a):
    return pr.Batch(bt.structure, bt.A_vals * a, bt.b * a, bt.c * a, None if bt.P_vals is None else bt.P_vals * a,
                    bt.x_star, bt.y_star, bt.s_star * a, bt.name + f"_x{a:g}")


@pytest.mark.parametrize("name, a", [("dense_qp", 1e-4), ("dense_qp", 1e3), ("soc_sizes", 1e3)])
def test_scaled_instance_refines_to_the_scaled_result(name, a):
    """A whole instance multiplied by a has the same x and y and a times s: from an oracle solve of the scaled instance (eps_abs
    relative to its data) the refinement returns x*, y* and a s*.  (soc_sizes at 1e-4 does not: LSQR's relative tolerance
    leaves each step short there, DESIGN.md section 9.)"""
    bt = _scaled(_batch(name), a)
    x, y, s, status, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps_abs=1e-4 * a, eps_rel=1e-4, max_iters=100000)
    assert (status == 1).all(), status
    flags, X, Y, S = rref.refine_batch(bt, x, y, s, status, precond=1)
    assert (flags == 1).all(), flags
    err = max(_rel(X, bt.x_star), _rel(Y, bt.y_star), _rel(S / a, bt.s_star / a))
    assert err <= 1e-9 < max(_rel(x, bt.x_star), _rel(y, bt.y_star)), err


def test_not_attempted_for_other_status_or_non_finite_input():
    bt = _batch("soc_sizes", 1)
    x, y, s = bt.x_star[0], bt.y_star[0], bt.s_star[0]
    A, P = bt.A_dense(0), bt.P_dense(0)
    args = (bt.structure, A, P, bt.b[0], bt.c[0])
    for st in (-4, -2, -1, 0):
        assert rref.refine_one(*args, x, y, s, status=st)[0] == -1
    for bad in (np.nan, np.inf):
        xb = x.copy()
        xb[0] = bad
        out = rref.refine_one(*args, xb, y, s)
        assert out[0] == -1 and out[1] is xb


def test_refine_is_a_layer_option_not_a_solver_setting():
    st = make_settings({"refine": 3, "eps": 1e-5})
    assert st.eps_abs == 1e-5
