"""Forward-mode derivative of the solution map (diffcp's ``D``) on the CPU: the dense restatement ``tests/jvp_ref.jvp_dense``
against central differences of oracle solves, and against the committed adjoint ``np_ref.vjp_dense`` through the adjoint
identity <w, J t> = <J'w, t>.  These pin the definition the GPU kernel (``bcone_jvp``) is tested against."""
import numpy as np
import pytest

from cvxpylayers_b200 import problems as pr
from oracle import np_ref
from oracle import oracle as orc
from tests.jvp_ref import jvp_dense, random_tangents, shifted

FWD = {"eps": 1e-12, "max_iters": 400000}


def _solve(bt):
    x, y, s, status, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, **FWD)
    assert (status == 1).all()
    return x, y, s


def _jvp_instance(bt, t, i, x, y, s, **kw):
    P = bt.P_dense(i) if bt.P_vals is not None else None
    dP = t.P_dense(i) if t.P_vals is not None else None
    return jvp_dense(bt.structure, bt.A_dense(i), P, bt.b[i], bt.c[i], x[i], y[i], s[i], t.A_dense(i), dP, t.b[i], t.c[i], **kw)


@pytest.mark.parametrize("name", ["C1", "C3", "C5", "EXP"])
def test_jvp_dense_matches_central_differences(name):
    bt = pr.CONFIGS[name](B=2)
    t = random_tangents(bt, np.random.default_rng(11))
    x, y, s = _solve(bt)
    h = 1e-6
    xp, yp, sp_ = _solve(shifted(bt, t, h))
    xm, ym, sm = _solve(shifted(bt, t, -h))
    for i in range(bt.B):
        dx, dy, ds, _ = _jvp_instance(bt, t, i, x, y, s)
        for d, fd, what in ((dx, (xp[i] - xm[i]) / (2 * h), "dx"), (dy, (yp[i] - ym[i]) / (2 * h), "dy"), (ds, (sp_[i] - sm[i]) / (2 * h), "ds")):
            scale = max(np.abs(fd).max(), 1.0)
            assert np.abs(d - fd).max() <= 1e-5 * scale, (name, i, what, np.abs(d - fd).max(), scale)


@pytest.mark.parametrize("name", ["C1", "C3", "C5"])
def test_jvp_dense_is_the_transpose_of_vjp_dense(name):
    """All four data tangents perturbed; exact least squares in both directions (np_ref has no exponential-cone Jacobian)."""
    bt = pr.CONFIGS[name](B=2)
    st = bt.structure
    rng = np.random.default_rng(12)
    t = random_tangents(bt, rng)
    x, y, s = _solve(bt)
    for i in range(bt.B):
        dx, dy, _, _ = _jvp_instance(bt, t, i, x, y, s)
        wx, wy = rng.standard_normal(st.n), rng.standard_normal(st.m)
        P = bt.P_dense(i) if bt.P_vals is not None else None
        gA, gP, gb, gc, _ = np_ref.vjp_dense(bt.A_dense(i), P, bt.b[i], bt.c[i], x[i], y[i], s[i], wx, wy, st.cones, exact=True)
        lhs = wx @ dx + wy @ dy
        rhs = (gA * t.A_dense(i)).sum() + gb @ t.b[i] + gc @ t.c[i]
        if t.P_vals is not None:
            rhs += (gP * t.P_dense(i)).sum()
        assert abs(lhs - rhs) <= 1e-10 * max(abs(lhs), abs(rhs)), (name, i, lhs, rhs)


def test_zero_tangent_gives_zero():
    bt = pr.CONFIGS["C3"](B=1)
    x, y, s = _solve(bt)
    z = random_tangents(bt, np.random.default_rng(0))
    z = shifted(z, z, -1.0)   # all zeros, same shapes
    dx, dy, ds, zz = _jvp_instance(bt, z, 0, x, y, s)
    assert not np.any(dx) and not np.any(dy) and not np.any(ds) and not np.any(zz)
