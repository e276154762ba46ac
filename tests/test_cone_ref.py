"""The independent cone reference (tests/cone_ref.py), the C oracle's exponential cone against it, and the planted
mixed-cone batches the GPU cone tests run (tests/cone_planted.py).  CPU only."""
from __future__ import annotations

import numpy as np
import pytest

from cvxpylayers_b200.problems import svec_to_mat
from cvxpylayers_b200.structure import ConeSpec, Structure
from oracle import oracle as orc
from tests import cone_planted as cp
from tests import cone_ref as cr

_ED = Structure(1, 3, np.arange(4), np.zeros(3, np.int32), ConeSpec(ed=1))   # y-block projection onto K_exp
_EP = Structure(1, 3, np.arange(4), np.zeros(3, np.int32), ConeSpec(ep=1))   # y-block projection onto K_exp*

# the first fixture: r > 0 small, s < 0, t > 0, projection at rho = x / y ~ 16.5; the parent scheme returned a point on
# the y = 0 face 1.1e-6 ||v|| away from it
FAILING = [(0.02114319, -0.32819536, 1.20518042), (0.01, -0.2, 2.0), (2.21160257e-12, -7.90544810e-10, 1.41877828e-10)]


def _oracle_J(st, v):
    return np.stack([orc.dproj_dual_cone(st, v, e) for e in np.eye(3)], axis=1)


def _points():
    rng = np.random.default_rng(11)
    pts = [np.array(v) for v in FAILING]
    for mag in (1e-9, 1e-6, 1e-3, 1.0, 1e3):
        pts += [rng.standard_normal(3) * mag for _ in range(16)]
        pts += [cp.exp_point(k % 4, rng) * mag for k in range(8)]
    for _ in range(6):   # near each case boundary: on the inside / polar boundary, just off the r = 0 and s = 0 planes
        rho, a = rng.uniform(-3, 3), rng.uniform(0.5, 2)
        on_k = a * np.array([rho, 1.0, np.exp(rho)])
        u, w = -a, rng.uniform(-2, 2)
        on_polar = -np.array([u, w, -u * np.exp(w / u) / np.e])
        for base in (on_k, on_polar):
            pts += [base * (1 + d) for d in (1e-9, -1e-9)]
        pts += [np.array([d, -a, rho]) for d in (1e-10, -1e-10)] + [np.array([-a, d, rho]) for d in (1e-10, -1e-10)]
    return pts


def test_exp_reference_is_a_projection():
    """Certificates hold by construction; here: the Jacobian is symmetric with eigenvalues in [0, 1] (a projection onto a
    convex set is the gradient of a convex function and nonexpansive), and the projection is positively homogeneous."""
    rng = np.random.default_rng(3)
    for k in range(32):
        v = cp.exp_point(k % 4, rng) if k % 2 else rng.standard_normal(3)
        J = cr.dproj_exp(v)
        assert np.abs(J - J.T).max() <= 1e-12 * max(1, np.abs(J).max())
        ev = np.linalg.eigvalsh(0.5 * (J + J.T))
        assert ev.min() >= -1e-12 and ev.max() <= 1 + 1e-12
        assert np.allclose(cr.proj_exp(1e5 * v), 1e5 * cr.proj_exp(v), rtol=1e-14, atol=0)
        assert cr.exp_case(v) == cr.exp_case(1e-7 * v)


@pytest.mark.parametrize("q,k", [(1, 1), (5, 3), (33, 9)])
def test_soc_psd_reference_certificates_and_jacobian(q, k):
    """SOC and PSD closed forms: Moreau certificate (p in K, p - v in K, p'(p - v) = 0; self-dual) and the Jacobian against
    central differences."""
    cones = ConeSpec(q=[q], s=[k])
    rng = np.random.default_rng(q + k)
    for _ in range(20):
        v = rng.standard_normal(cones.m)
        p = cr.proj_dual(v, cones)
        d = p - v
        for blk in (p, d):
            assert blk[0] >= np.linalg.norm(blk[1:q]) - 1e-12
            assert np.linalg.eigvalsh(svec_to_mat(blk[q:], k)).min() >= -1e-12
        assert abs(p[:q] @ d[:q]) <= 1e-12 and abs(p[q:] @ d[q:]) <= 1e-12
        D, h = cr.dproj_dual(v, cones), 1e-6
        fd = np.stack([(cr.proj_dual(v + h * e, cones) - cr.proj_dual(v - h * e, cones)) / (2 * h) for e in np.eye(cones.m)], axis=1)
        assert np.abs(fd - D).max() <= 1e-7


def test_oracle_exp_projection_and_jacobian_match_reference():
    """The C oracle's K_exp and K_exp* projections (the device's scheme) against the 120-digit reference: random points at
    magnitudes 1e-9..1e3, points of every case, points at and next to each case boundary, and the region r > 0 small,
    s < 0, t > 0 (FAILING).  Projection to 1e-10 ||v|| [worst 6.5e-11]; Jacobian to 1e-8 [2.6e-9] away from the case
    boundaries, where it jumps."""
    worst_p = worst_j = 0.0
    for v in _points():
        nv = np.linalg.norm(v)
        for st, ref in ((_ED, cr.proj_exp), (_EP, cr.proj_exp_dual)):
            err = np.abs(orc.proj_dual_cone(st, v) - ref(v)).max() / nv
            worst_p = max(worst_p, err)
            assert err <= 1e-10, (v, st.cones, err)
        margin = min(abs(v[0]), abs(v[1])) / nv
        if margin > 1e-6 and cr.exp_case(v * (1 + 1e-6)) == cr.exp_case(v * (1 - 1e-6)) == cr.exp_case(v + 1e-6 * nv) == cr.exp_case(v - 1e-6 * nv):
            Jref = cr.dproj_exp(v)
            for st, ref in ((_ED, Jref), (_EP, None)):
                R = ref if ref is not None else cr.dproj_exp_dual(v)
                err = np.abs(_oracle_J(st, v) - R).max()
                worst_j = max(worst_j, err)
                assert err <= 1e-8, (v, st.cones, err)
    print(f"worst projection error {worst_p:.2e} ||v||, worst Jacobian error {worst_j:.2e}")


# r > 0 tiny, s < 0, t > 0: the projection's y underflows (rho = x / y ~ -s / r), the oracle's and the device's Jacobian take
# dproj_exp_mat's y = 0 branch (J = diag([r < 0], 0, [p_z > 0]))
Y0_FACE = [(1e-10, -0.83, 2.26), (1e-9, -1.5, 1.0), (3e-11, -0.2, 0.7), (1e-7, -2.0, 1.0), (1e-12, -1.0, 0.5)]


def test_oracle_exp_jacobian_on_the_y0_branch():
    for v in map(np.array, Y0_FACE):
        p = orc.proj_dual_cone(_ED, v)
        assert p[1] <= 1e-12 * np.abs(v).max() / 2   # below the branch's threshold after the power-of-two scaling
        assert np.abs(_oracle_J(_ED, v) - cr.dproj_exp(v)).max() <= 1e-12
        assert np.abs(_oracle_J(_EP, -v) - cr.dproj_exp_dual(-v)).max() <= 1e-12


@pytest.mark.parametrize("name", list(cp.structures()))
def test_planted_structure_is_certified(name):
    """KKT at the planted point to 1e-12, the oracle solves to it, and central differences of oracle solves along a random
    b, c direction match the reference adjoint (so the solution map is differentiable there and the GPU comparisons have
    one answer)."""
    bt = cp.make(name, B=4)
    st = bt.structure
    for i in range(bt.B):
        A, P = bt.A_dense(i), bt.P_dense(i)
        x, y, s = bt.x_star[i], bt.y_star[i], bt.s_star[i]
        sc = max(1.0, np.abs(bt.b[i]).max(), np.abs(bt.c[i]).max())
        assert np.abs(A @ x + s - bt.b[i]).max() <= 1e-12 * sc
        assert np.abs(P @ x + A.T @ y + bt.c[i]).max() <= 1e-12 * sc
        assert abs(s @ y) <= 1e-12 * sc * sc
        assert np.abs(cr.proj_dual(y - s, st.cones) - y).max() <= 1e-12 * sc
    xo, yo, so, sto, its = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-10, max_iters=200000)
    assert (sto == 1).all()
    assert np.abs(xo - bt.x_star).max() <= 1e-6 and np.abs(so - bt.s_star).max() <= 1e-6 and np.abs(yo - bt.y_star).max() <= 1e-4   # y: m up to 1910 rows
    rng = np.random.default_rng(1)
    i, h = int(np.argmin(its)), 1e-5   # the quickest instance: the two solves at 1e-12 dominate the run time
    dx, dy = rng.standard_normal(st.n), rng.standard_normal(st.m)
    tb, tc = rng.standard_normal(st.m), rng.standard_normal(st.n)
    _, _, db, dc = cr.exact_adjoint(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i], dx, dy, st.cones)
    one = bt.select([i, i])
    bp = np.stack([one.b[0] + h * tb, one.b[1] - h * tb])
    cpl = np.stack([one.c[0] + h * tc, one.c[1] - h * tc])
    xs, ys, _, stf, _ = orc.solve_batch(st, one.A_vals, bp, cpl, one.P_vals, eps=1e-12, max_iters=400000)
    assert (stf == 1).all()
    fd = (dx @ (xs[0] - xs[1]) + dy @ (ys[0] - ys[1])) / (2 * h)
    assert abs(fd - (db @ tb + dc @ tc)) <= 1e-5 * max(1.0, abs(fd))
