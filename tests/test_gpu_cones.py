"""Every cone shape the generic kernels accept, on planted mixed-cone batches (tests/cone_planted.py), against the
independent reference of tests/cone_ref.py: the forward solve against the planted optimum (default plan, warm start, values
off chip, the 4-CTA/SM build, the indirect forward), the adjoint and the forward-mode derivative at the planted point
against dense least squares with the reference cone Jacobian, their adjoint identity, central differences of GPU solves
against the GPU adjoint, and the scale covariance of the solution map.

Tolerances: TOL, with the worst errors measured on an H100 80GB HBM3 (700 W) over all structures below it.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cvxpylayers_b200.engine import Engine, make_settings
from tests import cone_planted as cp
from tests import cone_ref as cr

pytestmark = pytest.mark.gpu

NAMES = list(cp.structures())
_CACHE: dict = {}
FWD = {"eps_abs": 1e-10, "eps_rel": 1e-10, "max_iters": 400000}
TIGHT = {"lsqr_atol": 1e-14, "lsqr_btol": 1e-14, "lsqr_conlim": 1e14}
TOL = {
    # relative to max(1, |planted|_inf).  y is the least well determined: its error is the dual residual over the smallest
    # singular value of A' on the dual face (many_blocks: 1910 rows)
    "x": 1e-6, "s": 1e-6, "y": 1e-4,
    # relative to the exact answer's largest entry
    "adjoint_precond1": 1e-9, "adjoint_precond0": 1e-7, "jvp": 1e-9, "identity": 1e-8,
    # relative to max(1, |fd|): the solve error over h, largest on many_blocks whose y is the least well determined
    "central_differences": 1e-4, "scale": 1e-8,
}
# worst measured: x 1.3e-7, s 6.7e-9, y 3.5e-6 (many_blocks); adjoint lsqr_precond 1 1.3e-11, 0 1.6e-9; jvp 1.4e-11;
# identity 3.3e-10; central differences 2.3e-5 (many_blocks; the others <= 3.3e-6); scale 1.0e-11


def _batch(name):
    if name not in _CACHE:
        _CACHE[name] = cp.make(name, B=4)
    return _CACHE[name]


def _dense_M(name, i):
    """The reference's dense M, D, pi_y at instance i's planted point (cached: the exponential Jacobians are 120-digit)."""
    key = (name, i)
    if key not in _CACHE:
        bt = _batch(name)
        _CACHE[key] = cr.dense_M(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i], bt.structure.cones)
    return _CACHE[key]


def _t(a, dev):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _lsqr(bt, precond):
    return make_settings({**TIGHT, "lsqr_precond": precond, "lsqr_iter_lim": 50 * (bt.structure.n + bt.structure.m + 1)})


def _solve(eng, bt, dev, **extra):
    return eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings({**FWD, **extra}))


def _check_forward(bt, sol, what, tol=TOL):
    st = sol.status.cpu().numpy()
    assert (st == 1).all(), (what, st, sol.iters.cpu().numpy())
    x, y, s = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s))
    errs = {k: max(_rel(got[i], ref[i]) for i in range(bt.B)) for k, got, ref in (("x", x, bt.x_star), ("y", y, bt.y_star), ("s", s, bt.s_star))}
    print(f"{what}: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()) + f" iters {sol.iters.cpu().numpy()}")
    assert all(errs[k] <= tol[k] for k in errs), (what, errs)


def _sym(st, vals):
    """Full symmetric matrix from values on P's upper-triangular pattern."""
    rows = np.repeat(np.arange(st.n), np.diff(st.P_indptr))
    U = np.zeros((st.n, st.n)); U[rows, st.P_indices] = vals
    return U + U.T - np.diag(np.diag(U))


def _upper(st, G):
    """Gradient with respect to the values on P's upper-triangular pattern from the gradient G of a full unsymmetric P."""
    rows = np.repeat(np.arange(st.n), np.diff(st.P_indptr))
    cols = st.P_indices
    return np.where(rows == cols, G[rows, cols], G[rows, cols] + G[cols, rows])


@pytest.mark.parametrize("name", NAMES)
def test_forward_matches_planted_optimum(name, cuda_device, monkeypatch):
    """Default plan, warm start at the planted point, and the values-off-chip tier."""
    bt, dev = _batch(name), cuda_device
    eng = Engine(bt.structure, dev)
    info, path = eng.kernel_info(), eng.path_info()
    print(name, info, path)
    if name == "many_blocks":   # keeps covering the strided loops if the geometry rule changes
        ncb = len(bt.structure.cones.q) + len(bt.structure.cones.s)
        ne = bt.structure.cones.ep + bt.structure.cones.ed
        assert ncb > info["fwd_threads"] // 32 and ncb > info["bwd_threads"] // 32
        assert ne > info["fwd_threads"] and ne > info["bwd_threads"]
    _check_forward(bt, _solve(eng, bt, dev), f"{name} default [{path['fwd']}]")
    warm = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings(FWD),
                     warm=(_t(bt.x_star, dev), _t(bt.y_star, dev), _t(bt.s_star, dev)))
    _check_forward(bt, warm, f"{name} warm")
    monkeypatch.setenv("BCONE_VALUES_GLOBAL", "1")
    eng_g = Engine(bt.structure, dev)
    _check_forward(bt, _solve(eng_g, bt, dev), f"{name} values global [{eng_g.path_info()['fwd']}]")


@pytest.mark.parametrize("name", NAMES)
def test_forward_small_cta(name, cuda_device, monkeypatch):
    """BCONE_SMALL_CTA=2: every forward launch takes the 4-CTA/SM build, where the structure has one."""
    bt, dev = _batch(name), cuda_device
    monkeypatch.setenv("BCONE_SMALL_CTA", "2")
    eng = Engine(bt.structure, dev)
    small, info = eng.small_cta_info(), eng.kernel_info()
    if not small["fwd"]:
        pytest.skip(f"no 4-CTA/SM forward build: {info['fwd_threads']} threads, {info['fwd_smem']} B of shared memory, "
                    f"{info['fwd_ctas_per_sm']} CTAs/SM already ({eng.path_info()['fwd']})")
    assert small["fwd"] > info["fwd_ctas_per_sm"]
    _check_forward(bt, _solve(eng, bt, dev), f"{name} small CTA ({small['fwd']} CTAs/SM)")


# The indirect forward exists for instances whose Cholesky factor does not fit on chip: of these structures only
# many_blocks (n = 72, m = 1910) is one.  Its inexact CG solves (tolerance 0.1 / k^1.5 relative at iteration k, at most 1e-6)
# bound the accuracy it reaches, hence the looser eps.
INDIRECT_EPS = 1e-7
INDIRECT_TOL = {"x": 1e-4, "s": 1e-4, "y": 1e-3}


@pytest.mark.xfail(strict=True, reason="the indirect (CG) forward does not converge on many_blocks, at eps 1e-10 in 400000 "
                   "iterations nor at eps 1e-7 in 100000 (status 2 on every instance); cause not found yet (DESIGN section 9)")
def test_forward_indirect(cuda_device, monkeypatch):
    bt, dev = _batch("many_blocks"), cuda_device
    monkeypatch.setenv("BCONE_FWD_MODE", "indirect")
    eng = Engine(bt.structure, dev)
    assert "indirect" in eng.path_info()["fwd"]
    sol = _solve(eng, bt, dev, eps_abs=INDIRECT_EPS, eps_rel=INDIRECT_EPS, max_iters=100000)
    _check_forward(bt, sol, "many_blocks indirect", INDIRECT_TOL)


def _at_planted(bt, dev):
    return [_t(a, dev) for a in (bt.A_vals, bt.b, bt.c, bt.x_star, bt.y_star, bt.s_star)]


@pytest.mark.parametrize("precond", [1, 0])
@pytest.mark.parametrize("name", NAMES)
def test_adjoint_matches_exact_least_squares(name, precond, cuda_device):
    """Engine.vjp at the exact planted (x, y, s), so v = y - s sits where the generator put it (every exponential case),
    against lstsq with the reference cone Jacobian: dA, dP, db, dc."""
    bt, dev = _batch(name), cuda_device
    st = bt.structure
    eng = Engine(st, dev)
    rng = np.random.default_rng(7)
    dx, dy = rng.standard_normal((bt.B, st.n)), rng.standard_normal((bt.B, st.m))
    A, b, c, x, y, s = _at_planted(bt, dev)
    gA, gP, gb, gc, its = eng.vjp(A, b, c, x, y, s, _t(dx, dev), _t(dy, dev), _t(bt.P_vals, dev), _lsqr(bt, precond))
    gA, gP, gb, gc = (t.cpu().numpy() for t in (gA, gP, gb, gc))
    rows = np.repeat(np.arange(st.m), np.diff(st.A_indptr))
    worst = 0.0
    for i in range(bt.B):
        dA, dP, db, dc = cr.exact_adjoint(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i],
                                          dx[i], dy[i], st.cones, _dense_M(name, i))
        ref = np.concatenate([dA[rows, st.A_indices], _upper(st, dP), db, dc])
        got = np.concatenate([gA[i], gP[i], gb[i], gc[i]])
        worst = max(worst, np.abs(got - ref).max() / np.abs(ref).max())
    print(f"{name} precond {precond}: adjoint worst {worst:.1e}, LSQR iterations {its.cpu().numpy()}")
    assert worst <= TOL[f"adjoint_precond{precond}"]


@pytest.mark.parametrize("name", NAMES)
def test_jvp_matches_exact_and_adjoint_identity(name, cuda_device):
    """Engine.jvp against M^-1 g with the reference Jacobian (tangents on A, P, b, c), and
    <(dx, dy), jvp(t)> = <vjp(dx, dy), t>."""
    bt, dev = _batch(name), cuda_device
    st = bt.structure
    eng = Engine(st, dev)
    rng = np.random.default_rng(8)
    tA, tb, tc = rng.standard_normal((bt.B, st.nnzA)), rng.standard_normal((bt.B, st.m)), rng.standard_normal((bt.B, st.n))
    tP = rng.standard_normal(bt.P_vals.shape)
    A, b, c, x, y, s = _at_planted(bt, dev)
    set1 = _lsqr(bt, 1)
    jx, jy, js, _ = eng.jvp(A, b, c, x, y, s, _t(tA, dev), _t(tb, dev), _t(tc, dev), _t(bt.P_vals, dev), _t(tP, dev), set1)
    jx, jy, js = (t.cpu().numpy() for t in (jx, jy, js))
    wx, wy = rng.standard_normal((bt.B, st.n)), rng.standard_normal((bt.B, st.m))
    gA, gP, gb, gc, _ = eng.vjp(A, b, c, x, y, s, _t(wx, dev), _t(wy, dev), _t(bt.P_vals, dev), set1)
    gA, gP, gb, gc = (t.cpu().numpy() for t in (gA, gP, gb, gc))
    rows = np.repeat(np.arange(st.m), np.diff(st.A_indptr))
    worst = worst_id = 0.0
    for i in range(bt.B):
        dAd = np.zeros((st.m, st.n)); dAd[rows, st.A_indices] = tA[i]
        rx, ry, rs = cr.exact_jvp(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i],
                                  dAd, _sym(st, tP[i]), tb[i], tc[i], st.cones, _dense_M(name, i))
        ref = np.concatenate([rx, ry, rs])
        worst = max(worst, np.abs(np.concatenate([jx[i], jy[i], js[i]]) - ref).max() / np.abs(ref).max())
        lhs = wx[i] @ jx[i] + wy[i] @ jy[i]
        rhs = gA[i] @ tA[i] + gP[i] @ tP[i] + gb[i] @ tb[i] + gc[i] @ tc[i]
        worst_id = max(worst_id, abs(lhs - rhs) / max(abs(lhs), abs(rhs), 1e-300))
    print(f"{name}: jvp worst {worst:.1e}, adjoint identity {worst_id:.1e}")
    assert worst <= TOL["jvp"] and worst_id <= TOL["identity"]


@pytest.mark.parametrize("name", NAMES)
def test_central_differences_of_gpu_solves(name, cuda_device):
    """The whole chain without M: for two instances, (<(dx, dy), sol(theta + h t) - sol(theta - h t)>) / 2h from GPU solves
    at eps 1e-12 against <vjp(dx, dy), t> from the GPU adjoint at the planted point; t perturbs A, P, b and c.  h = 1e-7: the
    truncation error is O(h^2) with a large constant where an exponential cone's rho is far from 0 (the same batch through
    the C oracle: 1.5e-3 at h = 1e-5, 1.5e-5 at 1e-6, 1.5e-6 at 1e-7), while the solve error over h stays near 1e-5."""
    bt, dev = _batch(name), cuda_device
    st = bt.structure
    eng = Engine(st, dev)
    rng = np.random.default_rng(10)
    two, h = bt.select([0, 1]), 1e-7
    tA, tP = rng.standard_normal((2, st.nnzA)), rng.standard_normal((2, st.nnzP))
    tb, tc = rng.standard_normal((2, st.m)), rng.standard_normal((2, st.n))
    dx, dy = rng.standard_normal((2, st.n)), rng.standard_normal((2, st.m))
    pm = lambda a, t: np.concatenate([a + h * t, a - h * t])  # noqa: E731   rows: 0+, 1+, 0-, 1-
    sol = eng.solve(_t(pm(two.A_vals, tA), dev), _t(pm(two.b, tb), dev), _t(pm(two.c, tc), dev), _t(pm(two.P_vals, tP), dev),
                    make_settings({"eps_abs": 1e-12, "eps_rel": 1e-12, "max_iters": 400000}))
    assert (sol.status.cpu().numpy() == 1).all(), sol.status
    x, y = sol.x.cpu().numpy(), sol.y.cpu().numpy()
    fd = np.array([(dx[i] @ (x[i] - x[2 + i]) + dy[i] @ (y[i] - y[2 + i])) / (2 * h) for i in range(2)])
    A, b, c, xs, ys, ss = _at_planted(two, dev)
    gA, gP, gb, gc, _ = eng.vjp(A, b, c, xs, ys, ss, _t(dx, dev), _t(dy, dev), _t(two.P_vals, dev), _lsqr(two, 1))
    an = np.array([(gA[i].cpu().numpy() @ tA[i] + gP[i].cpu().numpy() @ tP[i] + gb[i].cpu().numpy() @ tb[i]
                    + gc[i].cpu().numpy() @ tc[i]) for i in range(2)])
    err = np.abs(fd - an) / np.maximum(1.0, np.abs(fd))
    print(f"{name}: central differences {fd}, adjoint {an}, relative error {err.max():.1e}")
    assert err.max() <= TOL["central_differences"]


def _check_scaled_solve(eng, bt, b, c, alpha, dev):
    sol = eng.solve(_t(bt.A_vals, dev), b, c, _t(bt.P_vals, dev), make_settings({**FWD, "eps_abs": 1e-10 * alpha}))
    assert (sol.status.cpu().numpy() == 1).all(), (alpha, sol.status.cpu().numpy())
    errs = [max(_rel(got[i] / alpha, ref[i]) for i in range(bt.B))
            for got, ref in ((sol.x.cpu().numpy(), bt.x_star), (sol.y.cpu().numpy(), bt.y_star), (sol.s.cpu().numpy(), bt.s_star))]
    print(f"alpha {alpha:.0e}: solution / alpha - planted: x {errs[0]:.1e} y {errs[1]:.1e} s {errs[2]:.1e}")
    assert errs[0] <= TOL["x"] and errs[1] <= TOL["y"] and errs[2] <= TOL["s"], (alpha, errs)


@pytest.mark.parametrize("name", ["exp", "mixed", "mixed_scales"])
def test_scale_covariance(name, cuda_device):
    """b, c -> alpha (b, c) with A, P fixed: the solution scales by alpha; at the same O(1) (dx, dy), db and dc are unchanged
    and dA, dP are multiplied by alpha (the cone projection is positively homogeneous, its Jacobian of degree 0).
    mixed_scales: the blocks of one instance span 1e-6 ... 1e3, so every exponential cone is scaled on its own; there only the
    derivative is checked, at alpha times the planted point, because the forward's termination test is relative to the
    largest block and does not reach eps 1e-10 on every such instance."""
    bt, dev = _batch(name), cuda_device
    st = bt.structure
    eng = Engine(st, dev)
    rng = np.random.default_rng(9)
    dx, dy = rng.standard_normal((bt.B, st.n)), rng.standard_normal((bt.B, st.m))
    out = {}
    for alpha in (1.0, 1e-6, 1e6):
        b, c = _t(alpha * bt.b, dev), _t(alpha * bt.c, dev)
        if name != "mixed_scales":
            _check_scaled_solve(eng, bt, b, c, alpha, dev)
        x, y, s = (_t(alpha * a, dev) for a in (bt.x_star, bt.y_star, bt.s_star))
        g = eng.vjp(_t(bt.A_vals, dev), b, c, x, y, s, _t(dx, dev), _t(dy, dev), _t(bt.P_vals, dev), _lsqr(bt, 1))
        out[alpha] = [t.cpu().numpy() for t in (g[0], g[1], g[2], g[3])]
    worst = 0.0
    for alpha in (1e-6, 1e6):
        for k, p in enumerate((1, 1, 0, 0)):   # dA, dP scale with alpha; db, dc do not
            worst = max(worst, np.abs(out[alpha][k] / alpha ** p - out[1.0][k]).max() / np.abs(out[1.0][k]).max())
    print(f"{name}: scale covariance of the gradients, worst {worst:.1e}")
    assert worst <= TOL["scale"]
