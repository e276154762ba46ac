"""Instances whose CSR values do not fit in a CTA's shared memory: the values-off-chip tier of the generic kernels.

* The QP of BASELINE C2 in the form cvxpy's DIFFCP canonicalisation emits (dense eigen factor, 30,002 values): solve, adjoint
  against the oracle, the same QPs through the triangular form on chip, the forward mode against the adjoint.
* The eigen form at n = 200 / m = 400 (120,002 values, HBM-resident for a full grid) and a 400-asset portfolio SOCP in CSR.
* BCONE_VALUES_GLOBAL=1 (the tier forced on structures that fit on chip) against the default: bit-identical outputs.
* Every BASELINE config keeps its on-chip path; the layer (_CvxpyLayer) runs the tier in both directions and in forward AD.
"""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200._lib import EngineUnavailable
from cvxpylayers_b200.engine import Engine, make_settings
from cvxpylayers_b200.interface import B200_ctx, _CvxpyLayer
from cvxpylayers_b200.structure import ConeSpec, Structure
from oracle import np_ref
from oracle import oracle as orc
from tests.util import rel_err

pytestmark = pytest.mark.gpu

TIGHT = {"lsqr_precond": 1, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12}
NEW_FWD, NEW_BWD = set(Engine.FWD_PATHS[4:]), Engine.BWD_PATHS[3]
SAMPLE = 32   # instances checked against the oracle (it runs on the host cores)


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _np(a):
    return a.cpu().numpy()


def _qp_cotangents(B, n, m, rng):
    """Cotangents on x and on the duals of the original rows only (zero on the epigraph variable and the SOC rows)."""
    dx = np.concatenate([rng.standard_normal((B, n)), np.zeros((B, 1))], axis=1)
    dy = np.concatenate([rng.standard_normal((B, m)), np.zeros((B, n + 2))], axis=1)
    return dx, dy


def _check_planted_x(x, x_star, n):
    """x of a solve at eps 1e-8 against the planted optimum, to 1e-5 relative: the QP's variables against their largest entry,
    the epigraph variable t* = 1/2 x'Px (O(50)) against itself.  Returns the two errors."""
    ex = np.abs(x[:, :n] - x_star[:, :n]).max() / max(1.0, np.abs(x_star[:, :n]).max())
    et = rel_err(x[:, n], x_star[:, n])
    assert ex < 1e-5 and et < 1e-5, (ex, et)
    return ex, et


def _adjoint_identity(eng, bt, x, y, s, dev, args, seed=9):
    """max over instances of |<w, J t> - <J'w, t>| / (|w| |J t|) for random tangents t and cotangents w."""
    st, B = bt.structure, bt.B
    rng = np.random.default_rng(seed)
    tA, tb, tc = rng.standard_normal((B, st.nnzA)), rng.standard_normal((B, st.m)), rng.standard_normal((B, st.n))
    w = (rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m)))
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    dx, dy, _, its = eng.jvp(A, b, c, x, y, s, _t(tA, dev), _t(tb, dev), _t(tc, dev), settings=make_settings(args))
    dx, dy = _np(dx), _np(dy)
    assert (_np(its) > 0).all()
    lhs = (w[0] * dx).sum(1) + (w[1] * dy).sum(1)
    scale = np.sqrt((w[0] ** 2).sum(1) + (w[1] ** 2).sum(1)) * np.sqrt((dx ** 2).sum(1) + (dy ** 2).sum(1))
    gA, _, gb, gc, _ = eng.vjp(A, b, c, x, y, s, _t(w[0], dev), _t(w[1], dev), settings=make_settings(args))
    rhs = (_np(gA) * tA).sum(1) + (_np(gb) * tb).sum(1) + (_np(gc) * tc).sum(1)
    return (np.abs(lhs - rhs) / scale).max()


def _check_planted_eigen_form(bq, dev, B_oracle=SAMPLE):
    """Solve + adjoint + forward mode of the eigen (cvxpy) form of the QPs ``bq`` on the values-off-chip tier."""
    n, m, B = bq.structure.n, bq.structure.m, bq.B
    bt = pr.qp_as_socp(bq, factor="eigen")
    st = bt.structure
    eng = Engine(st, dev)
    paths = eng.path_info()
    assert paths["fwd"] in NEW_FWD and paths["bwd"] == NEW_BWD, paths
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    sol = eng.solve(A, b, c, settings=make_settings({"eps": 1e-8, "max_iters": 200000}))
    assert int((sol.status == 1).sum()) == B, (_np(sol.status), _np(sol.iters))
    _check_planted_x(_np(sol.x), bt.x_star, n)
    # adjoint at the planted optimum against the oracle's, cotangents on (x, original duals)
    x, y, s = _t(bt.x_star, dev), _t(bt.y_star, dev), _t(bt.s_star, dev)
    dx, dy = _qp_cotangents(B, n, m, np.random.default_rng(3))
    args = {**TIGHT, "lsqr_iter_lim": 40 * (st.n + st.m + 1)}
    gA, _, gb, gc, its = eng.vjp(A, b, c, x, y, s, _t(dx, dev), _t(dy, dev), settings=make_settings(args))
    assert (_np(its) > 0).all()
    k = slice(0, B_oracle)
    rA, _, rb, rc, _ = orc.vjp_batch(st, bt.A_vals[k], bt.b[k], bt.c[k], bt.x_star[k], bt.y_star[k], bt.s_star[k], dx[k], dy[k], None,
                                     lsqr_precond=1, lsqr_iter_lim=args["lsqr_iter_lim"], lsqr_atol=1e-12, lsqr_btol=1e-12)
    errs = (rel_err(_np(gA)[k], rA), rel_err(_np(gb)[k], rb), rel_err(_np(gc)[k], rc))
    assert max(errs) < 1e-4, errs
    assert _adjoint_identity(eng, bt, x, y, s, dev, args) < 1e-6
    return bt, eng, (_np(gb), _np(gc), dx, dy, args)


# ----------------------------------------------------------------------------- the C2 QP as cvxpy's DIFFCP path emits it
def test_c2_diffcp_form_with_cvxpys_factor(cuda_device):
    dev = cuda_device
    bq = pr.dense_qp(1024, 100, 200, 50, seed=0)
    bt, eng, (gb, gc, dx, dy, args) = _check_planted_eigen_form(bq, dev)
    assert (bt.structure.nnzA, bt.structure.n, bt.structure.m) == (30002, 101, 302)
    assert eng.path_info()["fwd"] == Engine.FWD_PATHS[4]   # the 5,151-double factor and the vectors still fit on chip
    # the same QPs in the triangular form (values on chip): the same function of (b, c), so the same dc / db
    tri = pr.qp_as_socp(bq)
    e2 = Engine(tri.structure, dev)
    assert e2.path_info()["fwd"] not in NEW_FWD and e2.path_info()["bwd"] != NEW_BWD
    # the forward reaches the same accuracy as the triangular form on chip
    fs = make_settings({"eps": 1e-8, "max_iters": 200000})
    s_eig = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), settings=fs)
    s_tri = e2.solve(_t(tri.A_vals, dev), _t(tri.b, dev), _t(tri.c, dev), settings=fs)
    assert int((s_tri.status == 1).sum()) == bq.B
    e_eig, e_tri = _check_planted_x(_np(s_eig.x), bt.x_star, 100), _check_planted_x(_np(s_tri.x), tri.x_star, 100)
    assert max(e_eig) < 3 * max(e_tri) + 1e-7, (e_eig, e_tri)
    _, _, gb2, gc2, _ = e2.vjp(_t(tri.A_vals, dev), _t(tri.b, dev), _t(tri.c, dev), _t(tri.x_star, dev), _t(tri.y_star, dev),
                               _t(tri.s_star, dev), _t(dx, dev), _t(dy, dev), settings=make_settings(args))
    n, m = 100, 200
    assert rel_err(gc[:, :n], _np(gc2)[:, :n]) < 1e-4 and rel_err(gb[:, :m], _np(gb2)[:, :m]) < 1e-4


def test_eigen_form_n200_hbm_resident_values(cuda_device):
    bq = pr.dense_qp(64, 200, 400, 100, seed=1)
    bt, eng, _ = _check_planted_eigen_form(bq, cuda_device, B_oracle=16)
    assert bt.structure.nnzA == 120002


def test_portfolio_socp_400_assets_csr(cuda_device):
    dev, B = cuda_device, 256
    bt = pr.socp_portfolio(B, n_assets=400, n_soc=5, k=20, seed=2)
    st = bt.structure
    assert st.nnzA == 40800 and st.nnzA < st.m * st.n   # CSR, not dense
    eng = Engine(st, dev)
    paths = eng.path_info()
    assert paths["fwd"] in NEW_FWD and paths["bwd"] == NEW_BWD, paths
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    eps = 1e-8
    sol = eng.solve(A, b, c, settings=make_settings({"eps": eps, "max_iters": 200000}))
    assert int((sol.status == 1).sum()) == B, (_np(sol.status), _np(sol.iters))
    x, y, s = _np(sol.x), _np(sol.y), _np(sol.s)
    for i in range(0, B, 8):   # the solver's own certificate, recomputed on the host
        r = np_ref.kkt_residuals(bt.A_dense(i), None, bt.b[i], bt.c[i], x[i], y[i], s[i])
        assert np_ref.is_converged(r, eps, eps, 1.001), (i, r)
    k = slice(0, SAMPLE)
    xo, yo, so, sto, _ = orc.solve_batch(st, bt.A_vals[k], bt.b[k], bt.c[k], None, eps=1e-10, max_iters=400000)
    assert (sto == 1).all()
    assert np.abs(x[k] - xo).max() < 1e-5 * max(1.0, np.abs(xo).max())
    rng = np.random.default_rng(4)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    lim = 40 * (st.n + st.m + 1)
    xs, ys, ss = np.array(x), np.array(y), np.array(s)
    xs[k], ys[k], ss[k] = xo, yo, so   # the sample is differentiated at the oracle's solution on both sides
    gA, _, gb, gc, _ = eng.vjp(A, b, c, _t(xs, dev), _t(ys, dev), _t(ss, dev), _t(dx, dev), _t(dy, dev),
                               settings=make_settings({"lsqr_precond": 1, "lsqr_iter_lim": lim}))
    rA, _, rb, rc, _ = orc.vjp_batch(st, bt.A_vals[k], bt.b[k], bt.c[k], xo, yo, so, dx[k], dy[k], None, lsqr_precond=1, lsqr_iter_lim=lim)
    errs = (rel_err(_np(gA)[k], rA), rel_err(_np(gb)[k], rb), rel_err(_np(gc)[k], rc))
    assert max(errs) < 1e-4, errs
    assert np.isfinite(_np(gA)).all()


# ----------------------------------------------------------------------------- the forced tier is the same arithmetic
def _run_all(bt, dev, fwd_args, at=None):
    """solve, then vjp and jvp at ``at`` (a Solution; default: this solve's) -> engine, forward outputs, derivative outputs."""
    st = bt.structure
    eng = Engine(st, dev)
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    sol = eng.solve(A, b, c, P, make_settings(fwd_args))
    at = at or sol
    rng = np.random.default_rng(11)
    dx, dy = _t(rng.standard_normal((bt.B, st.n)), dev), _t(rng.standard_normal((bt.B, st.m)), dev)
    args = make_settings({"lsqr_precond": 1, "lsqr_iter_lim": 20 * (st.n + st.m + 1)})
    g = eng.vjp(A, b, c, at.x, at.y, at.s, dx, dy, P, args)
    tA, tb, tc = (_t(rng.standard_normal(sh), dev) for sh in ((bt.B, st.nnzA), (bt.B, st.m), (bt.B, st.n)))
    tP = _t(rng.standard_normal((bt.B, st.nnzP)), dev) if st.nnzP else None
    j = eng.jvp(A, b, c, at.x, at.y, at.s, tA, tb, tc, P, tP, args)
    torch.cuda.synchronize()
    return eng, sol, [v.cpu() for v in (sol.x, sol.y, sol.s, sol.status, sol.iters)], [v.cpu() for v in (*g, *j) if v is not None]


@pytest.mark.parametrize("name,B,fwd_args", [("C3", 256, {"eps": 1e-6}), ("C5", 64, {"eps": 1e-6}), ("EXP", 64, {"eps": 1e-6}),
                                             ("C4", 4, {"eps": 1e-4, "max_iters": 100000})])
def test_forced_values_off_chip_matches_the_default(name, B, fwd_args, cuda_device, monkeypatch):
    """The same arithmetic on values read from another memory.  The adjoint and the forward mode at the same point are
    bit-identical.  So is the forward on C4 (conjugate gradients).  The direct forward of C3 / C5 / EXP forms K = A'RA with
    floating-point atomics (fwd.cu, factor_and_g), whose order -- and so the last bits of K -- varies from one launch to the
    next on either path; the solves then differ far below their tolerance."""
    bt = pr.CONFIGS[name](B=B)
    monkeypatch.delenv("BCONE_VALUES_GLOBAL", raising=False)
    e0, sol0, f0, d0 = _run_all(bt, cuda_device, fwd_args)
    monkeypatch.setenv("BCONE_VALUES_GLOBAL", "1")
    e1, _, f1, d1 = _run_all(bt, cuda_device, fwd_args, at=sol0)
    p0, p1 = e0.path_info(), e1.path_info()
    assert p0["fwd"] not in NEW_FWD and p0["bwd"] != NEW_BWD, p0
    assert p1["fwd"] in NEW_FWD and p1["bwd"] == NEW_BWD, p1
    k0, k1 = e0.kernel_info(), e1.kernel_info()
    assert k0["fwd_threads"] == k1["fwd_threads"] and k0["bwd_threads"] == k1["bwd_threads"], (k0, k1)
    assert int((f0[3] == 1).sum()) == B and torch.equal(f0[3], f1[3])
    for i, (a, b_) in enumerate(zip(d0, d1)):
        assert torch.equal(a, b_), (name, i, (a - b_).abs().max() if a.is_floating_point() else None)
    if name == "C4":
        assert all(torch.equal(a, b_) for a, b_ in zip(f0, f1))
    for a, b_ in zip(f0[:3], f1[:3]):
        assert (a - b_).abs().max() <= 1e-8 * max(1.0, a.abs().max()), (name, (a - b_).abs().max())


def test_psd_scratch_that_does_not_fit_is_refused_loudly(cuda_device):
    """With values and vectors off chip, the on-chip PSD scratch is what is left: a 70 x 70 PSD block does not fit."""
    import re

    k, n = 70, 10
    m = k * (k + 1) // 2
    st = Structure(n, m, np.arange(m + 1, dtype=np.int32), (np.arange(m) % n).astype(np.int32), ConeSpec(s=[k]))
    with pytest.raises(EngineUnavailable) as ei:
        Engine(st, cuda_device)
    msg = str(ei.value)
    hit = re.search(r"the largest PSD order that fits is (\d+)", msg)
    assert "PSD scratch" in msg and hit and 0 < int(hit.group(1)) < k, msg


def test_every_baseline_config_keeps_its_on_chip_path(cuda_device, monkeypatch):
    monkeypatch.delenv("BCONE_VALUES_GLOBAL", raising=False)
    for name, make in pr.CONFIGS.items():
        p = Engine(make(B=1).structure, cuda_device).path_info()
        assert p["fwd"] not in NEW_FWD and p["bwd"] != NEW_BWD, (name, p)


# ----------------------------------------------------------------------------- through the layer
def _layer(bt, dev, args):
    bd = pr.to_boundary(bt)
    ctx = B200_ctx(None, (bd.con_indices, bd.con_ptr, bd.shape), bd.dims, options=args, device=dev)
    cl = type("CL", (), {"solver_ctx": ctx})()
    return bd, ctx, (lambda q, A: _CvxpyLayer.apply(None, q, A, cl, {}, True, None)[:2])


def test_layer_forward_and_backward_on_the_c2_diffcp_form(cuda_device):
    dev = cuda_device
    bt = pr.qp_as_socp(pr.dense_qp(1024, 100, 200, 50, seed=0), factor="eigen")
    st = bt.structure
    args = {"eps": 1e-8, "max_iters": 200000, "lsqr_precond": 1}
    bd, ctx, f = _layer(bt, dev, args)
    q = _t(bd.q_eval, dev).requires_grad_(True)
    A = _t(bd.A_eval, dev).requires_grad_(True)
    primal, dual = f(q, A)
    assert ctx.engine(dev).path_info()["fwd"] in NEW_FWD
    _check_planted_x(_np(primal.detach()), bt.x_star, st.n - 1)
    rng = np.random.default_rng(0)
    dx, dy = rng.standard_normal(primal.shape), rng.standard_normal(dual.shape)
    ((primal * _t(dx, dev)).sum() + (dual * _t(dy, dev)).sum()).backward()
    k = slice(0, SAMPLE)
    # the layer differentiates at its own solution: the sample's (x, y, s) again (per-instance arithmetic, same for any batch)
    sol = ctx.engine(dev).solve(_t(bt.A_vals[k], dev), _t(bt.b[k], dev), _t(bt.c[k], dev), settings=make_settings(args))
    x, y, s = _np(sol.x), _np(sol.y), _np(sol.s)
    gA, _, gb, gc, _ = orc.vjp_batch(st, bt.A_vals[k], bt.b[k], bt.c[k], x, y, s, dx[k], dy[k], None, lsqr_precond=1)
    dq, dAe = _np(q.grad), _np(A.grad)
    assert np.abs(dq[-1]).max() == 0.0
    assert rel_err(dq[:-1, k].T, gc) < 1e-4
    assert rel_err(dAe[st.nnzA:, k].T, gb[:, np.asarray(ctx.b_idx)]) < 1e-4
    assert rel_err(-dAe[ctx.gather][:, k].T, gA) < 1e-4


def test_layer_forward_ad_equals_reverse_jacobian_on_the_eigen_form(cuda_device):
    dev = cuda_device
    bt = pr.qp_as_socp(pr.dense_qp(2, 100, 200, 50, seed=5), factor="eigen")
    bd, ctx, f = _layer(bt, dev, {"eps": 1e-11, "max_iters": 200000, **TIGHT})
    q, A = _t(bd.q_eval, dev), _t(bd.A_eval, dev)
    assert ctx.engine(dev).path_info()["bwd"] == NEW_BWD
    g = torch.Generator().manual_seed(1)
    tq, tA = (torch.randn(v.shape, dtype=torch.float64, generator=g).to(dev) for v in (q, A))
    with fwAD.dual_level():
        outs = f(fwAD.make_dual(q, tq), fwAD.make_dual(A, tA))
        got = [fwAD.unpack_dual(o).tangent for o in outs]
    J = torch.autograd.functional.jacobian(f, (q, A))
    for o, Jo in zip(got, J):
        ref = sum((Jo[jj].reshape(-1, x.numel()) @ t.reshape(-1)).reshape(o.shape) for jj, (x, t) in enumerate(((q, tq), (A, tA))))
        err = (o - ref).abs().max().item()
        assert err <= 1e-6 * max(1.0, ref.abs().max().item()), err
