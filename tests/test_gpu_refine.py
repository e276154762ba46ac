"""Solution refinement on the GPU (csrc/refine.cu): against the NumPy restatement (tests/refine_ref.py) and the planted optimum,
starting from eps-1e-3 forward solves, on the cone_planted structures, a dense QP and an LP; more than one wave of instances on
a dense and a CSR pattern; the 4-CTA/SM and 128-register builds, values off chip and a dense QP of C2's shape; statuses, and
rejected and not-attempted rows (the infeasible and unbounded batches of tests/infeas_planted.py) keep their bits; the shared
entry point; and through the layer with ``solver_args={"refine": ...}``: the reverse-mode gradient at the refined point against
the exact adjoint at the planted optimum, forward AD, the warm start and the option's refusals."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, Solution, make_settings
from tests import cone_planted as cp
from tests import cone_ref as cr
from tests import infeas_planted as ip
from tests import refine_ref as rref
from tests import tiled_shapes as ts
from tests.test_refine_host import EXP_BOUND

pytestmark = pytest.mark.gpu
DEV = "cuda"
LOOSE = {"eps": 1e-3}


def _t(a):
    return None if a is None else torch.tensor(a, dtype=torch.float64, device=DEV)


def _solve(bt, args=LOOSE, eng=None):
    eng = eng or Engine(bt.structure, DEV)
    A, P, b, c = _t(bt.A_vals), _t(bt.P_vals), _t(bt.b), _t(bt.c)
    sol = eng.solve(A, b, c, P, make_settings(args))
    return eng, A, P, b, c, sol


def _copy(sol):
    return Solution(*(t.clone() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)))


def _np(sol):
    return tuple(t.cpu().numpy() for t in (sol.x, sol.y, sol.s, sol.status))


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _agree(got, ref):
    """max over x, y, s of the error relative to each array's max-abs"""
    return max(np.abs(g - r).max() / max(np.abs(r).max(), 1e-300) for g, r in zip(got, ref))


BATCHES = {
    **{k: (lambda k=k: cp.make(k, 2)) for k in ("soc_sizes", "psd_warm", "psd_serial", "exp", "mixed")},
    "dense_qp": lambda: pr.dense_qp(2, 20, 30, 5, seed=11),
    "lp_vertex": lambda: ts.planted(ts.Case(12, 30, 4, 8, False, 1), 2, seed=3),
}


@pytest.mark.parametrize("pre", [0, 1])
@pytest.mark.parametrize("key", list(BATCHES))
def test_kernel_matches_restatement_and_planted_optimum(key, pre):
    bt = BATCHES[key]()
    eng, A, P, b, c, sol = _solve(bt)
    x0, y0, s0, status = _np(sol)
    flags = eng.refine(A, b, c, sol, P, make_settings({"lsqr_precond": pre}), steps=3).cpu().numpy()
    fr, X, Y, S = rref.refine_batch(bt, x0, y0, s0, status, steps=3, precond=pre)
    x, y, s, st = _np(sol)
    assert (st == status).all()
    assert (flags == fr).all() and (flags == 1).all(), (key, flags, fr)
    # (exp without the equilibration: LSQR stops at its iteration limit on every step, where the two LSQRs' rounding has
    #  drifted apart -- 6e-5 measured)
    tol = 1e-3 if (key == "exp" and pre == 0) else 1e-9
    assert _agree((x, y, s), (X, Y, S)) <= tol, (key, pre, _agree((x, y, s), (X, Y, S)))
    if pre == 1 or key not in EXP_BOUND:
        err = max(_rel(x, bt.x_star), _rel(y, bt.y_star))
        assert err <= EXP_BOUND.get(key, 1e-9) and err < max(_rel(x0, bt.x_star), _rel(y0, bt.y_star)), (key, err)


@pytest.mark.parametrize("key", ["soc_sizes", "psd_warm"])   # (dense A, CSR A)
def test_more_than_one_wave(monkeypatch, key):
    """600 instances, more than twice what the 128-register build keeps resident, so every CTA refines several instances in
    turn; every 7th row is not attempted (status FAILED) between refined ones.  From the planted optimum perturbed by 1e-4 (a
    start that does not depend on a forward solve), three steps reach 1e-9 on the SOC structure; on the PSD one the kernel
    stalls at up to 5e-9 (one instance of 600, the same when refined alone) where the NumPy twin reaches 2.5e-12 from the same
    inputs -- DESIGN.md section 9 -- so its bound is 1e-7.  The not-attempted rows keep their bits."""
    monkeypatch.setenv("BCONE_SMALL_CTA", "0")
    bt = cp.make(key, 600)
    eng = Engine(bt.structure, DEV)
    rng = np.random.default_rng(3)
    x, y, s = (_t(a + 1e-4 * rng.standard_normal(a.shape)) for a in (bt.x_star, bt.y_star, bt.s_star))
    status = torch.ones(bt.B, dtype=torch.int32, device=DEV)
    skip = np.arange(bt.B) % 7 == 3
    status[torch.as_tensor(skip, device=DEV)] = -4
    sol = Solution(x, y, s, status, torch.zeros_like(status), torch.zeros((bt.B, 3), dtype=torch.float64, device=DEV))
    before = _copy(sol)
    A, P, b, c = _t(bt.A_vals), _t(bt.P_vals), _t(bt.b), _t(bt.c)
    flags = eng.refine(A, b, c, sol, P, make_settings({"lsqr_precond": 1}), steps=3).cpu().numpy()
    info = eng.refine_info()
    assert info["last_small"] == 0 and bt.B > 2 * info["num_sms"] * info["ctas_per_sm"], info
    assert (flags[skip] == -1).all() and (flags[~skip] == 1).all(), np.unique(flags, return_counts=True)
    for u, v in ((sol.x, before.x), (sol.y, before.y), (sol.s, before.s), (sol.resid, before.resid)):
        assert torch.equal(u[torch.as_tensor(skip, device=DEV)], v[torch.as_tensor(skip, device=DEV)])
    xr, yr, _, _ = _np(sol)
    bound = 1e-7 if key == "psd_warm" else 1e-9
    assert _rel(xr[~skip], bt.x_star[~skip]) <= bound and _rel(yr[~skip], bt.y_star[~skip]) <= bound


def test_many_blocks_improves_or_keeps_its_bits():
    """600 exponential cones and more SOC / PSD blocks than warps: every row is accepted with residuals that do not grow, or
    keeps its bits."""
    bt = cp.make("many_blocks", 4)
    eng, A, P, b, c, sol = _solve(bt)
    before = _copy(sol)
    flags = eng.refine(A, b, c, sol, P, make_settings({"lsqr_precond": 1})).cpu().numpy()
    assert set(flags.tolist()) <= {0, 1}
    for i in np.flatnonzero(flags == 0):
        assert torch.equal(sol.x[i], before.x[i]) and torch.equal(sol.y[i], before.y[i]) and torch.equal(sol.s[i], before.s[i])
    x0, y0, s0, _ = _np(before)
    x, y, s, _ = _np(sol)
    for i in np.flatnonzero(flags == 1):
        A_, P_ = bt.A_dense(i), bt.P_dense(i)
        r0 = rref.metrics(A_, P_, bt.b[i], bt.c[i], x0[i], y0[i], s0[i])
        r1 = rref.metrics(A_, P_, bt.b[i], bt.c[i], x[i], y[i], s[i])
        assert np.all(r1 <= r0 * (1 + 1e-12)), (i, r0, r1)


TIERS = {   # name -> (structure, environment, what bcone_refine_info must report)
    "small_cta": ("exp", {"BCONE_SMALL_CTA": "2"}, {"last_small": 1}),
    "big_cta": ("exp", {"BCONE_SMALL_CTA": "0"}, {"last_small": 0, "small_ctas_per_sm": 0}),
    "values_off_chip": ("mixed", {"BCONE_VALUES_GLOBAL": "1"}, {"vals_global": 1, "last_small": 0}),
    "c2_shape": ("c2_shape", {}, {"vals_global": 0}),
}


@pytest.mark.parametrize("tier", list(TIERS))
def test_tiers(monkeypatch, tier):
    """The 4-CTA/SM build (forced), the 128-register build, values off chip, and C2's shape (the forward mode's generic
    geometry): the same input refined by an engine created under each setting matches the restatement, and the refinement plan
    reports the build that ran."""
    key, env, expect = TIERS[tier]
    bt = ts.planted(ts.Case(100, 200, 50, 40, True, 2), 4, 11) if key == "c2_shape" else cp.make(key, 2)
    _, A, P, b, c, sol = _solve(bt)
    x0, y0, s0, status = _np(sol)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = Engine(bt.structure, DEV)
    flags = eng.refine(A, b, c, sol, P, make_settings({"lsqr_precond": 1})).cpu().numpy()
    info = eng.refine_info()
    assert info["threads"] > 0 and all(info[k] == v for k, v in expect.items()), (tier, info)
    fr, X, Y, S = rref.refine_batch(bt, x0, y0, s0, status, precond=1)
    assert (flags == fr).all() and (flags == 1).all(), (flags, fr)
    x, y, s, _ = _np(sol)
    assert _agree((x, y, s), (X, Y, S)) <= 1e-9
    assert max(_rel(x, bt.x_star), _rel(y, bt.y_star)) <= EXP_BOUND.get(key, 1e-9)


@pytest.mark.parametrize("key", ["tiled", "mixed"])
def test_status_rejected_and_not_attempted_rows_keep_their_bits(key):
    """Infeasible and unbounded instances are not attempted and keep every bit, as does a row with a non-finite input and a
    rejected row; statuses are never changed; the controls are refined (the near-degenerate ``control_near`` may be
    rejected)."""
    if key == "tiled":
        kinds = ip.MIX
        bt = ip.mixed(ts.planted(ts.CASES["kr4"], len(kinds), 5), kinds, seed=6)
    else:
        bt = ip.mixed(cp.make("mixed", B=len(ip.MIX)), ip.MIX, seed=1)
    eng, A, P, b, c, sol = _solve(bt, {"eps": 1e-4, "max_iters": 20000})
    sol.x[0, 0] = float("nan")   # (instance 0: a non-finite input)
    before = _copy(sol)
    flags = eng.refine(A, b, c, sol, P, make_settings({"lsqr_precond": 1})).cpu().numpy()
    status = before.status.cpu().numpy()
    assert torch.equal(sol.status, before.status)
    assert flags[0] == -1
    assert (flags[(status != 1) & (status != 2)] == -1).all()
    for i in np.flatnonzero(flags <= 0):
        for u, v in ((sol.x, before.x), (sol.y, before.y), (sol.s, before.s), (sol.resid, before.resid)):
            assert torch.equal(u[i].isnan(), v[i].isnan()) and torch.equal(torch.nan_to_num(u[i]), torch.nan_to_num(v[i])), i
    ok = [i for i, k in enumerate(ip.MIX) if k == "control" and i != 0]
    assert (flags[ok] == 1).all() and (flags[[i for i in ip.controls(bt) if i != 0]] >= 0).all(), flags


def test_rejected_row_keeps_its_bits():
    bt = pr.dense_qp(16, 20, 30, 5, seed=11)
    eng, A, P, b, c, sol = _solve(bt, {"eps": 1e-3, "max_iters": 20, "acceleration_lookback": 0})
    sol.status.fill_(1)
    x0, y0, s0, status = _np(sol)
    fr, *_ = rref.refine_batch(bt, x0, y0, s0, status, steps=1, precond=0, iter_lim=2)
    before = _copy(sol)
    flags = eng.refine(A, b, c, sol, P, make_settings({"lsqr_iter_lim": 2}), steps=1).cpu().numpy()
    assert (flags == fr).all() and (flags == 0).any() and (flags == 1).any(), (flags, fr)
    for i in np.flatnonzero(flags == 0):
        assert torch.equal(sol.x[i], before.x[i]) and torch.equal(sol.y[i], before.y[i]) and torch.equal(sol.s[i], before.s[i])


@pytest.mark.parametrize("key", ["tiled", "mixed"])
def test_shared_entry_point(key):
    if key == "tiled":
        bt = ts.planted(ts.CASES["nch1_live_eq_n"], 8, seed=9, shared=True)
    else:
        bt = ip.shared(cp.make("mixed", B=len(ip.SHARED_MIX)), seed=4)
    eng, A, P, b, c, sol = _solve(bt, {"eps": 1e-4, "max_iters": 20000})
    one = _copy(sol)
    f_rep = eng.refine(A, b, c, sol, P, make_settings({"lsqr_precond": 1}))
    f_sh = eng.refine(A[0].clone(), b, c, one, None if P is None else P[0].clone(), make_settings({"lsqr_precond": 1}))
    assert torch.equal(f_rep, f_sh) and (f_rep == 1).any()
    for u, v in zip(_np(one)[:3] + (one.resid.cpu().numpy(),), _np(sol)[:3] + (sol.resid.cpu().numpy(),)):   # (the same bits, NaN included)
        assert np.array_equal(u, v, equal_nan=True)


def test_steps_outside_1_to_10_are_refused():
    bt = pr.dense_qp(2, 6, 9, 2, seed=1)
    eng, A, P, b, c, sol = _solve(bt)
    for bad in (0, 11, 2.0, True):
        with pytest.raises(ValueError, match="steps"):
            eng.refine(A, b, c, sol, P, steps=bad)


def _apply_fn(bt, opts, dev=DEV):
    from cvxpylayers_b200.interface import B200_ctx, _CvxpyLayer

    st = bt.structure
    bd = pr.to_boundary(bt)
    P_struct = (st.P_indices, st.P_indptr, (st.n, st.n)) if st.nnzP else None
    ctx = B200_ctx(P_struct, (bd.con_indices, bd.con_ptr, bd.shape), bd.dims, options=opts, device=dev)
    cl = type("CL", (), {"solver_ctx": ctx})()
    return bd, ctx, (lambda P, q, A, args=None: _CvxpyLayer.apply(P, q, A, cl, args or {}, True, None)[:2])


def _layer(monkeypatch, bt, opts=None):
    from cvxpylayers_b200 import interface as itf
    from tests.util import fake_param_prob, install_fake_cvxpylayers

    fake = install_fake_cvxpylayers(monkeypatch)
    problem, params = fake_param_prob(bt)
    itf.register(fuse=False)
    layer = fake.tl.CvxpyLayer(problem, [], [], solver="B200", solver_args=opts or {})
    return layer, [torch.tensor(p, device=DEV, requires_grad=True) for p in params]


@pytest.mark.parametrize("bad, match", [({"polish": True, "refine": True}, "exclude"), ({"refine": 2.5}, "refine"),
                                        ({"refine": 0}, "refine"), ({"refine": 11}, "refine"), ({"refine": "3"}, "refine")])
def test_layer_refusals_come_before_staging_any_chunk(monkeypatch, bad, match):
    """Pageable host inputs over several pipeline chunks take the staged path; a refused option raises before a chunk is
    staged, and the engine's stager still serves the next call."""
    from cvxpylayers_b200 import interface as itf

    monkeypatch.setattr(itf, "PIPE_CHUNK", 4)
    bt = pr.qp_as_socp(pr.dense_qp(24, 6, 9, 2, seed=1))   # 6 chunks: more than the stager's ring of 3 slots
    bd, ctx, f = _apply_fn(bt, {"eps": 1e-6})
    P, q, A = (None if a is None else torch.tensor(a) for a in (bd.P_eval, bd.q_eval, bd.A_eval))   # pageable CPU tensors
    assert itf._stage_ok(24, A, q, P)
    with pytest.raises(ValueError, match=match):
        f(P, q, A, bad)
    primal, _ = f(P, q, A, {"refine": 2, "eps": 1e-3})
    assert primal.shape == (24, bt.structure.n) and torch.isfinite(primal).all()
    assert _rel(primal.numpy(), bt.x_star) <= 1e-9
    eng, = ctx._engines.values()
    assert getattr(eng, "_stager", None) is not None   # (the staged path ran)


def test_layer_refined_solution_gradient_forward_ad_and_warm_start(monkeypatch):
    bt = pr.qp_as_socp(pr.dense_qp(3, 10, 15, 3, seed=4))
    layer, th = _layer(monkeypatch, bt, {"refine": True, "eps": 1e-3, "warm_start": True})
    primal, dual = layer(*th)
    assert _rel(primal.detach().cpu().numpy(), bt.x_star) < 1e-9 and _rel(dual.detach().cpu().numpy(), bt.y_star) < 1e-9
    ctx = layer.ctx.solver_ctx
    (xw, yw, _), = ctx._last_solution.values()
    assert torch.equal(xw, primal.detach()) and torch.equal(yw, dual.detach())   # the warm start keeps the refined point
    with torch.no_grad():
        p_un, _ = layer(*th, solver_args={"refine": False, "warm_start": False})
    assert _rel(p_un.cpu().numpy(), bt.x_star) > 1e-6

    # reverse mode through the layer against the exact adjoint at the planted optimum, emitted to the boundary layout
    rng = np.random.default_rng(0)
    dx, dy = rng.standard_normal(bt.x_star.shape), rng.standard_normal(bt.y_star.shape)
    exact = [cr.exact_adjoint(bt.A_dense(i), bt.P_dense(i) if bt.P_vals is not None else None, bt.b[i], bt.c[i], bt.x_star[i],
                              bt.y_star[i], bt.s_star[i], dx[i], dy[i], bt.structure.cones) for i in range(bt.B)]
    bd, lctx, f = _apply_fn(bt, {"eps": 1e-3, "lsqr_atol": 1e-14, "lsqr_btol": 1e-14, "lsqr_conlim": 1e14})
    eng = lctx.engine(torch.device(DEV, torch.cuda.current_device()))
    eA, eq, _ = eng.emit(_t(np.stack([e[0].ravel() for e in exact])), None, _t(np.stack([e[2] for e in exact])),
                         _t(np.stack([e[3] for e in exact])))
    eA, eq = eA.cpu().numpy(), eq.cpu().numpy()
    for pre in (1, 2):
        errs = []
        for ref in (True, False):
            P, q, A = (None if a is None else _t(a).requires_grad_(True) for a in (bd.P_eval, bd.q_eval, bd.A_eval))
            x, y = f(P, q, A, {"refine": ref, "lsqr_precond": pre})
            ((x * _t(dx)).sum() + (y * _t(dy)).sum()).backward()
            errs.append(max(_rel(A.grad.cpu().numpy(), eA), _rel(q.grad.cpu().numpy(), eq)))
        assert errs[0] < errs[1], (pre, errs)

    # forward AD through the refined layer
    import torch.autograd.forward_ad as fwAD

    bd, _, f = _apply_fn(bt, {"refine": 3, "eps": 1e-3})
    Pe, qe, Ae = (None if a is None else _t(a) for a in (bd.P_eval, bd.q_eval, bd.A_eval))
    with fwAD.dual_level():
        out = f(None if Pe is None else fwAD.make_dual(Pe, torch.randn_like(Pe)), fwAD.make_dual(qe, torch.randn_like(qe)),
                fwAD.make_dual(Ae, torch.randn_like(Ae)))
        x_fw, tan = fwAD.unpack_dual(out[0])
    assert _rel(x_fw.cpu().numpy(), bt.x_star) < 1e-9
    assert tan is not None and torch.isfinite(tan).all()


@pytest.mark.parametrize("shared", [False, True])
def test_fused_layer_refines_replicated_and_shared_matrices(shared):
    from cvxpylayers_b200.interface import _CvxpyLayerFused, get_solver_ctx
    from tests.util import fake_param_prob

    bt = ts.planted(ts.CASES["nch1_live_eq_n"], 4, seed=9, shared=True)
    problem, params = fake_param_prob(bt)
    ctx = get_solver_ctx("B200", problem["param_prob"], problem["dims"], {}, {"eps": 1e-3})
    ctx.device = torch.device(DEV, torch.cuda.current_device())
    cl = type("CL", (), {"solver_ctx": ctx})()
    p_stack = torch.as_tensor(np.concatenate([p.T for p in params] + [np.ones((1, bt.B))]), dtype=torch.float64, device=DEV)
    args = {"shared_matrices": shared, "lsqr_precond": 1}   # (without the equilibration three steps reach 1e-2 here)
    with pytest.raises(ValueError, match="exclude"):
        _CvxpyLayerFused.apply(p_stack, cl, {**args, "polish": True, "refine": 3}, True, None)
    primal, dual, _, _ = _CvxpyLayerFused.apply(p_stack, cl, {**args, "refine": 3}, True, None)
    assert _rel(primal.cpu().numpy(), bt.x_star) <= 1e-9 and _rel(dual.cpu().numpy(), bt.y_star) <= 1e-9
    p_un, _, _, _ = _CvxpyLayerFused.apply(p_stack, cl, args, True, None)
    assert _rel(p_un.cpu().numpy(), bt.x_star) > 1e-7
