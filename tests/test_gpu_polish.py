"""Solution polishing on the GPU (csrc/polish.cu): against the NumPy restatement (tests/polish_ref.py) and the planted optimum,
starting from eps-1e-3 forward solves -- dense QPs, a CSR pattern, representatives of the register-tiled shape classes
(n > m, every row an equality, an LP at a vertex, m = 512, odd n), more than one wave of instances; rejected and
not-attempted instances keep their bits; the shared entry point and misaligned A / P give the same bits; structures with an
SOC are refused; and through the layer with ``solver_args={"polish": True}``: the planted optimum, the reverse-mode gradient
at it (tests/cone_ref.py exact adjoint), forward AD and the warm start."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, Solution, make_settings
from tests import cone_ref as cr
from tests import polish_ref as pref
from tests import tiled_shapes as ts
from tests.test_polish_host import _csr_qp

pytestmark = pytest.mark.gpu
DEV = "cuda"
LOOSE = {"eps": 1e-3}


def _t(a):
    return None if a is None else torch.tensor(a, dtype=torch.float64, device=DEV)


def _solve(bt, args=LOOSE):
    eng = Engine(bt.structure, DEV)
    A, P, b, c = _t(bt.A_vals), _t(bt.P_vals), _t(bt.b), _t(bt.c)
    sol = eng.solve(A, b, c, P, make_settings(args))
    return eng, A, P, b, c, sol


def _copy(sol):
    return Solution(*(t.clone() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)))


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


BATCHES = {
    "c1_like": lambda: pr.dense_qp(8, 40, 60, 10, seed=21),
    "csr_qp": lambda: _csr_qp(8, 16, 24, 3, seed=7),
    **{k: (lambda k=k: ts.planted(ts.CASES[k], 4, seed=5)) for k in ("kr4", "n_gt_m", "all_equality", "lp_vertex", "full_cta", "odd_mn")},
}


@pytest.mark.parametrize("key", list(BATCHES))
def test_kernel_matches_restatement_and_planted_optimum(key):
    bt = BATCHES[key]()
    eng, A, P, b, c, sol = _solve(bt)
    x0, y0, s0, status = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s, sol.status))
    flags = eng.polish(A, b, c, sol, P).cpu().numpy()
    fr, X, Y, S = pref.polish_batch(bt, x0, y0, s0, status)
    assert (flags == 1).all() and (fr == 1).all(), (key, flags, fr, status)
    x, y, s = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s))
    ref = max(_rel(x, X), _rel(y, Y), _rel(s, S))
    opt = max(_rel(x, bt.x_star), _rel(y, bt.y_star), _rel(s, bt.s_star))
    assert ref < 1e-10 and opt < 1e-9, (key, ref, opt)
    assert (sol.status.cpu().numpy() == status).all()


def test_more_than_one_wave():
    bt = ts.planted(ts.Case(10, 16, 3, 4, True, 0), 6000, seed=2)   # (strictly complementary: every iterate names the right set)
    eng, A, P, b, c, sol = _solve(bt)
    flags = eng.polish(A, b, c, sol, P).cpu().numpy()
    assert (flags == 1).all(), np.unique(flags, return_counts=True)
    x, y = sol.x.cpu().numpy(), sol.y.cpu().numpy()
    assert _rel(x, bt.x_star) < 1e-9 and _rel(y, bt.y_star) < 1e-9


def test_rejected_and_not_attempted_instances_keep_their_bits():
    bt = pr.dense_qp(64, 20, 30, 5, seed=11)
    eng, A, P, b, c, sol = _solve(bt, {"eps": 1e-3, "max_iters": 5, "acceleration_lookback": 0})
    sol.status.fill_(1)
    sol.status[0] = -4                     # FAILED: not attempted
    sol.x[1, 0] = float("nan")             # non-finite input: not attempted
    before = _copy(sol)
    flags = eng.polish(A, b, c, sol, P).cpu().numpy()
    assert flags[0] == -1 and flags[1] == -1
    assert (flags == 0).any(), flags
    for i in np.flatnonzero(flags <= 0):
        for a_, b_ in ((sol.x, before.x), (sol.y, before.y), (sol.s, before.s), (sol.resid, before.resid)):
            assert torch.equal(a_[i], b_[i]) or (i == 1 and torch.equal(a_[i].isnan(), b_[i].isnan())), i
    fr, X, _, _ = pref.polish_batch(bt, *(t.cpu().numpy() for t in (before.x, before.y, before.s)), before.status.cpu().numpy())
    assert (fr == flags).all(), (fr, flags)
    acc = flags == 1
    if acc.any():
        assert _rel(sol.x.cpu().numpy()[acc], X[acc]) < 1e-10


def test_shared_entry_point_and_misaligned_inputs_give_the_same_bits():
    bt = ts.planted(ts.CASES["nch1_live_eq_n"], 8, seed=9, shared=True)
    eng, A, P, b, c, sol = _solve(bt)
    base = _copy(sol)
    f_rep = eng.polish(A, b, c, sol, P)
    one = _copy(base)
    f_sh = eng.polish(A[0].clone(), b, c, one, P[0].clone())
    assert torch.equal(f_rep, f_sh) and (f_rep == 1).all()
    for u, v in ((sol.x, one.x), (sol.y, one.y), (sol.s, one.s), (sol.resid, one.resid)):
        assert torch.equal(u, v)
    mis = _copy(base)
    Am = torch.empty(A.numel() + 1, dtype=torch.float64, device=DEV)[1:].view(A.shape)
    Pm = torch.empty(P.numel() + 1, dtype=torch.float64, device=DEV)[1:].view(P.shape)
    Am.copy_(A)
    Pm.copy_(P)
    assert Am.data_ptr() % 16 == 8
    f_mis = eng.polish(Am, b, c, mis, Pm)
    assert torch.equal(f_mis, f_rep)
    for u, v in ((sol.x, mis.x), (sol.y, mis.y), (sol.s, mis.s)):
        assert torch.equal(u, v)


def test_soc_structure_is_refused():
    bt = pr.qp_as_socp(pr.dense_qp(2, 6, 9, 2, seed=1))
    eng, A, P, b, c, sol = _solve(bt)
    with pytest.raises(ValueError, match="zero and nonneg"):
        eng.polish(A, b, c, sol, P)


def _layer(monkeypatch, bt, opts=None):
    from cvxpylayers_b200 import interface as itf
    from tests.util import fake_param_prob, install_fake_cvxpylayers

    fake = install_fake_cvxpylayers(monkeypatch)
    problem, params = fake_param_prob(bt)
    itf.register(fuse=False)
    layer = fake.tl.CvxpyLayer(problem, [], [], solver="B200", solver_args=opts or {})
    return layer, [torch.tensor(p, device=DEV, requires_grad=True) for p in params]


def test_layer_refuses_polish_on_an_soc_structure(monkeypatch):
    layer, th = _layer(monkeypatch, pr.qp_as_socp(pr.dense_qp(2, 6, 9, 2, seed=1)))
    with pytest.raises(ValueError, match="zero and nonneg"):
        layer(*th, solver_args={"polish": True})


def _apply_fn(bt, opts, dev=DEV):
    """(P_eval, q_eval, A_eval) -> (primal, dual) through _CvxpyLayer.apply on the boundary layout of ``bt`` (as
    tests/test_gpu_jvp.py), and the layer's solver context."""
    from cvxpylayers_b200.interface import B200_ctx, _CvxpyLayer

    st = bt.structure
    bd = pr.to_boundary(bt)
    P_struct = (st.P_indices, st.P_indptr, (st.n, st.n)) if st.nnzP else None
    ctx = B200_ctx(P_struct, (bd.con_indices, bd.con_ptr, bd.shape), bd.dims, options=opts, device=dev)
    cl = type("CL", (), {"solver_ctx": ctx})()
    return bd, ctx, (lambda P, q, A, args=None: _CvxpyLayer.apply(P, q, A, cl, args or {}, True, None)[:2])


def test_layer_refuses_polish_before_staging_any_chunk(monkeypatch):
    """Pageable host inputs over several pipeline chunks take the staged path; an unsupported structure is refused before a chunk
    is staged, and the engine's stager still serves the next call."""
    from cvxpylayers_b200 import interface as itf

    monkeypatch.setattr(itf, "PIPE_CHUNK", 4)
    bt = pr.qp_as_socp(pr.dense_qp(24, 6, 9, 2, seed=1))   # 6 chunks: more than the stager's ring of 3 slots
    bd, ctx, f = _apply_fn(bt, {"eps": 1e-6})
    P, q, A = (None if a is None else torch.tensor(a) for a in (bd.P_eval, bd.q_eval, bd.A_eval))   # pageable CPU tensors
    assert itf._stage_ok(24, A, q, P)
    with pytest.raises(ValueError, match="zero and nonneg"):
        f(P, q, A, {"polish": True})
    primal, _ = f(P, q, A)
    assert primal.shape == (24, bt.structure.n) and torch.isfinite(primal).all()
    eng, = ctx._engines.values()
    assert getattr(eng, "_stager", None) is not None   # (the staged path ran)


def test_layer_polished_solution_gradient_forward_ad_and_warm_start(monkeypatch):
    bt = ts.planted(ts.CASES["nch1_live_eq_n"], 3, seed=4)
    layer, th = _layer(monkeypatch, bt, {"polish": True, "eps": 1e-3, "warm_start": True})
    primal, dual = layer(*th)
    assert _rel(primal.detach().cpu().numpy(), bt.x_star) < 1e-9 and _rel(dual.detach().cpu().numpy(), bt.y_star) < 1e-9
    ctx = layer.ctx.solver_ctx
    (xw, yw, _), = ctx._last_solution.values()
    assert torch.equal(xw, primal.detach()) and torch.equal(yw, dual.detach())   # the warm start keeps the polished point
    with torch.no_grad():
        p_un, _ = layer(*th, solver_args={"polish": False, "warm_start": False})
    assert _rel(p_un.cpu().numpy(), bt.x_star) > 1e-6

    # reverse mode through the layer (its saved point feeds the backward) against the exact adjoint at the planted optimum, emitted
    # to the boundary layout by the same engine map the layer's backward uses
    rng = np.random.default_rng(0)
    dx, dy = rng.standard_normal(bt.x_star.shape), rng.standard_normal(bt.y_star.shape)
    exact = [cr.exact_adjoint(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i], dx[i], dy[i],
                              bt.structure.cones) for i in range(bt.B)]
    bd, lctx, f = _apply_fn(bt, {"eps": 1e-3, "lsqr_atol": 1e-14, "lsqr_btol": 1e-14, "lsqr_conlim": 1e14})
    eng = lctx.engine(torch.device(DEV, torch.cuda.current_device()))
    eA, eq, _ = eng.emit(_t(np.stack([e[0].ravel() for e in exact])), None, _t(np.stack([e[2] for e in exact])),
                         _t(np.stack([e[3] for e in exact])))
    eA, eq = eA.cpu().numpy(), eq.cpu().numpy()
    for pre in (1, 2):
        errs = []
        for pol in (True, False):
            P, q, A = (_t(a).requires_grad_(True) for a in (bd.P_eval, bd.q_eval, bd.A_eval))
            x, y = f(P, q, A, {"polish": pol, "lsqr_precond": pre})
            ((x * _t(dx)).sum() + (y * _t(dy)).sum()).backward()
            errs.append(max(_rel(A.grad.cpu().numpy(), eA), _rel(q.grad.cpu().numpy(), eq)))
        assert errs[0] < 1e-7 and errs[1] > 10 * errs[0], (pre, errs)

    # forward AD through the polished layer
    import torch.autograd.forward_ad as fwAD

    bd, _, f = _apply_fn(bt, {"polish": True, "eps": 1e-3})
    Pe, qe, Ae = _t(bd.P_eval), _t(bd.q_eval), _t(bd.A_eval)
    with fwAD.dual_level():
        out = f(fwAD.make_dual(Pe, torch.randn_like(Pe)), fwAD.make_dual(qe, torch.randn_like(qe)), fwAD.make_dual(Ae, torch.randn_like(Ae)))
        x_fw, tan = fwAD.unpack_dual(out[0])
    assert _rel(x_fw.cpu().numpy(), bt.x_star) < 1e-9
    assert tan is not None and torch.isfinite(tan).all()
