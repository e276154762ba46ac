"""Solution polishing past the on-chip limit on the GPU (csrc/polish_large.cu, the slab tier): against the NumPy restatement
(tests/polish_ref.py) and the planted optimum -- the host test's batches, n = 129 with a dense A, odd n = 257, every row an
equality, an LP at a vertex and a C4-shaped sparse LP -- from a real eps-1e-3 forward, not-attempted and rejected instances
keeping their bits, more than one wave of instances, the shared entry point and misaligned A / P, and through both layers
with ``solver_args={"polish": True}``.  The on-chip structures of tests/test_gpu_polish.py keep the on-chip tier."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, Solution, make_settings
from tests import cone_ref as cr
from tests import polish_ref as pref
from tests import tiled_shapes as ts
from tests.test_gpu_polish import BATCHES as ON_CHIP
from tests.test_polish_large_host import large_batches, perturbed_start

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _t(a):
    return None if a is None else torch.tensor(a, dtype=torch.float64, device=DEV)


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _copy(sol):
    return Solution(*(t.clone() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)))


def _start(bt, x, y, s):
    B = bt.B
    return Solution(_t(x), _t(y), _t(s), torch.ones(B, dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV),
                    torch.full((B, 3), 1.0, dtype=torch.float64, device=DEV))


BATCHES = {
    **large_batches(),
    "dense_129": lambda: ts.planted(ts.Case(129, 160, 20, 40, True, 0), 3, seed=5),
    "odd_257": lambda: ts.planted(ts.Case(257, 301, 41, 60, True, 0), 2, seed=6),
    "all_equality": lambda: ts.planted(ts.Case(150, 100, 100, 0, True, 0), 3, seed=7),
    "lp_vertex": lambda: pr.dense_lp(3, 140, 300, seed=8),
    "c4_shape": lambda: pr.sparse_lp(4, 1000, 2000, seed=1),
}
# C4's live rows are a random sparse 1000 x 1000 matrix, not conditioned like the dense planted ones: the twin itself lands about
# 1e-9 from the planted vertex there, and the kernel's Schur-complement solve agrees with its direct solve to that order
TOL = {"c4_shape": 1e-8}


@pytest.mark.parametrize("key", list(BATCHES))
def test_slab_tier_matches_restatement_and_planted_optimum(key):
    bt = BATCHES[key]()
    eng = Engine(bt.structure, DEV)
    assert eng.polish_info()["tier"] == 1
    x0, y0, s0 = perturbed_start(bt, seed=11)
    sol = _start(bt, x0, y0, s0)
    flags = eng.polish(_t(bt.A_vals), _t(bt.b), _t(bt.c), sol, _t(bt.P_vals)).cpu().numpy()
    fr, X, Y, S = pref.polish_batch(bt, x0, y0, s0)
    assert (flags == fr).all() and (flags == 1).all(), (key, flags, fr)
    x, y, s = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s))
    ref = max(_rel(x, X), _rel(y, Y), _rel(s, S))
    opt = max(_rel(x, bt.x_star), _rel(y, bt.y_star), _rel(s, bt.s_star))
    assert ref < TOL.get(key, 1e-10) and opt < TOL.get(key, 1e-9), (key, ref, opt)
    assert (sol.status.cpu().numpy() == 1).all()
    r = sol.resid.cpu().numpy()
    assert (r < 1e-8).all(), (key, r.max(0))


@pytest.mark.parametrize("key", list(ON_CHIP))
def test_on_chip_structures_keep_the_on_chip_tier(key):
    info = Engine(ON_CHIP[key]().structure, DEV).polish_info()
    assert info["tier"] == 0 and info["slab_bytes_per_cta"] == 0, info


@pytest.mark.parametrize("key", ["sparse_lp_200", "dense_qp_200"])
def test_from_a_real_forward_matches_restatement(key):
    """An eps-1e-3 forward's iterate as the input.  On the sparse LP it names more live rows than n (nothing is attempted, as on C4
    at that eps); on the strictly complementary dense QP it names the planted active set."""
    bt = pr.sparse_lp(4, 200, 400, density=0.05, seed=12) if key == "sparse_lp_200" else ts.planted(LAYER_CASE, 4, seed=20)
    eng = Engine(bt.structure, DEV)
    A, P, b, c = _t(bt.A_vals), _t(bt.P_vals), _t(bt.b), _t(bt.c)
    sol = eng.solve(A, b, c, P, make_settings({"eps": 1e-3}))
    x0, y0, s0, status = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s, sol.status))
    flags = eng.polish(A, b, c, sol, P).cpu().numpy()
    fr, X, Y, S = pref.polish_batch(bt, x0, y0, s0, status)
    assert (flags == fr).all(), (flags, fr, status)
    if key == "dense_qp_200":
        assert (flags == 1).all(), flags
    acc = flags == 1
    x, y, s = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s))
    if acc.any():
        assert max(_rel(x[acc], X[acc]), _rel(y[acc], Y[acc]), _rel(s[acc], S[acc])) < 1e-10
    assert (sol.status.cpu().numpy() == status).all()


def test_not_attempted_and_rejected_instances_keep_their_bits():
    bt = ts.planted(ts.Case(140, 200, 20, 40, True, 0), 16, seed=13)
    eng = Engine(bt.structure, DEV)
    A, P, b, c = _t(bt.A_vals), _t(bt.P_vals), _t(bt.b), _t(bt.c)
    sol = eng.solve(A, b, c, P, make_settings({"eps": 1e-3, "max_iters": 5, "acceleration_lookback": 0}))
    sol.status.fill_(1)
    sol.status[0] = -4                     # FAILED: not attempted
    sol.x[1, 0] = float("nan")             # non-finite input: not attempted
    sol.y[2] = 1.0                         # every row live: nl = m > n, not attempted
    sol.s[2] = 0.0
    before = _copy(sol)
    flags = eng.polish(A, b, c, sol, P).cpu().numpy()
    assert flags[0] == -1 and flags[1] == -1 and flags[2] == -1, flags
    assert (flags == 0).any(), flags
    for i in np.flatnonzero(flags <= 0):
        for a_, b_ in ((sol.x, before.x), (sol.y, before.y), (sol.s, before.s), (sol.resid, before.resid)):
            assert torch.equal(a_[i], b_[i]) or (i == 1 and torch.equal(a_[i].isnan(), b_[i].isnan())), i
    fr, X, _, _ = pref.polish_batch(bt, *(t.cpu().numpy() for t in (before.x, before.y, before.s)), before.status.cpu().numpy())
    assert (fr == flags).all(), (fr, flags)
    acc = flags == 1
    if acc.any():
        assert _rel(sol.x.cpu().numpy()[acc], X[acc]) < 1e-10


def test_more_than_one_wave():
    probe = ts.planted(ts.Case(136, 150, 10, 30, True, 0), 1, seed=14)
    grid = Engine(probe.structure, DEV).polish_info()["ctas"]
    bt = ts.planted(ts.Case(136, 150, 10, 30, True, 0), 3 * grid + 5, seed=14)
    eng = Engine(bt.structure, DEV)
    x0, y0, s0 = perturbed_start(bt, seed=15)
    sol = _start(bt, x0, y0, s0)
    flags = eng.polish(_t(bt.A_vals), _t(bt.b), _t(bt.c), sol, _t(bt.P_vals)).cpu().numpy()
    assert (flags == 1).all(), np.unique(flags, return_counts=True)
    x, y = sol.x.cpu().numpy(), sol.y.cpu().numpy()
    assert _rel(x, bt.x_star) < 1e-9 and _rel(y, bt.y_star) < 1e-9


def test_shared_entry_point_and_misaligned_inputs_give_the_same_bits():
    bt = ts.planted(ts.Case(160, 200, 20, 50, True, 0), 6, seed=16, shared=True)
    eng = Engine(bt.structure, DEV)
    A, P, b, c = _t(bt.A_vals), _t(bt.P_vals), _t(bt.b), _t(bt.c)
    base = _start(bt, *perturbed_start(bt, seed=17))
    rep = _copy(base)
    f_rep = eng.polish(A, b, c, rep, P)
    one = _copy(base)
    f_sh = eng.polish(A[0].clone(), b, c, one, P[0].clone())
    assert torch.equal(f_rep, f_sh) and (f_rep == 1).all()
    for u, v in ((rep.x, one.x), (rep.y, one.y), (rep.s, one.s), (rep.resid, one.resid)):
        assert torch.equal(u, v)
    mis = _copy(base)
    Am = torch.empty(A.numel() + 1, dtype=torch.float64, device=DEV)[1:].view(A.shape)
    Pm = torch.empty(P.numel() + 1, dtype=torch.float64, device=DEV)[1:].view(P.shape)
    Am.copy_(A)
    Pm.copy_(P)
    assert Am.data_ptr() % 16 == 8
    f_mis = eng.polish(Am, b, c, mis, Pm)
    assert torch.equal(f_mis, f_rep)
    for u, v in ((rep.x, mis.x), (rep.y, mis.y), (rep.s, mis.s)):
        assert torch.equal(u, v)


LAYER_CASE = ts.Case(200, 260, 30, 50, True, 0)


def _apply_fn(bt, opts):
    from cvxpylayers_b200.interface import B200_ctx, _CvxpyLayer

    st = bt.structure
    bd = pr.to_boundary(bt)
    ctx = B200_ctx((st.P_indices, st.P_indptr, (st.n, st.n)), (bd.con_indices, bd.con_ptr, bd.shape), bd.dims, options=opts, device=DEV)
    cl = type("CL", (), {"solver_ctx": ctx})()
    return bd, ctx, (lambda P, q, A, args=None: _CvxpyLayer.apply(P, q, A, cl, args or {}, True, None)[:2])


def test_layer_polishes_past_the_on_chip_limit(monkeypatch):
    """_CvxpyLayer on device inputs and on pageable inputs over several chunks (the staged path): the planted optimum, the
    reverse-mode gradient at it against the exact adjoint (lsqr_precond 1 and 2), forward AD and the warm start."""
    from cvxpylayers_b200 import interface as itf

    bt = ts.planted(LAYER_CASE, 6, seed=18)
    bd, ctx, f = _apply_fn(bt, {"polish": True, "eps": 1e-3, "warm_start": True})
    primal, dual = f(_t(bd.P_eval), _t(bd.q_eval), _t(bd.A_eval))
    assert _rel(primal.detach().cpu().numpy(), bt.x_star) < 1e-9 and _rel(dual.detach().cpu().numpy(), bt.y_star) < 1e-9
    (xw, yw, _), = ctx._last_solution.values()
    assert torch.equal(xw, primal.detach()) and torch.equal(yw, dual.detach())   # the warm start keeps the polished point

    monkeypatch.setattr(itf, "PIPE_CHUNK", 2)
    bd2, ctx2, f2 = _apply_fn(bt, {"polish": True, "eps": 1e-3})
    P, q, A = (torch.tensor(a) for a in (bd2.P_eval, bd2.q_eval, bd2.A_eval))   # pageable CPU tensors
    assert itf._stage_ok(bt.B, A, q, P)
    p_st, d_st = f2(P, q, A)
    assert _rel(p_st.cpu().numpy(), bt.x_star) < 1e-9 and _rel(d_st.cpu().numpy(), bt.y_star) < 1e-9
    eng, = ctx2._engines.values()
    assert getattr(eng, "_stager", None) is not None   # (the staged path ran)
    monkeypatch.undo()

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
        P, q, A = (_t(a).requires_grad_(True) for a in (bd.P_eval, bd.q_eval, bd.A_eval))
        x, y = f(P, q, A, {"polish": True, "lsqr_precond": pre})
        ((x * _t(dx)).sum() + (y * _t(dy)).sum()).backward()
        err = max(_rel(A.grad.cpu().numpy(), eA), _rel(q.grad.cpu().numpy(), eq))
        assert err < 1e-7, (pre, err)

    import torch.autograd.forward_ad as fwAD

    bd, _, f = _apply_fn(bt, {"polish": True, "eps": 1e-3})
    Pe, qe, Ae = _t(bd.P_eval), _t(bd.q_eval), _t(bd.A_eval)
    with fwAD.dual_level():
        out = f(fwAD.make_dual(Pe, torch.randn_like(Pe)), fwAD.make_dual(qe, torch.randn_like(qe)), fwAD.make_dual(Ae, torch.randn_like(Ae)))
        x_fw, tan = fwAD.unpack_dual(out[0])
    assert _rel(x_fw.cpu().numpy(), bt.x_star) < 1e-9
    assert tan is not None and torch.isfinite(tan).all()


def test_fused_layer_polishes_past_the_on_chip_limit(monkeypatch):
    """The registered fused layer (_CvxpyLayerFused) with polish=True, replicated matrices."""
    from cvxpylayers_b200 import interface as itf
    from tests.util import fake_param_prob, install_fake_cvxpylayers

    bt = ts.planted(LAYER_CASE, 3, seed=19)
    fake = install_fake_cvxpylayers(monkeypatch)
    problem, params = fake_param_prob(bt)
    itf.register(fuse=True)
    layer = fake.tl.CvxpyLayer(problem, [], [], solver="B200", solver_args={"polish": True, "eps": 1e-3})
    th = [torch.tensor(p, device=DEV, requires_grad=True) for p in params]
    primal, dual = layer(*th)
    assert _rel(primal.detach().cpu().numpy(), bt.x_star) < 1e-9 and _rel(dual.detach().cpu().numpy(), bt.y_star) < 1e-9
    (primal.sum() + dual.sum()).backward()
    assert all(t.grad is not None and torch.isfinite(t.grad).all() for t in th)
