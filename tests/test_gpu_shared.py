"""Batch-shared A and P (bcone_solve_shared / bcone_vjp_shared / bcone_jvp_shared, Engine with 1-D matrices, the fused layer's
``shared_matrices`` option).  "Replicated" is the same data through the existing entry points with ``A.expand(B, -1).contiguous()``:
the shared paths must compute what they compute -- bit for bit where the kernels involve no floating-point atomics, and to
rounding for the batch-summed gradient."""
import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from cvxpylayers_b200.interface import _CvxpyLayerFused, get_solver_ctx

pytestmark = pytest.mark.gpu

TIGHT = {"lsqr_precond": 1, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12}


def _t(a, dev):
    return torch.tensor(np.ascontiguousarray(a), device=dev)


def shared_batch(name, B, seed=0):
    """A batch of `name`'s structure whose instances share instance 0's A and P.  Dense QPs get a planted optimum per instance
    (b, c vary widely); the other structures perturb instance 0's b and c (stays feasible, keeps the cone data meaningful)."""
    base = pr.CONFIGS[name](B=1, seed=seed)
    st = base.structure
    rng = np.random.default_rng(seed + 17)
    A = np.repeat(base.A_vals[:1], B, 0)
    P = None if base.P_vals is None else np.repeat(base.P_vals[:1], B, 0)
    if name in ("C1", "C2"):
        return pr.plant(st, A, P, rng, active_frac=0.2)
    b = base.b[:1] + 1e-3 * rng.standard_normal((B, st.m)) * (np.abs(base.b[:1]).max() + 1.0)
    c = base.c[:1] * (1.0 + 1e-3 * rng.standard_normal((B, st.n)))
    return pr.Batch(st, A, np.ascontiguousarray(b), np.ascontiguousarray(c), P, name=base.name)


def _data(bt, dev):
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    P = None if bt.P_vals is None else _t(bt.P_vals, dev)
    return A, P, b, c


def _shared(A, P):
    return A[0].contiguous(), (None if P is None else P[0].contiguous())


def _same_sol(a, b, keys=("x", "y", "s", "status", "iters")):
    return {k: torch.equal(getattr(a, k), getattr(b, k)) for k in keys}


def _rel_close(a, b, tol):
    scale = max(float(b.abs().max()), 1e-300)
    return float((a - b).abs().max()) <= tol * scale


@pytest.fixture(scope="module")
def c2_4096(cuda_device):
    return shared_batch("C2", 4096, seed=3)


# ----------------------------------------------------------------------------- forward
@pytest.mark.parametrize("name", ["C1", "C2"])
def test_solve_shared_is_bit_identical_cold_and_warm(name, cuda_device, c2_4096):
    dev = cuda_device
    bt = c2_4096 if name == "C2" else shared_batch("C1", 512, seed=5)
    eng = Engine(bt.structure, dev)
    if name == "C2":
        assert "register-tiled" in eng.path_info()["fwd"]
    A, P, b, c = _data(bt, dev)
    As, Ps = _shared(A, P)
    S = make_settings({})
    rep = eng.solve(A, b, c, P, S)
    got = eng.solve(As, b, c, Ps, S)
    assert all(_same_sol(got, rep).values()), _same_sol(got, rep)
    assert int((rep.status == 1).sum()) == bt.B
    if name == "C2":
        # instances whose adaptive scale moved re-factorised privately (the shared record is read only): they are the ones
        # whose iterations change when the adaptive scaling is off, and they are among the bit-identical ones above
        fixed = eng.solve(A, b, c, P, make_settings({"adaptive_scale": 0}))
        moved = (fixed.iters != rep.iters) | (fixed.x != rep.x).any(1)
        assert int(moved.sum()) >= 1
        again = eng.solve(As, b, c, Ps, S)   # the set-up record of the previous call is rebuilt, not trusted
        assert all(_same_sol(again, rep).values())
    rng = np.random.default_rng(1)
    b2 = b + 1e-3 * _t(rng.standard_normal(bt.b.shape), dev)
    warm = (rep.x.clone(), rep.y.clone(), rep.s.clone())
    rep_w = eng.solve(A, b2, c, P, S, warm=warm)
    got_w = eng.solve(As, b2, c, Ps, S, warm=warm)
    assert all(_same_sol(got_w, rep_w).values()), _same_sol(got_w, rep_w)


def test_solve_shared_cg_is_bit_identical(cuda_device):
    bt = shared_batch("C4", 32, seed=2)
    eng = Engine(bt.structure, cuda_device)
    A, P, b, c = _data(bt, cuda_device)
    S = make_settings({"max_iters": 20000})
    As, Ps = _shared(A, P)
    rep, got = eng.solve(A, b, c, P, S), eng.solve(As, b, c, Ps, S)
    assert all(_same_sol(got, rep).values())


@pytest.mark.parametrize("name,vals_global", [("C3", False), ("C5", False), ("EXP", False), ("C2SOC", False), ("C3", True)])
def test_solve_shared_atomic_K_agrees(name, vals_global, cuda_device, monkeypatch):
    if vals_global:
        monkeypatch.setenv("BCONE_VALUES_GLOBAL", "1")
    bt = shared_batch(name, 64, seed=4)
    eng = Engine(bt.structure, cuda_device)
    A, P, b, c = _data(bt, cuda_device)
    S = make_settings({"eps": 1e-8, "max_iters": 100000})
    rep = eng.solve(A, b, c, P, S)
    As, Ps = _shared(A, P)
    got = eng.solve(As, b, c, Ps, S)
    assert torch.equal(got.status, rep.status)
    for k in ("x", "y", "s"):
        assert _rel_close(getattr(got, k), getattr(rep, k), 1e-8), k


# ----------------------------------------------------------------------------- adjoint
def _check_vjp(bt, dev, args):
    eng = Engine(bt.structure, dev)
    A, P, b, c = _data(bt, dev)
    As, Ps = _shared(A, P)
    S = make_settings(args)
    sol = eng.solve(A, b, c, P, S)
    rng = np.random.default_rng(7)
    dx, dy = _t(rng.standard_normal((bt.B, bt.structure.n)), dev), _t(rng.standard_normal((bt.B, bt.structure.m)), dev)
    dA, dP, db, dc, its = eng.vjp(A, b, c, sol.x, sol.y, sol.s, dx, dy, P, S)
    g1 = eng.vjp(As, b, c, sol.x, sol.y, sol.s, dx, dy, Ps, S)
    g2 = eng.vjp(As, b, c, sol.x, sol.y, sol.s, dx, dy, Ps, S)
    assert g1[0].shape == (bt.structure.nnzA,)
    assert torch.equal(g1[2], db) and torch.equal(g1[3], dc) and torch.equal(g1[4], its)
    assert all(torch.equal(u, v) for u, v in zip(g1, g2) if u is not None)   # fixed-order reduction: identical bits
    for got, per in ((g1[0], dA), (g1[1], dP)):
        if per is None:
            continue
        err = (got - per.sum(0)).abs()
        assert bool((err <= 1e-12 * per.abs().sum(0) + 1e-300).all()), float((err / per.abs().sum(0).clamp_min(1e-300)).max())
    return eng


@pytest.mark.parametrize("name", ["C1", "C2"])
@pytest.mark.parametrize("precond", [0, 1, 2])
def test_vjp_shared_dense(name, precond, cuda_device):
    bt = shared_batch(name, 512, seed=9)
    eng = _check_vjp(bt, cuda_device, {"lsqr_precond": precond})
    if precond == 2 and name == "C2":   # the block pass wrote every record: nothing was handed to the fallback
        assert eng.path_info()["bwd"].startswith("bwd_block_kernel") and eng.fallback_count() == 0


def test_vjp_shared_block_fallback(cuda_device):
    """A P with an exactly zero row and column: the block factorisation rejects it, so with a shared P every instance goes to the
    fallback pass (bwd_fast_kernel on the rejected list), which writes the records instead."""
    base = pr.CONFIGS["C2"](B=1, seed=11)
    n = base.structure.n
    Pd = base.P_dense(0)
    Pd[45, :] = 0.0
    Pd[:, 45] = 0.0
    iu = np.triu_indices(n)
    B = 64
    bt = pr.plant(base.structure, np.repeat(base.A_vals, B, 0), np.repeat(Pd[iu][None], B, 0), np.random.default_rng(12), active_frac=0.2)
    eng = _check_vjp(bt, cuda_device, {"lsqr_precond": 2})
    assert eng.path_info()["bwd"].startswith("bwd_block_kernel") and eng.fallback_count() == B


@pytest.mark.parametrize("name,vals_global", [("C3", False), ("C5", False), ("EXP", False), ("C2SOC", False), ("C5", True)])
def test_vjp_shared_generic(name, vals_global, cuda_device, monkeypatch):
    if vals_global:
        monkeypatch.setenv("BCONE_VALUES_GLOBAL", "1")
    _check_vjp(shared_batch(name, 64, seed=4), cuda_device, {"eps": 1e-8, **TIGHT})


# ----------------------------------------------------------------------------- forward mode
@pytest.mark.parametrize("name", ["C2", "C3"])
def test_jvp_shared(name, cuda_device):
    dev = cuda_device
    bt = shared_batch(name, 128, seed=6)
    st = bt.structure
    eng = Engine(st, dev)
    A, P, b, c = _data(bt, dev)
    As, Ps = _shared(A, P)
    S = make_settings({"eps": 1e-8, **TIGHT})
    sol = eng.solve(As, b, c, Ps, S)
    rng = np.random.default_rng(8)
    tA = _t(rng.standard_normal(st.nnzA), dev)
    tP = None if P is None else _t(rng.standard_normal(st.nnzP), dev)
    tb, tc = _t(rng.standard_normal((bt.B, st.m)), dev), _t(rng.standard_normal((bt.B, st.n)), dev)
    rep = eng.jvp(A, b, c, sol.x, sol.y, sol.s, tA.expand(bt.B, -1).contiguous(), tb, tc, P,
                  None if tP is None else tP.expand(bt.B, -1).contiguous(), S)
    got = eng.jvp(As, b, c, sol.x, sol.y, sol.s, tA, tb, tc, Ps, tP, S)
    assert all(torch.equal(u, v) for u, v in zip(got, rep))
    # adjoint identity: sum_b <w_b, jvp(t)_b> = <vjp_shared(w), t>
    wx, wy = _t(rng.standard_normal((bt.B, st.n)), dev), _t(rng.standard_normal((bt.B, st.m)), dev)
    gA, gP, gb, gc, _ = eng.vjp(As, b, c, sol.x, sol.y, sol.s, wx, wy, Ps, S)
    lhs = float((wx * got[0]).sum() + (wy * got[1]).sum())
    rhs = float((gA * tA).sum() + (gb * tb).sum() + (gc * tc).sum() + (0.0 if tP is None else (gP * tP).sum()))
    assert abs(lhs - rhs) <= 1e-10 * max(1.0, abs(lhs), abs(rhs)), (lhs, rhs)


# ----------------------------------------------------------------------------- the fused layer
def _fused(bt, dev, args):
    from tests.util import fake_param_prob

    problem, params = fake_param_prob(bt)
    ctx = get_solver_ctx("B200", problem["param_prob"], problem["dims"], {}, args)
    ctx.device = dev
    cl = type("CL", (), {"solver_ctx": ctx})()
    p_stack = torch.as_tensor(np.concatenate([p.T for p in params] + [np.ones((1, bt.B))]), dtype=torch.float64, device=dev)
    return ctx, cl, p_stack


def test_fused_layer_shared_matrices(cuda_device):
    dev = cuda_device
    bt = shared_batch("C2", 256, seed=11)
    st = bt.structure
    ctx, cl, p_stack = _fused(bt, dev, {})
    matrix_rows = torch.zeros(p_stack.shape[0], dtype=torch.bool)
    matrix_rows[:st.nnzA] = True
    matrix_rows[st.nnzA + ctx.b_idx.size + st.n:-1] = True   # P values
    outs = {}
    g = torch.Generator().manual_seed(2)
    dprimal = torch.randn((bt.B, st.n), dtype=torch.float64, generator=g).to(dev)
    ddual = torch.randn((bt.B, st.m), dtype=torch.float64, generator=g).to(dev)
    for on in (False, True):
        ps = p_stack.clone().requires_grad_(True)
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        primal, dual, _, _ = _CvxpyLayerFused.apply(ps, cl, {"shared_matrices": on}, True, None)
        ((primal * dprimal).sum() + (dual * ddual).sum()).backward()
        outs[on] = (primal.detach(), dual.detach(), ps.grad.detach(), torch.cuda.max_memory_allocated(dev) - base)
    assert torch.equal(outs[True][0], outs[False][0]) and torch.equal(outs[True][1], outs[False][1])
    g_on, g_off = outs[True][2], outs[False][2]
    assert torch.equal(g_on[~matrix_rows], g_off[~matrix_rows])
    s_on, s_off, s_abs = g_on[matrix_rows].sum(1), g_off[matrix_rows].sum(1), g_off[matrix_rows].abs().sum(1)
    assert bool(((s_on - s_off).abs() <= 1e-12 * s_abs + 1e-300).all())
    # no [B, nnzA] / [B, nnzP] tensor on the shared path: its peak stays below the replicated path's by at least that much
    assert outs[True][3] + bt.B * st.nnzA * 8 <= outs[False][3], (outs[True][3], outs[False][3])


def test_fused_layer_shared_forward_ad_and_gradcheck(cuda_device):
    dev = cuda_device
    bt = shared_batch("C1", 3, seed=12)   # inequality rows only (the OptNet shape): tangents on inactive rows reach the forward mode
    _, cl, p_stack = _fused(bt, dev, {})
    args = {"eps": 1e-11, "max_iters": 200000, "shared_matrices": True, **TIGHT}

    def f(ps):
        return _CvxpyLayerFused.apply(ps, cl, args, True, None)[:2]

    assert torch.autograd.gradcheck(f, (p_stack.clone().requires_grad_(True),), eps=1e-6, atol=1e-4, rtol=1e-3,
                                    check_forward_ad=True, check_undefined_grad=False)


def test_shared_matrices_excludes_reuse_setup(cuda_device):
    bt = shared_batch("C1", 4, seed=1)
    _, cl, p_stack = _fused(bt, cuda_device, {})
    with pytest.raises(ValueError, match="reuse_setup"):
        _CvxpyLayerFused.apply(p_stack, cl, {"shared_matrices": True, "reuse_setup": True}, True, None)
