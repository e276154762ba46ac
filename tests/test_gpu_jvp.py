"""Forward-mode derivative of the solution map on the GPU (``bcone_jvp``, diffcp's ``D``):

* against the exact least-squares solve of the dense restatement (``tests/jvp_ref.py``) for every LSQR variant;
* the adjoint identity <w, J t> = <J'w, t> between ``bcone_jvp`` and ``bcone_vjp`` at full batch, including C2 where the
  adjoint runs the fused and block-preconditioned kernels, and C4's large instances (vectors in the global slab);
* central differences of GPU solves on the reference's PSD / SOC gradcheck programs, and ``gradcheck(check_forward_ad=True)``;
* ``torch.autograd.forward_ad`` through every autograd Function of the layer against the reverse-mode Jacobian.
"""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from cvxpylayers_b200.interface import B200_ctx, _CvxpyLayer, _CvxpyLayerFused, get_solver_ctx
from oracle import oracle as orc
from tests.jvp_ref import dense_M, jvp_dense, jvp_rhs, random_tangents
from tests.util import ref_sdp_batch, ref_soc_batch

pytestmark = pytest.mark.gpu

TIGHT = {"lsqr_precond": 1, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12}


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _rel_rows(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return np.abs(a - b).reshape(a.shape[0], -1).max(1) / np.maximum(np.abs(b).reshape(b.shape[0], -1).max(1), 1e-30)


def _gpu_jvp(eng, bt, t, x, y, s, dev, args):
    return eng.jvp(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(x, dev), _t(y, dev), _t(s, dev), _t(t.A_vals, dev), _t(t.b, dev),
                   _t(t.c, dev), _t(bt.P_vals, dev), _t(t.P_vals, dev), make_settings(args))


def _dense_instance(bt, t, i, x, y, s, **kw):
    P = bt.P_dense(i) if bt.P_vals is not None else None
    dP = t.P_dense(i) if t.P_vals is not None else None
    return jvp_dense(bt.structure, bt.A_dense(i), P, bt.b[i], bt.c[i], x[i], y[i], s[i], t.A_dense(i), dP, t.b[i], t.c[i], **kw)


# ----------------------------------------------------------------------------- every LSQR variant vs an exact least-squares solve
@pytest.mark.parametrize("name,B", [("C1", 4), ("C2", 4), ("C3", 4), ("C5", 3), ("EXP", 4)])
def test_jvp_lsqr_variants_against_exact_least_squares(name, B, cuda_device):
    bt = pr.CONFIGS[name](B=B)
    st, dev = bt.structure, cuda_device
    xo, yo, so, sto, _ = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-11, max_iters=400000)
    assert (sto == 1).all()
    t = random_tangents(bt, np.random.default_rng(5))
    lim = 40 * (st.n + st.m + 1)
    exact = [_dense_instance(bt, t, i, xo, yo, so) for i in range(B)]
    eng = Engine(st, dev)
    out, err = {}, {}
    for pc in (0, 1, 2):
        out[pc] = [a.cpu() for a in _gpu_jvp(eng, bt, t, xo, yo, so, dev, {"lsqr_precond": pc, "lsqr_iter_lim": lim})]
        err[pc] = max(_rel_rows(out[pc][k], np.stack([e[k] for e in exact])).max() for k in range(3))
    assert err[1] < 1e-4, (name, err)
    assert all(torch.equal(out[2][k], out[1][k]) for k in range(4)), "lsqr_precond = 2 must run as 1"
    assert err[0] < 5e-3, (name, err)
    if err[0] > 1e-4:   # plain LSQR's stopping rule: SciPy on the same explicit M misses by as much
        sp_ = [_dense_instance(bt, t, i, xo, yo, so, exact=False, iter_lim=lim) for i in range(B)]
        err_s = max(_rel_rows(np.stack([e[k] for e in sp_]), np.stack([e[k] for e in exact])).max() for k in range(3))
        assert err[0] <= 10 * err_s, (name, err[0], err_s)


# ----------------------------------------------------------------------------- the adjoint identity against bcone_vjp
@pytest.mark.parametrize("name,B", [("C3", 2048), ("C5", 256), ("C2", 4096), ("C4", 64)])
def test_jvp_is_the_transpose_of_vjp(name, B, cuda_device):
    bt = pr.CONFIGS[name](B=B)
    st, dev = bt.structure, cuda_device
    eng = Engine(st, dev)
    if bt.x_star is not None:   # planted optimum: exact
        x, y, s = _t(bt.x_star, dev), _t(bt.y_star, dev), _t(bt.s_star, dev)
    else:
        sol = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings({"eps": 1e-9, "max_iters": 200000}))
        assert int((sol.status == 1).sum()) == B
        x, y, s = sol.x, sol.y, sol.s
    rng = np.random.default_rng(9)
    t = random_tangents(bt, rng)
    w = (rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m)))
    args = {**TIGHT, "lsqr_iter_lim": 40 * (st.n + st.m + 1)}
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    dx, dy, ds, its = eng.jvp(A, b, c, x, y, s, _t(t.A_vals, dev), _t(t.b, dev), _t(t.c, dev), P, _t(t.P_vals, dev), make_settings(args))
    dx, dy = dx.cpu().numpy(), dy.cpu().numpy()
    assert (its.cpu().numpy() > 0).all()
    lhs = (w[0] * dx).sum(1) + (w[1] * dy).sum(1)
    scale = np.sqrt((w[0] ** 2).sum(1) + (w[1] ** 2).sum(1)) * np.sqrt((dx ** 2).sum(1) + (dy ** 2).sum(1))
    for pc in ((1, 2) if name == "C2" else (1,)):   # C2: the adjoint takes the fused kernel (1) and the block kernel (2)
        gA, gP, gb, gc, _ = eng.vjp(A, b, c, x, y, s, _t(w[0], dev), _t(w[1], dev), P, make_settings({**args, "lsqr_precond": pc}))
        rhs = (gA.cpu().numpy() * t.A_vals).sum(1) + (gb.cpu().numpy() * t.b).sum(1) + (gc.cpu().numpy() * t.c).sum(1)
        if gP is not None:
            rhs += (gP.cpu().numpy() * t.P_vals).sum(1)
        e = np.abs(lhs - rhs) / scale
        assert e.max() < 1e-6, (name, pc, e.max(), int(e.argmax()))


# ----------------------------------------------------------------------------- the reference's gradcheck programs
def _fd_jvp_check(make, p0, dirs, dev):
    """Central differences of GPU solves along parameter directions vs the GPU JVP (the programs are affine in p)."""
    fwd = {"eps": 1e-12, "max_iters": 400000}
    h = 1e-6
    bt0 = make(p0[None])
    eng = Engine(bt0.structure, dev)
    sol0 = eng.solve(_t(bt0.A_vals, dev), _t(bt0.b, dev), _t(bt0.c, dev), _t(bt0.P_vals, dev), make_settings(fwd))
    assert int(sol0.status[0]) == 1
    for d in dirs:
        t1 = make((p0 + d)[None])
        t = pr.Batch(t1.structure, t1.A_vals - bt0.A_vals, t1.b - bt0.b, t1.c - bt0.c, None if t1.P_vals is None else t1.P_vals - bt0.P_vals)
        dx, dy, _, _ = eng.jvp(_t(bt0.A_vals, dev), _t(bt0.b, dev), _t(bt0.c, dev), sol0.x, sol0.y, sol0.s, _t(t.A_vals, dev), _t(t.b, dev),
                               _t(t.c, dev), _t(bt0.P_vals, dev), _t(t.P_vals, dev), make_settings({**TIGHT, "lsqr_iter_lim": 20000}))
        btp = make(np.stack([p0 + h * d, p0 - h * d]))
        sol = Engine(btp.structure, dev).solve(_t(btp.A_vals, dev), _t(btp.b, dev), _t(btp.c, dev), _t(btp.P_vals, dev), make_settings(fwd))
        assert int((sol.status == 1).sum()) == 2
        for got, val in ((dx, sol.x), (dy, sol.y)):
            fd = ((val[0] - val[1]) / (2 * h)).cpu().numpy()
            got = got[0].cpu().numpy()
            assert (np.abs(fd - got) <= 1e-4 + 1e-3 * np.abs(fd)).all(), (fd, got)


def _sdp_make(Pm):
    iu = np.triu_indices(3)
    Cs = []
    for p in np.atleast_2d(Pm):
        C = np.zeros((3, 3)); C[iu] = p; Cs.append(C + C.T - np.diag(np.diag(C)))
    return ref_sdp_batch(Cs)


def _soc_make(Pm):
    return ref_soc_batch(np.atleast_2d(Pm)[:, :3], np.atleast_2d(Pm)[:, 3])


def test_psd_and_soc_gradcheck_programs_central_differences(cuda_device):
    rng = np.random.default_rng(4)
    C0 = np.array([[2.0, 0.5, 0.1], [0.5, 3.0, 0.2], [0.1, 0.2, 1.5]])
    p_sdp = C0[np.triu_indices(3)].copy()
    _fd_jvp_check(_sdp_make, p_sdp, list(np.eye(6)) + [rng.standard_normal(6)], cuda_device)
    p_soc = np.array([0.5, 0.3, -0.2, 2.0])
    _fd_jvp_check(_soc_make, p_soc, list(np.eye(4)) + [rng.standard_normal(4)], cuda_device)


def _layer_fn(bt, dev, args):
    """(P_eval, q_eval, A_eval) -> (primal, dual) through _CvxpyLayer.apply on the boundary layout of ``bt``."""
    st = bt.structure
    bd = pr.to_boundary(bt)
    P_struct = (st.P_indices, st.P_indptr, (st.n, st.n)) if st.nnzP else None
    ctx = B200_ctx(P_struct, (bd.con_indices, bd.con_ptr, bd.shape), bd.dims, options=args, device=dev)
    cl = type("CL", (), {"solver_ctx": ctx})()
    return bd, (lambda P, q, A: _CvxpyLayer.apply(P, q, A, cl, {}, True, None)[:2])


@pytest.mark.parametrize("make,p0", [(_sdp_make, np.array([2.0, 0.5, 0.1, 3.0, 0.2, 1.5])), (_soc_make, np.array([0.5, 0.3, -0.2, 2.0]))])
def test_gradcheck_with_forward_ad_through_the_layer(make, p0, cuda_device):
    bt = make(p0[None])
    args = {"eps": 1e-12, "max_iters": 400000, **TIGHT, "lsqr_iter_lim": 20000}
    bd, f = _layer_fn(bt, cuda_device, args)
    A = _t(bd.A_eval, cuda_device).requires_grad_(True)
    q = _t(bd.q_eval, cuda_device).requires_grad_(True)
    if bd.P_eval is not None:
        P = _t(bd.P_eval, cuda_device).requires_grad_(True)
        fn, inputs = f, (P, q, A)
    else:
        fn, inputs = (lambda q_, A_: f(None, q_, A_)), (q, A)
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-4, rtol=1e-3, check_forward_ad=True, check_undefined_grad=False)


# ----------------------------------------------------------------------------- the layer: forward AD vs the reverse-mode Jacobian
def _fwd_ad(f, inputs, tangents):
    with fwAD.dual_level():
        duals = [None if x is None else fwAD.make_dual(x, t) for x, t in zip(inputs, tangents)]
        outs = f(*duals)
        return [fwAD.unpack_dual(o).tangent for o in outs]


def _jac_times(f, inputs, tangents):
    idx = [k for k, x in enumerate(inputs) if x is not None]

    def g(*xs):
        full = list(inputs)
        for k, x in zip(idx, xs):
            full[k] = x
        return f(*full)

    J = torch.autograd.functional.jacobian(g, tuple(inputs[k] for k in idx))
    res = []
    for o, Jo in enumerate(J):
        acc = 0
        for jj, k in enumerate(idx):
            x = inputs[k]
            acc = acc + (Jo[jj].reshape(-1, x.numel()) @ tangents[k].reshape(-1).to(Jo[jj])).reshape(Jo[jj].shape[:Jo[jj].dim() - x.dim()])
        res.append(acc)
    return res


def _close(a, b, tol=1e-6):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert (a - b).abs().max() <= tol * max(1.0, b.abs().max()), ((a - b).abs().max(), b.abs().max())


@pytest.mark.parametrize("where", ["device", "pinned", "pageable"])
@pytest.mark.parametrize("unbatched", [False, True])
def test_layer_forward_ad_equals_reverse_jacobian(where, unbatched, cuda_device):
    bt = pr.dense_qp(1 if unbatched else 3, 8, 14, 3, seed=6)
    args = {"eps": 1e-11, "max_iters": 200000, **TIGHT}
    bd, f = _layer_fn(bt, cuda_device, args)
    g = torch.Generator().manual_seed(1)

    def put(a):
        x = torch.as_tensor(np.ascontiguousarray(a[:, 0] if unbatched else a), dtype=torch.float64)
        return x.to(cuda_device) if where == "device" else (x.pin_memory() if where == "pinned" else x)

    inputs = [put(bd.P_eval), put(bd.q_eval), put(bd.A_eval)]
    tangents = [torch.randn(x.shape, dtype=torch.float64, generator=g).to(x.device) for x in inputs]
    got = _fwd_ad(f, inputs, tangents)
    for o, ref in zip(got, _jac_times(f, inputs, tangents)):
        assert o.device == inputs[0].device
        _close(o, ref)


def _fused_setup(bt, dev, args):
    from tests.util import fake_param_prob

    problem, params = fake_param_prob(bt)
    pp = problem["param_prob"]
    ctx = get_solver_ctx("B200", pp, problem["dims"], {}, args)
    ctx.device = dev
    cl = type("CL", (), {"solver_ctx": ctx})()
    B = bt.B
    p_stack = torch.as_tensor(np.concatenate([p.T for p in params] + [np.ones((1, B))]), dtype=torch.float64, device=dev)
    return p_stack, (lambda ps: _CvxpyLayerFused.apply(ps, cl, {}, True, None)[:2])


def test_fused_layer_forward_ad_equals_reverse_jacobian(cuda_device):
    bt = pr.dense_qp(3, 8, 14, 3, seed=7)
    p_stack, f = _fused_setup(bt, cuda_device, {"eps": 1e-11, "max_iters": 200000, **TIGHT})
    tp = torch.randn(p_stack.shape, dtype=torch.float64, device=cuda_device)
    tp[-1] = 0.0
    for o, ref in zip(_fwd_ad(f, [p_stack], [tp]), _jac_times(f, [p_stack], [tp])):
        _close(o, ref)


@pytest.mark.parametrize("requires_grad", [True, False])
def test_registered_fused_layer_forward_ad(requires_grad, cuda_device, monkeypatch):
    """register(fuse=True) with a native P: parameters -> layer_io prologue -> _CvxpyLayerFused -> layer_io epilogue, all forward
    AD.  Dual inputs that do not require grad still get their tangent (the layer's needs_grad is False for them)."""
    from cvxpylayers_b200 import interface as itf
    from tests.util import fake_param_prob, install_fake_cvxpylayers

    fake = install_fake_cvxpylayers(monkeypatch)
    bt = pr.dense_qp(4, 8, 14, 3, seed=4)
    problem, params = fake_param_prob(bt)
    itf.register(fuse=True)
    layer = fake.tl.CvxpyLayer(problem, [], [], solver="B200", solver_args={"eps": 1e-11, "max_iters": 200000, **TIGHT})
    layer.ctx.solver_ctx.device = cuda_device
    th = [torch.tensor(p, device=cuda_device) for p in params]
    g = torch.Generator().manual_seed(2)
    tg = [torch.randn(p.shape, dtype=torch.float64, generator=g).to(cuda_device) for p in th]
    with fwAD.dual_level():
        duals = [fwAD.make_dual(p.requires_grad_(requires_grad), t) for p, t in zip(th, tg)]
        outs = [fwAD.unpack_dual(o).tangent for o in layer(*duals)]
    ref = _jac_times(lambda *ps: layer(*ps), [p.detach() for p in th], tg)
    for o, r in zip(outs, ref):
        _close(o, r)


def test_gp_prologue_and_epilogue_forward_ad_equal_the_reference_chains(cuda_device):
    """layer_io's _FlattenParams (GP log) and _GatherCols (GP exp) under forward AD vs forward AD of plain torch chains."""
    from types import SimpleNamespace

    from cvxpylayers_b200 import layer_io

    dev, B = cuda_device, 5
    g = torch.Generator().manual_seed(3)
    params = ((torch.rand((B, 3, 2), dtype=torch.float64, generator=g) + 0.5).to(dev), (torch.rand(4, dtype=torch.float64, generator=g) + 0.5).to(dev))
    tans = [torch.randn(p.shape, dtype=torch.float64, generator=g).to(dev) for p in params]
    lctx = SimpleNamespace(batch_sizes=[B, 0], user_order_to_col_order=(1, 0), gp=True, gp_log_mask=(False, True))

    def ref_flatten(p0, p1):
        f0 = p0.permute(0, 2, 1).reshape(B, -1)          # Fortran order of each instance's 3 x 2 block
        f1 = torch.log(p1).unsqueeze(0).expand(B, 4)
        return torch.cat([f1, f0, torch.ones((B, 1), dtype=torch.float64, device=dev)], -1).T

    with fwAD.dual_level():
        d = [fwAD.make_dual(p, t) for p, t in zip(params, tans)]
        got = fwAD.unpack_dual(layer_io.flatten_and_batch_params(tuple(d), lctx, (B,))).tangent
        ref = fwAD.unpack_dual(ref_flatten(*d)).tangent
    assert torch.allclose(got, ref, rtol=1e-13, atol=1e-13)
    primal = torch.randn((B, 12), dtype=torch.float64, generator=g).to(dev)
    tprimal = torch.randn((B, 12), dtype=torch.float64, generator=g).to(dev)
    rctx = SimpleNamespace(gp=True, var_recover=[SimpleNamespace(primal=slice(2, 8), dual=None, shape=(2, 3), source="primal", unpack_fn="reshape")])
    with fwAD.dual_level():
        dp = fwAD.make_dual(primal, tprimal)
        got = fwAD.unpack_dual(layer_io.recover_results(dp, dp, rctx, (B,))[0]).tangent
        ref = fwAD.unpack_dual(torch.exp(dp[:, 2:8].reshape(B, 3, 2).permute(0, 2, 1))).tangent
    assert torch.allclose(got, ref, rtol=1e-13, atol=1e-13)


def test_zero_tangent_is_zero_with_no_lsqr_iterations(cuda_device):
    bt = pr.CONFIGS["C3"](B=8)
    st, dev = bt.structure, cuda_device
    eng = Engine(st, dev)
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    sol = eng.solve(A, b, c, None, make_settings({"eps": 1e-8}))
    z = lambda *shape: torch.zeros(shape, dtype=torch.float64, device=dev)  # noqa: E731
    dx, dy, ds, its = eng.jvp(A, b, c, sol.x, sol.y, sol.s, z(8, st.nnzA), z(8, st.m), z(8, st.n), settings=make_settings({"lsqr_precond": 1}))
    assert not dx.any() and not dy.any() and not ds.any() and not its.any()
