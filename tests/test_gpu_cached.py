"""Cached set-up (SURVEY.md 8f.2, second half): equilibration + factorisation kept across calls while A and P do not change
(the reference's template: the one-time ``setup()`` under ``PA_is_constant``, interfaces/moreau_if.py:233-256,316-320).
The cached path must be the SAME algorithm minus the recomputation: bit-identical to the uncached warm solve whenever the
cached scale is the initial one, and equal to the oracle started at the cached scale otherwise."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from cvxpylayers_b200.interface import B200_ctx, _CvxpyLayer
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def _t(a, dev):
    return torch.tensor(np.ascontiguousarray(a), device=dev)


def _same(a, b):
    return all(torch.equal(getattr(a, k), getattr(b, k)) for k in ("x", "y", "s", "status", "iters"))


# the compile-time geometry and two runtime ones at B = 96; then, at B = 16 (the oracle checks below run on the CPU), shape
# classes of tests/tiled_shapes.py: 4-row K^-1 tiles at the shared-memory limit, n > m, the compile-time geometry at its widest
# padding with odd m n.  (The classes with m >> n are not here: dense_qp plants more active rows than variables there, and the
# perturbed b below then has no feasible point; tests/test_gpu_tiled_shapes.py runs them on planted batches.)
@pytest.mark.parametrize("shape", [(100, 200, 50, 96), (80, 200, 40, 96), (75, 190, 30, 96),
                                   (110, 136, 30, 16), (101, 93, 10, 16), (91, 197, 20, 16)])
def test_cached_setup_is_the_uncached_algorithm(cuda_device, shape):
    n, m, z, B = shape
    dev = cuda_device
    bt = pr.dense_qp(B, n, m, z, seed=21)
    st = bt.structure
    eng = Engine(st, dev)
    assert "register-tiled" in eng.path_info()["fwd"]
    A, P, b, c = _t(bt.A_vals, dev), _t(bt.P_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    args = dict(eps=1e-6, max_iters=100000)
    S = make_settings(args)
    cache = eng.new_cache(B)
    assert cache is not None and cache.numel() * 8 == eng.cache_bytes(B)
    stride = cache.numel() // B
    plain = eng.solve(A, b, c, P, S)
    fill = eng.solve(A, b, c, P, S, cache=cache, reuse=False)
    assert _same(plain, fill)                                        # writing the cache does not touch the algorithm
    hdr = cache.view(B, stride)[:, :3].cpu().numpy()
    assert (hdr[:, 1] == 1.0).all() and (hdr[:, 2] == S.rho_x).all()
    fresh = eng.solve(A, b, c, P, S, cache=eng.new_cache(B), reuse=True)
    assert _same(plain, fresh)                                       # reuse on a zero-filled cache rebuilds every record

    rng = np.random.default_rng(3)
    b2 = bt.b + 1e-3 * rng.standard_normal(bt.b.shape)
    c2 = bt.c + 1e-3 * rng.standard_normal(bt.c.shape)
    b2t, c2t = _t(b2, dev), _t(c2, dev)
    warm = (plain.x.clone(), plain.y.clone(), plain.s.clone())
    ref_w = eng.solve(A, b2t, c2t, P, S, warm=warm)                   # uncached, warm
    got = eng.solve(A, b2t, c2t, P, S, warm=warm, cache=cache, reuse=True)
    assert int((got.status == 1).sum()) == B
    kept = hdr[:, 0] == S.scale                                        # records whose factorisation is at the initial scale
    assert kept.any()
    ki = torch.tensor(np.nonzero(kept)[0], device=dev)
    for k in ("x", "y", "s", "iters"):
        assert torch.equal(getattr(got, k)[ki], getattr(ref_w, k)[ki]), k   # bit-identical: same Kinv, same E / D, same loop
    # re-scaled records: the solve starts at the cached scale; the oracle told the same thing agrees
    moved = np.nonzero(~kept)[0][:6]
    for i in moved:
        xo, yo, so, sto, ito = orc.solve_batch(st, bt.A_vals[i:i + 1], b2[i:i + 1], c2[i:i + 1], bt.P_vals[i:i + 1],
                                               warm=tuple(w[i:i + 1].cpu().numpy() for w in warm), scale=float(hdr[i, 0]), **args)
        assert sto[0] == 1 and abs(int(got.iters[i]) - int(ito[0])) <= 25
        assert np.abs(got.x[i].cpu().numpy() - xo[0]).max() < 1e-5
    # whatever the route, the answer is the optimum of the new data (cold oracle, tight eps): as close to it as the uncached solve
    xc, yc, sc, stc, _ = orc.solve_batch(st, bt.A_vals, b2, c2, bt.P_vals, eps=1e-9, max_iters=200000)
    assert (stc == 1).all()
    for got_, ref_, opt in ((got.x, ref_w.x, xc), (got.y, ref_w.y, yc)):
        e_got, e_ref = np.abs(got_.cpu().numpy() - opt).max(), np.abs(ref_.cpu().numpy() - opt).max()
        assert e_got < 1e-2 and e_got <= 2.0 * e_ref + 1e-6, (e_got, e_ref)   # (eps 1e-6 on residuals: ~1e-3 on the duals)
    # a third call: records refreshed by re-scalings of the second call are valid too
    third = eng.solve(A, b2t, c2t, P, S, warm=got, cache=cache, reuse=True)
    assert int((third.status == 1).sum()) == B and int(third.iters.max()) <= 25


def test_cached_setup_without_quadratic_term(cuda_device):
    """An LP of the register-tiled shape (no P): the cached path has nothing to load but Kinv.  (90 x 170: the tile grid
    keeps at least half of the CTA's threads busy, which the register-tiled kernel requires.)"""
    B, dev = 48, cuda_device
    bt = pr.dense_qp(B, 90, 170, 20, seed=4, with_P=False)
    st = bt.structure
    eng = Engine(st, dev)
    assert "register-tiled" in eng.path_info()["fwd"]
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    S = make_settings(dict(eps=1e-6, max_iters=200000))
    cache = eng.new_cache(B)
    assert cache is not None and cache.numel() * 8 == eng.cache_bytes(B)
    one = eng.solve(A, b, c, None, S, cache=cache, reuse=False)
    two = eng.solve(A, b, c, None, S, warm=one, cache=cache, reuse=True)
    ref = eng.solve(A, b, c, None, S, warm=one)
    hdr = cache.view(B, -1)[:, 0].cpu().numpy()
    assert (hdr == S.scale).any()
    ki = torch.tensor(np.nonzero(hdr == S.scale)[0], device=dev)
    assert torch.equal(two.x[ki], ref.x[ki]) and torch.equal(two.iters[ki], ref.iters[ki])


def test_structures_without_a_cached_path_say_so(cuda_device):
    bt = pr.socp_portfolio(4, seed=1)
    eng = Engine(bt.structure, cuda_device)
    assert eng.cache_bytes(4) == 0 and eng.new_cache(4) is None
    dev = cuda_device
    with pytest.raises(Exception, match="cache"):
        eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev) if bt.P_vals is not None else None,
                  make_settings({}), cache=torch.zeros(64, dtype=torch.float64, device=dev), reuse=True)


def test_layer_reuses_the_setup_when_asked(cuda_device):
    """{"reuse_setup": True, "warm_start": True}: the training-loop configuration.  Same results as the plain layer; the cache
    is filled by the first call and valid afterwards; forward + backward still agree with the oracle's gradient."""
    dev = cuda_device
    bt = pr.dense_qp(64, 100, 200, 50, seed=8)
    st = bt.structure
    bd = pr.to_boundary(bt)

    def layer(**opt):
        ctx = B200_ctx((st.P_indices, st.P_indptr, (st.n, st.n)), (bd.con_indices, bd.con_ptr, bd.shape), bd.dims, options=opt)
        return ctx, SimpleNamespace(solver_ctx=ctx)

    base = dict(eps=1e-7, max_iters=100000, lsqr_precond=2)
    ctx_c, cl_c = layer(**base, reuse_setup=True, warm_start=True)
    ctx_p, cl_p = layer(**base, warm_start=True)
    A, P = _t(bd.A_eval, dev), _t(bd.P_eval, dev)
    rng = np.random.default_rng(0)
    q = bd.q_eval.copy()
    for step in range(3):
        outs = []
        for cl in (cl_c, cl_p):
            qt = _t(q, dev).requires_grad_(True)
            primal, dual, _, _ = _CvxpyLayer.apply(P, qt, A, cl, {}, True, None)
            (primal.square().sum() + dual.sum()).backward()
            outs.append((primal.detach(), dual.detach(), qt.grad.clone()))
        for a_, b_, tol in zip(outs[0], outs[1], (1e-5, 1e-4, 1e-4)):
            assert float((a_ - b_).abs().max()) < tol * max(1.0, float(b_.abs().max()))
        q[:-1] += 1e-3 * rng.standard_normal(q[:-1].shape)
    cache = ctx_c._setup_cache[(dev, bt.B)]
    assert cache is not None and bool((cache.view(bt.B, -1)[:, 1] == 1.0).all())
    assert not hasattr(ctx_p, "_setup_cache")


def test_fused_layer_with_constant_matrices_caches_by_default(cuda_device):
    """The reference's `PA_is_constant` scenario end to end: the layer's parameters are b and c, A and P are constants in the last
    column of the parameter maps.  The context detects it, `_CvxpyLayerFused` solves with the cached set-up from the second call on,
    and solutions + parameter gradients equal those of a context with the cache switched off."""
    import scipy.sparse as sp

    from cvxpylayers_b200.interface import _CvxpyLayerFused

    dev, B = cuda_device, 40
    b0 = pr.dense_qp(1, 100, 200, 50, seed=2)
    st = b0.structure
    rng = np.random.default_rng(5)
    bs = pr.plant(st, np.tile(b0.A_vals, (B, 1)), np.tile(b0.P_vals, (B, 1)), rng, name="shared", active_frac=0.2)
    bd = pr.to_boundary(bs)
    nA, nb, n = st.nnzA, bd.A_eval.shape[0] - st.nnzA, st.n
    P1 = nb + n + 1
    A_map = sp.csr_matrix((np.concatenate([bd.A_eval[:nA, 0], np.ones(nb)]),
                           (np.arange(nA + nb), np.concatenate([np.full(nA, P1 - 1), np.arange(nb)]))), shape=(nA + nb, P1))
    q_map = sp.csr_matrix((np.ones(n), (np.arange(n), nb + np.arange(n))), shape=(n + 1, P1))
    P_map = sp.csr_matrix((bd.P_eval[:, 0], (np.arange(bd.P_eval.shape[0]), np.full(bd.P_eval.shape[0], P1 - 1))), shape=(bd.P_eval.shape[0], P1))
    p0 = np.concatenate([bd.A_eval[nA:], bd.q_eval[:n], np.ones((1, B))])

    def layer(**opt):
        ctx = B200_ctx((st.P_indices, st.P_indptr, (st.n, st.n)), (bd.con_indices, bd.con_ptr, bd.shape), bd.dims,
                       options=dict(eps=1e-7, max_iters=100000, lsqr_precond=2, **opt))
        ctx.set_param_maps(A_map, q_map, P_map)
        return ctx, SimpleNamespace(solver_ctx=ctx)

    ctx_auto, cl_auto = layer()
    ctx_off, cl_off = layer(reuse_setup=False)
    assert ctx_auto.PA_is_constant and ctx_off.PA_is_constant
    for step in range(3):
        p = p0.copy()
        p[:-1] += 1e-3 * step * rng.standard_normal(p[:-1].shape)
        res = []
        for cl in (cl_auto, cl_off):
            pt = _t(p, dev).requires_grad_(True)
            primal, dual, _, _ = _CvxpyLayerFused.apply(pt, cl, {}, True, None)
            (primal.square().sum() + dual.sum()).backward()
            res.append((primal.detach(), dual.detach(), pt.grad.clone()))
        for a_, b_, tol in zip(res[0], res[1], (1e-6, 1e-5, 1e-5)):
            assert float((a_ - b_).abs().max()) <= tol * max(1.0, float(b_.abs().max()))
        assert float(res[0][2][-1].abs().max()) == 0.0            # the constant's row carries no gradient
    if step == 0:
        assert np.abs(res[0][0].cpu().numpy() - bs.x_star).max() < 1e-4
    cache = ctx_auto._setup_cache[(dev, B)]
    assert bool((cache.view(B, -1)[:, 1] == 1.0).all()) and not getattr(ctx_off, "_setup_cache", {}).get((dev, B))
