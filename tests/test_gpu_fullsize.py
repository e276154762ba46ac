"""GPU parity at the BASELINE.json batch sizes and the parity holes VERDICT round 1 named:

* every BASELINE config at its real batch (C2 4096, C3 2048, C4 512 forward AND backward at n=1000/m=2000, C5 256):
  work-queue, wave and multi-CTA/SM effects are only exercised there;
* the gradient a user actually gets -- GPU adjoint at the GPU's OWN solution -- against the oracle's pipeline;
* the reference's own finite-difference programs (PSD: tests/test_torch.py:233-248, SOC:
  tests/test_dual_variables.py:346-369, atol 1e-4 / rtol 1e-3) through the CUDA path;
* every LSQR variant against an EXACT dense least-squares solve of diffcp's adjoint system, which is what justifies the
  tolerance of the reference-semantics recurrence (lsqr_precond = 0).

All through the C ABI (cvxpylayers_b200.engine -> libbcone.so); the oracle is the checker only.
"""
import os

import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from oracle import np_ref
from oracle import oracle as orc
from tests.util import ref_sdp_batch, ref_soc_batch

pytestmark = pytest.mark.gpu

NT = len(os.sched_getaffinity(0))   # oracle threads: all host cores (torchrun / pytest may pin OMP_NUM_THREADS)


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _rel_rows(a, b):
    """per-instance relative error max|a_i - b_i| / max|b_i|"""
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return np.abs(a - b).reshape(a.shape[0], -1).max(1) / np.maximum(np.abs(b).reshape(b.shape[0], -1).max(1), 1e-30)


def _gpu_pipeline(bt, dev, fwd_args, bwd_args, dx, dy):
    eng = Engine(bt.structure, dev)
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    sol = eng.solve(A, b, c, P, make_settings(fwd_args))
    g = eng.vjp(A, b, c, sol.x, sol.y, sol.s, _t(dx, dev), _t(dy, dev), P, make_settings(bwd_args))
    torch.cuda.synchronize()
    return eng, sol, g


def _certified(bt, x, y, s, eps, idx):
    for i in idx:
        P = bt.P_dense(i) if bt.P_vals is not None else None
        r = np_ref.kkt_residuals(bt.A_dense(i), P, bt.b[i], bt.c[i], x[i], y[i], s[i])
        assert np_ref.is_converged(r, eps, eps, 1.001), (i, r)


# ----------------------------------------------------------------------------- C3 and C5 at their BASELINE batch
@pytest.mark.parametrize("name,B", [("C3", 2048), ("C5", 256)])
def test_full_batch_forward_and_own_solution_gradient(name, B, cuda_device):
    bt = pr.CONFIGS[name](B=B)
    st, dev = bt.structure, cuda_device
    eps = 1e-9
    fwd = {"eps": eps, "max_iters": 200000}
    bwd = {"lsqr_precond": 1, "lsqr_iter_lim": 40 * (st.n + st.m + 1)}
    rng = np.random.default_rng(5)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    eng, sol, (dA, dP, db, dc, its) = _gpu_pipeline(bt, dev, fwd, bwd, dx, dy)
    assert int((sol.status == 1).sum()) == B, torch.unique(sol.status, return_counts=True)
    x, y, s = sol.x.cpu().numpy(), sol.y.cpu().numpy(), sol.s.cpu().numpy()
    _certified(bt, x, y, s, eps, range(0, B, max(1, B // 64)))
    xo, yo, so, sto, ito = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, bt.P_vals, nthreads=NT, **fwd)
    assert (sto == 1).all()
    # same algorithm on the same data: solutions agree far inside the solver tolerance, iteration counts track
    assert np.abs(x - xo).max() <= 1e-6 * max(1.0, np.abs(xo).max())
    assert np.abs(y - yo).max() <= 1e-6 * max(1.0, np.abs(yo).max())
    it_g = sol.iters.cpu().numpy()
    assert abs(it_g.mean() - ito.mean()) <= 0.05 * ito.mean() + 5, (it_g.mean(), ito.mean())
    # (1) same inputs into both adjoints: 1e-4 relative on EVERY instance
    gA, gP, gb, gc, _ = eng.vjp(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(xo, dev), _t(yo, dev), _t(so, dev), _t(dx, dev), _t(dy, dev),
                                _t(bt.P_vals, dev), make_settings(bwd))
    rA, rP, rb, rc, _ = orc.vjp_batch(st, bt.A_vals, bt.b, bt.c, xo, yo, so, dx, dy, bt.P_vals, nthreads=NT, **bwd)
    for g_, r_ in ((gA, rA), (gb, rb), (gc, rc)):
        e = _rel_rows(g_, r_)
        assert e.max() < 1e-4, (name, e.max(), int(e.argmax()))
    # (2) the gradient the user gets: GPU adjoint at the GPU's own solution vs the oracle's whole pipeline.  Two 1e-9 solutions
    # of the same instance differ by ~1e-9 and the adjoint amplifies that by the conditioning of the instance: 1e-4 holds for
    # all but the odd ill-conditioned instance of 2048 (measured worst case 1.2e-4), hence the quantile + a hard cap
    for g_, r_ in ((dA, rA), (db, rb), (dc, rc)):
        e = _rel_rows(g_, r_)
        assert (e < 1e-4).mean() >= 0.998 and e.max() < 1e-3 and np.median(e) < 1e-6, (name, "own solution", e.max(), int(e.argmax()), np.median(e))


# ----------------------------------------------------------------------------- C2: the user's gradient at the headline batch
def test_c2_full_batch_gradient_from_own_solution(cuda_device):
    """B = 4096 through solve + adjoint (block-preconditioned LSQR, what bench.py times) at eps 1e-8; the oracle's
    pipeline (its own solve + plain-semantics adjoint with the equilibrated LSQR) on a 256-instance sample."""
    B, k = 4096, 256
    bt = pr.config_c2(B=B, seed=2)
    st, dev = bt.structure, cuda_device
    fwd = {"eps": 1e-8, "max_iters": 100000, "adaptive_check": 1}
    rng = np.random.default_rng(6)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    eng, sol, (dA, dP, db, dc, its) = _gpu_pipeline(bt, dev, fwd, {"lsqr_precond": 2}, dx, dy)
    assert int((sol.status == 1).sum()) == B
    assert np.abs(sol.x.cpu().numpy() - bt.x_star).max() < 1e-5
    sub = bt.select(slice(0, k))
    xo, yo, so, sto, _ = orc.solve_batch(st, sub.A_vals, sub.b, sub.c, sub.P_vals, nthreads=NT, eps=1e-8, max_iters=100000)
    assert (sto == 1).all()
    rA, rP, rb, rc, _ = orc.vjp_batch(st, sub.A_vals, sub.b, sub.c, xo, yo, so, dx[:k], dy[:k], sub.P_vals, nthreads=NT, lsqr_precond=1,
                                      lsqr_iter_lim=20000)
    for g_, r_ in ((dA[:k], rA), (dP[:k], rP), (db[:k], rb), (dc[:k], rc)):
        e = _rel_rows(g_, r_)
        assert e.max() < 1e-4, (e.max(), int(e.argmax()))
    # block solver: how many instances fell back to the equilibrated LSQR (reported by bench.py as well)
    assert int((its.cpu().numpy() > 40).sum()) <= B // 20


# ----------------------------------------------------------------------------- C4 at n = 1000, m = 2000, B = 512
def test_c4_full_batch_forward_and_backward(cuda_device):
    B = 512
    bt = pr.CONFIGS["C4"](B=B)
    st, dev = bt.structure, cuda_device
    eps = 1e-4
    eng = Engine(st, dev)
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    sol = eng.solve(A, b, c, None, make_settings({"eps": eps, "max_iters": 100000}))
    torch.cuda.synchronize()
    assert int((sol.status == 1).sum()) == B, (torch.unique(sol.status, return_counts=True), sol.iters.max())
    x, y, s = sol.x.cpu().numpy(), sol.y.cpu().numpy(), sol.s.cpu().numpy()
    # certificate on the original data for all 512 instances (batched CSR products in NumPy)
    Ax, ATy = pr._apply_A(st, bt.A_vals, x), pr._apply_AT(st, bt.A_vals, y)
    mx = lambda a: np.abs(a).max(1)  # noqa: E731
    rp, rd = mx(Ax + s - bt.b), mx(ATy + bt.c)
    ctx, bty = (bt.c * x).sum(1), (bt.b * y).sum(1)
    assert (rp <= 1.001 * (eps + eps * np.maximum(np.maximum(mx(Ax), mx(s)), mx(bt.b)))).all()
    assert (rd <= 1.001 * (eps + eps * np.maximum(mx(ATy), mx(bt.c)))).all()
    assert (np.abs(ctx + bty) <= 1.001 * (eps + eps * np.maximum(np.abs(ctx), np.abs(bty)))).all()
    assert (s >= -1e-12).all() and (y >= -1e-12).all() and np.abs((s * y).sum(1)).max() < 1e-8
    # LP: the objective value is unique even where x is not -- compare with the planted optimum
    opt = (bt.c * bt.x_star).sum(1)
    assert (np.abs(ctx - opt) <= 50 * eps * np.maximum(1.0, np.abs(opt))).all()
    # oracle forward on a sample (its dense n x n Cholesky makes the full batch a minutes-long CPU job)
    k = 8
    sub = bt.select(slice(0, k))
    xo, yo, so, sto, ito = orc.solve_batch(st, sub.A_vals, sub.b, sub.c, None, nthreads=NT, eps=eps, max_iters=100000)
    assert (sto == 1).all()
    assert np.abs((sub.c * xo).sum(1) - ctx[:k]).max() <= 50 * eps * max(1.0, np.abs(opt[:k]).max())
    # backward at full size, both adjoints fed the planted (exact) optimum: a non-degenerate vertex, unique derivative
    rng = np.random.default_rng(7)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    # (tight LSQR tolerances: a handful of the 512 planted vertices have an ill-conditioned active basis, where stopping
    #  at the default atol = btol = 1e-8 leaves two correct implementations 1e-2 apart -- measured, instance 261)
    bwd = {"lsqr_precond": 1, "lsqr_iter_lim": 4 * (st.n + st.m + 1), "lsqr_atol": 1e-13, "lsqr_btol": 1e-13}
    gA, gP, gb, gc, its = eng.vjp(A, b, c, _t(bt.x_star, dev), _t(bt.y_star, dev), _t(bt.s_star, dev), _t(dx, dev), _t(dy, dev), None, make_settings(bwd))
    torch.cuda.synchronize()
    rA, rP, rb, rc, rits = orc.vjp_batch(st, bt.A_vals, bt.b, bt.c, bt.x_star, bt.y_star, bt.s_star, dx, dy, None, nthreads=NT, **bwd)
    for g_, r_ in ((gA, rA), (gb, rb), (gc, rc)):
        e = _rel_rows(g_, r_)
        assert e.max() < 1e-4, (e.max(), int(e.argmax()), its.max(), rits.max())


# ----------------------------------------------------------------------------- the reference's gradcheck programs on the GPU
def _fd_through_gpu(make, p0, dev, dx, dy, fwd, h=1e-6):
    """Central differences of <x, dx> + <y, dy> in every parameter: the 2 len(p0) perturbed programs are ONE batch."""
    P = []
    for k in range(p0.size):
        for sgn in (+1, -1):
            p = p0.copy(); p[k] += sgn * h
            P.append(p)
    bt = make(np.stack(P))
    eng = Engine(bt.structure, dev)
    sol = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings(fwd))
    assert int((sol.status == 1).sum()) == bt.B
    val = (sol.x.cpu().numpy() @ dx + sol.y.cpu().numpy() @ dy).reshape(p0.size, 2)
    return (val[:, 0] - val[:, 1]) / (2 * h)


@pytest.mark.parametrize("precond", [0, 1])
def test_psd_gradcheck_program_on_gpu(precond, cuda_device):
    C0 = np.array([[2.0, 0.5, 0.1], [0.5, 3.0, 0.2], [0.1, 0.2, 1.5]])
    iu = np.triu_indices(3)

    def make(Pm):   # rows of Pm = the 6 free entries of the symmetric parameter C
        Cs = []
        for p in np.atleast_2d(Pm):
            C = np.zeros((3, 3)); C[iu] = p; Cs.append(C + C.T - np.diag(np.diag(C)))
        return ref_sdp_batch(Cs)

    p0 = C0[iu].copy()
    bt = make(p0)
    st, dev = bt.structure, cuda_device
    fwd = {"eps": 1e-12, "max_iters": 400000}
    rng = np.random.default_rng(4)
    dx, dy = rng.standard_normal(st.n), rng.standard_normal(st.m)
    eng, sol, (dA, dP, db, dc, its) = _gpu_pipeline(bt, dev, fwd, {"lsqr_precond": precond, "lsqr_iter_lim": 20000, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12},
                                                     dx[None], dy[None])
    assert int(sol.status[0]) == 1
    lam, V = np.linalg.eigh(C0)
    assert np.abs(pr.svec_to_mat(sol.x.cpu().numpy()[0], 3) - np.outer(V[:, 0], V[:, 0])).max() < 1e-7
    svec_pos = {(0, 0): 0, (1, 0): 1, (2, 0): 2, (1, 1): 3, (2, 1): 4, (2, 2): 5}
    dcn = dc.cpu().numpy()[0]
    grads = np.array([dcn[svec_pos[(max(i, j), min(i, j))]] * (1.0 if i == j else np.sqrt(2.0)) for i, j in zip(*iu)])
    fd = _fd_through_gpu(make, p0, dev, dx, dy, fwd)
    assert (np.abs(fd - grads) <= 1e-4 + 1e-3 * np.abs(fd)).all(), (fd, grads)


@pytest.mark.parametrize("precond", [0, 1])
def test_soc_gradcheck_program_on_gpu(precond, cuda_device):
    p0 = np.array([0.5, 0.3, -0.2, 2.0])
    make = lambda Pm: ref_soc_batch(np.atleast_2d(Pm)[:, :3], np.atleast_2d(Pm)[:, 3])  # noqa: E731
    bt = make(p0)
    st, dev = bt.structure, cuda_device
    fwd = {"eps": 1e-12, "max_iters": 400000}
    for dx, dy in ((np.zeros(3), np.ones(4)), (np.array([1.0, -2.0, 0.5]), np.array([0.3, -1.0, 2.0, 0.7]))):
        eng, sol, (dA, dP, db, dc, its) = _gpu_pipeline(bt, dev, fwd, {"lsqr_precond": precond, "lsqr_iter_lim": 20000, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12},
                                                         dx[None], dy[None])
        assert int(sol.status[0]) == 1
        grads = np.concatenate([dc.cpu().numpy()[0], db.cpu().numpy()[0, :1]])
        fd = _fd_through_gpu(make, p0, dev, dx, dy, fwd)
        assert (np.abs(fd - grads) <= 1e-4 + 1e-3 * np.abs(fd)).all(), (fd, grads)


# ----------------------------------------------------------------------------- every LSQR variant vs an exact least-squares solve
def _exact_adjoint(bt, i, x, y, s, dx, dy):
    """diffcp's adjoint with an explicit dense M (cone Jacobian column by column from the oracle, so exponential cones
    are covered too) and numpy.linalg.lstsq."""
    st = bt.structure
    n, m = st.n, st.m
    N = n + m + 1
    A = bt.A_dense(i)
    Pm = bt.P_dense(i) if bt.P_vals is not None else np.zeros((n, n))
    v = y - s
    D = np.stack([orc.dproj_dual_cone(st, v, e) for e in np.eye(m)], axis=1)
    piy = orc.proj_dual_cone(st, v)
    Px = Pm @ x
    DQ = np.zeros((N, N))
    DQ[:n, :n] = Pm; DQ[:n, n:n + m] = A.T; DQ[:n, -1] = bt.c[i]
    DQ[n:n + m, :n] = -A; DQ[n:n + m, -1] = bt.b[i]
    DQ[-1, :n] = -(2 * Px + bt.c[i]); DQ[-1, n:n + m] = -bt.b[i]; DQ[-1, -1] = x @ Px
    Dpi = np.eye(N); Dpi[n:n + m, n:n + m] = D
    M = (DQ - np.eye(N)) @ Dpi + np.eye(N)
    dz = np.concatenate([dx, D.T @ dy, [-(x @ dx + y @ dy)]])
    r = np.linalg.lstsq(M.T, dz, rcond=None)[0]
    rx, ry, rt = r[:n], r[n:n + m], r[-1]
    rows = np.repeat(np.arange(m), np.diff(st.A_indptr))
    dA = (np.outer(ry, x) - np.outer(piy, rx))[rows, st.A_indices]
    return dA, piy * rt - ry, x * rt - rx


@pytest.mark.parametrize("name,B", [("C1", 4), ("C2", 4), ("C3", 4), ("C5", 3), ("EXP", 4)])
def test_lsqr_variants_against_exact_least_squares(name, B, cuda_device):
    """The two deviations the engine ships (lsqr_precond 1 = diagonally equilibrated, 2 = KKT-block preconditioned) hit
    the EXACT least-squares solution of the reference's system to 1e-4 -- north_star's tolerance -- on every config.
    The reference-semantics recurrence (lsqr_precond 0: SciPy/diffcp LSQR, atol = btol = 1e-8, 2N cap lifted here) is
    measured against the same exact solution on the GPU and on the oracle: where it misses 1e-4 both implementations
    miss it by the same amount, i.e. the loss is the stopping rule's (it fires on an ill-conditioned system long
    before the iterate is 1e-4 accurate), not an implementation difference."""
    bt = pr.CONFIGS[name](B=B)
    st, dev = bt.structure, cuda_device
    xo, yo, so, sto, _ = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-11, max_iters=400000)
    assert (sto == 1).all()
    rng = np.random.default_rng(5)
    dx, dy = rng.standard_normal(xo.shape), rng.standard_normal(yo.shape)
    exact = [_exact_adjoint(bt, i, xo[i], yo[i], so[i], dx[i], dy[i]) for i in range(B)]
    eA, eb, ec = (np.stack([e[k] for e in exact]) for k in range(3))
    eng = Engine(st, dev)
    lim = 40 * (st.n + st.m + 1)
    err = {}
    for pc in (0, 1, 2):
        g = eng.vjp(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(xo, dev), _t(yo, dev), _t(so, dev), _t(dx, dev), _t(dy, dev), _t(bt.P_vals, dev),
                    make_settings({"lsqr_precond": pc, "lsqr_iter_lim": lim}))
        torch.cuda.synchronize()
        err[pc] = max(_rel_rows(g[0], eA).max(), _rel_rows(g[2], eb).max(), _rel_rows(g[3], ec).max())
    o = orc.vjp_batch(st, bt.A_vals, bt.b, bt.c, xo, yo, so, dx, dy, bt.P_vals, lsqr_precond=0, lsqr_iter_lim=lim)
    err_o = max(_rel_rows(o[0], eA).max(), _rel_rows(o[2], eb).max(), _rel_rows(o[3], ec).max())
    assert err[1] < 1e-4 and err[2] < 1e-4, (name, err)
    assert err[0] < 5e-3 and err_o < 5e-3, (name, err, err_o)
    if err[0] > 1e-4:   # the deviation is the recurrence's: the oracle running the same recurrence shows it too
        assert 0.1 < err[0] / err_o < 10.0, (name, err[0], err_o)


# ----------------------------------------------------------------------------- the QP in the form the reference's DIFFCP path produces
def test_c2_in_soc_form_through_the_generic_kernels(cuda_device):
    """C2-sized instances (n = 100, m = 200) as quad_form -> SOC (one cone of size n + 2, problems.qp_as_socp): what the
    reference's DIFFCP canonicalisation would really hand over (_quad_form_dpp.py:29-32).  25,052 values per instance: the
    generic kernels (CG forward, LSQR backward) take it.  Forward vs the native-P solve and the oracle; backward vs the
    oracle on the same inputs."""
    B = 32
    bq = pr.dense_qp(B, 100, 200, 50, seed=3)
    bt = pr.qp_as_socp(bq)
    st, dev = bt.structure, cuda_device
    eps = 1e-8
    eng = Engine(st, dev)
    assert eng.path_info()["fwd"].startswith("fwd_kernel")
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    sol = eng.solve(A, b, c, None, make_settings({"eps": eps, "max_iters": 200000}))
    torch.cuda.synchronize()
    assert int((sol.status == 1).sum()) == B, (sol.status, sol.iters)
    x = sol.x.cpu().numpy()
    assert np.abs(x[:, :100] - bq.x_star).max() < 1e-5 and np.abs(x - bt.x_star).max() < 1e-4
    xo, yo, so, sto, ito = orc.solve_batch(st, bt.A_vals, bt.b, bt.c, None, nthreads=NT, eps=eps, max_iters=200000)
    assert (sto == 1).all() and np.abs(x - xo).max() < 1e-5 * max(1.0, np.abs(xo).max())
    rng = np.random.default_rng(8)
    dx, dy = rng.standard_normal(xo.shape), rng.standard_normal(yo.shape)
    bwd = {"lsqr_precond": 1, "lsqr_iter_lim": 20 * (st.n + st.m + 1)}
    g = eng.vjp(A, b, c, _t(xo, dev), _t(yo, dev), _t(so, dev), _t(dx, dev), _t(dy, dev), None, make_settings(bwd))
    torch.cuda.synchronize()
    r = orc.vjp_batch(st, bt.A_vals, bt.b, bt.c, xo, yo, so, dx, dy, None, nthreads=NT, **bwd)
    for g_, r_ in ((g[0], r[0]), (g[2], r[2]), (g[3], r[3])):
        e = _rel_rows(g_, r_)
        assert e.max() < 1e-4, (e.max(), int(e.argmax()))
