"""diffcp's ``mode="lsmr"`` on the GPU: the adjoint (``bcone_vjp``) and the forward mode (``bcone_jvp``) with LSMR in place of
LSQR (settings.lsmr = 1), on every backward kernel.

* ``lsqr_precond = 0``: at fixed iteration limits the kernels' result is SciPy's ``lsmr`` on the explicit system (within the
  spread SciPy shows against itself under last-bit changes, see _scipy_with_spread), and they stop where SciPy does (within
  the range of iterations SciPy itself stops at under those changes);
* ``lsqr_precond`` 1 and 2 against exact least squares, the block-preconditioned pass and its fallback included;
* every tier of the generic kernel (values off chip, the 128-register and 4-CTA/SM builds, vectors in the global slab)
  gives the default tier's result and iteration counts;
* the adjoint identity between the LSMR forward mode and the LSMR adjoint, the inactive-row tangent and a zero tangent;
* the shared-matrix adjoint's batch sums, and ``gradcheck`` with forward AD through the plain and the fused layer.
"""
import numpy as np
import pytest
import torch
from scipy.sparse.linalg import lsmr as scipy_lsmr

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from oracle import oracle as orc
from tests import lsmr_ref
from tests.jvp_ref import dense_M, jvp_rhs, random_tangents

pytestmark = pytest.mark.gpu

LSMR = {"mode": "lsmr"}
TIGHT = {"mode": "lsmr", "lsqr_precond": 1, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12}
CONFIGS = [("C1", 4), ("C2", 4), ("C3", 4), ("C5", 3), ("EXP", 4)]


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _np(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _rel(a, b):
    a, b = _np(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


_SOLVED = {}


def _solved(name, B):
    """A batch of ``name`` and its oracle solution (cached: several tests differentiate the same points)."""
    if (name, B) not in _SOLVED:
        bt = pr.CONFIGS[name](B=B)
        xo, yo, so, sto, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-11, max_iters=400000)
        assert (sto == 1).all()
        _SOLVED[name, B] = (bt, xo, yo, so)
    return _SOLVED[name, B]


def _instance(bt, i, xo, yo, so):
    P = bt.P_dense(i) if bt.P_vals is not None else None
    return (bt.structure, bt.A_dense(i), P, bt.b[i], bt.c[i], xo[i], yo[i], so[i])


def _vjp(eng, bt, x, y, s, dx, dy, dev, args):
    return eng.vjp(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(x, dev), _t(y, dev), _t(s, dev), _t(dx, dev), _t(dy, dev),
                   _t(bt.P_vals, dev), make_settings(args))


def _jvp(eng, bt, t, x, y, s, dev, args):
    return eng.jvp(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(x, dev), _t(y, dev), _t(s, dev), _t(t.A_vals, dev), _t(t.b, dev),
                   _t(t.c, dev), _t(bt.P_vals, dev), _t(t.P_vals, dev), make_settings(args))


def _dense_problems(bt, xo, yo, so, dx, dy, t):
    """Per instance: (adjoint matrix M', dz, pi_y, forward-mode matrix M, g, D)."""
    out = []
    for i in range(bt.B):
        args = _instance(bt, i, xo, yo, so)
        M, D, piy = dense_M(*args)
        dz = np.concatenate([dx[i], D.T @ dy[i], [-(xo[i] @ dx[i] + yo[i] @ dy[i])]])
        dP = t.P_dense(i) if t.P_vals is not None else None
        g = jvp_rhs(bt.A_dense(i), xo[i], piy, t.A_dense(i), dP, t.b[i], t.c[i])
        out.append((M.T, dz, piy, M, g, D))
    return out


def _scipy_with_spread(Bm, rhs, maxiter, outputs, k=10):
    """SciPy's lsmr on (Bm, rhs) -> (outputs(x), (least, most) iterations, spread): ``spread`` is how far SciPy's own outputs move
    when Bm and rhs change in their last bits (relative 1e-15, k draws), and the iteration counts span the unchanged and the k
    changed runs.  The explicit M is singular (the embedding's homogeneity direction), and
    at a fixed iteration count a Krylov iterate of such a system amplifies rounding: SciPy against itself moves by up to 5e-2 at
    10 iterations on EXP.  A solver that computes the same recurrence with other rounding (the kernels' sums run in another order)
    can only be held to that spread, not to 1e-10.  Where a stopping test is close to its threshold the stopping iteration moves
    too (C1: 33 to 35, C3: 298 to 301 under last-bit changes), so the kernels' count is held to the range SciPy itself reaches (widened by two: k draws do not find all of it)."""
    kw = dict(atol=1e-8, btol=1e-8, conlim=1e8, maxiter=maxiter)
    x, _, itn = scipy_lsmr(Bm, rhs, **kw)[:3]
    ref = outputs(x)
    spread, lo, hi = 0.0, itn, itn
    for j in range(k):
        g = np.random.default_rng(100 + j)
        xp, _, itp = scipy_lsmr(Bm * (1 + 1e-15 * g.standard_normal(Bm.shape)), rhs * (1 + 1e-15 * g.standard_normal(rhs.shape)), **kw)[:3]
        spread = max(spread, *(_rel(a, b) for a, b in zip(outputs(xp), ref)))
        lo, hi = min(lo, itp), max(hi, itp)
    return ref, (lo, hi), spread


def _jvp_from_z(z, x, y, s, D, n):
    zx, zy, zt = z[:n], z[n:-1], z[-1]
    Dzy = D @ zy
    return zx - x * zt, Dzy - y * zt, Dzy - zy - s * zt


# ----------------------------------------------------------------------------- parity with SciPy (lsqr_precond = 0)
@pytest.mark.parametrize("name,B", CONFIGS)
def test_plain_lsmr_matches_scipy(name, B, cuda_device):
    dev = cuda_device
    bt, xo, yo, so = _solved(name, B)
    st = bt.structure
    n, N = st.n, st.n + st.m + 1
    rng = np.random.default_rng(7)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    t = random_tangents(bt, rng)
    dense = _dense_problems(bt, xo, yo, so, dx, dy, t)
    eng = Engine(st, dev)
    worst = 0.0
    for lim in (3, 10, 40, -1):
        args = {**LSMR, "lsqr_precond": 0, "lsqr_iter_lim": lim}
        _, _, gb, gc, its_a = _vjp(eng, bt, xo, yo, so, dx, dy, dev, args)
        jx, jy, js, its_j = _jvp(eng, bt, t, xo, yo, so, dev, args)
        maxiter = lim if lim > 0 else 2 * N
        for i, (MT, dz, piy, M, g, D) in enumerate(dense):
            (db, dc), itn_a, sp_a = _scipy_with_spread(MT, dz, maxiter, lambda r, i=i, piy=piy: lsmr_ref.adjoint_grads(r, xo[i], piy, n)[1:])
            ref_j, itn_j, sp_j = _scipy_with_spread(M, g, maxiter, lambda z, i=i, D=D: _jvp_from_z(z, xo[i], yo[i], so[i], D, n))
            # (10 draws do not find every count SciPy can stop at: two iterations of slack on either side)
            assert itn_a[0] - 2 <= int(its_a[i]) <= itn_a[1] + 2 and itn_j[0] - 2 <= int(its_j[i]) <= itn_j[1] + 2, (
                name, lim, i, int(its_a[i]), itn_a, int(its_j[i]), itn_j)
            ea = max(_rel(gb[i], db), _rel(gc[i], dc))
            ej = max(_rel(jx[i], ref_j[0]), _rel(jy[i], ref_j[1]), _rel(js[i], ref_j[2]))
            worst = max(worst, ea / max(sp_a, 1e-9), ej / max(sp_j, 1e-9))
            assert ea <= max(1e-9, 100 * sp_a) and ej <= max(1e-9, 100 * sp_j), (name, lim, i, ea, sp_a, ej, sp_j)
    print(f"{name}: largest difference to SciPy lsmr in units of SciPy's own spread (at least 1e-9): {worst:.2f}")


# ----------------------------------------------------------------------------- the equilibrated variants vs exact least squares
@pytest.mark.parametrize("name,B", CONFIGS)
def test_equilibrated_lsmr_against_exact_least_squares(name, B, cuda_device):
    dev = cuda_device
    bt, xo, yo, so = _solved(name, B)
    st = bt.structure
    n = st.n
    rng = np.random.default_rng(8)
    dx, dy = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m))
    t = random_tangents(bt, rng)
    dense = _dense_problems(bt, xo, yo, so, dx, dy, t)
    eng = Engine(st, dev)
    lim = 40 * (st.n + st.m + 1)
    block = eng.path_info()["bwd"].startswith("bwd_block_kernel")
    for pc in (1, 2):
        args = {**LSMR, "lsqr_precond": pc, "lsqr_iter_lim": lim}
        _, _, gb, gc, _ = _vjp(eng, bt, xo, yo, so, dx, dy, dev, args)
        if pc == 2 and block:
            assert eng.fallback_count() == 0, name
        jx, jy, js, _ = _jvp(eng, bt, t, xo, yo, so, dev, args)
        for i, (MT, dz, piy, M, g, D) in enumerate(dense):
            r = np.linalg.lstsq(MT, dz, rcond=None)[0]
            z = np.linalg.lstsq(M, g, rcond=None)[0]
            _, db, dc = lsmr_ref.adjoint_grads(r, xo[i], piy, n)
            ex, ey, es = _jvp_from_z(z, xo[i], yo[i], so[i], D, n)
            errs = [_rel(gb[i], db), _rel(gc[i], dc), _rel(jx[i], ex), _rel(jy[i], ey), _rel(js[i], es)]
            assert max(errs) < 1e-4, (name, pc, i, errs)


def test_block_preconditioned_lsmr_on_the_planted_batch_and_its_fallback(cuda_device):
    """C2's planted batch runs the block pass without a fallback; a P with a zero row and column (as in
    test_gpu_factor_sizes) is rejected by it and solved by the second LSMR pass."""
    dev = cuda_device
    n, m = 100, 200
    bt = pr.dense_qp(3, n, m, 50, seed=11)
    Pd = np.stack([bt.P_dense(i) for i in range(bt.B)])
    Pd[1, 45, :] = 0.0
    Pd[1, :, 45] = 0.0
    iu = np.triu_indices(n)
    bt = pr.plant(bt.structure, bt.A_vals, np.ascontiguousarray(Pd[:, iu[0], iu[1]]), np.random.default_rng(12), name="dense_qp_singular_P",
                  active_frac=0.2)
    eng = Engine(bt.structure, dev)
    assert eng.path_info()["bwd"].startswith("bwd_block_kernel")
    x, y, s = bt.x_star, bt.y_star, bt.s_star
    rng = np.random.default_rng(2)
    dx, dy = rng.standard_normal((bt.B, n)), rng.standard_normal((bt.B, m))
    args = {**LSMR, "lsqr_precond": 2, "lsqr_iter_lim": 20000}
    _, _, gb, gc, _ = _vjp(eng, bt, x, y, s, dx, dy, dev, args)
    assert eng.fallback_count() == 1
    good = pr.config_c2(B=8, seed=3)
    _vjp(eng, good, good.x_star, good.y_star, good.s_star, rng.standard_normal((8, n)), rng.standard_normal((8, m)), dev, args)
    assert eng.fallback_count() == 0
    for i in range(bt.B):
        M, dz, _, piy = lsmr_ref.adjoint_system(*_instance(bt, i, x, y, s), dx[i], dy[i])
        r = np.linalg.lstsq(M.T, dz, rcond=None)[0]
        _, db, dc = lsmr_ref.adjoint_grads(r, x[i], piy, n)
        assert max(_rel(gb[i], db), _rel(gc[i], dc)) < 1e-4, i


# ----------------------------------------------------------------------------- every tier of the generic kernel
def _tier_outputs(bt, x, y, s, dx, dy, t, dev, args):
    eng = Engine(bt.structure, dev)
    B = bt.B
    gA, gP, gb, gc, ia = _vjp(eng, bt, x, y, s, dx, dy, dev, args)
    jx, jy, js, ij = _jvp(eng, bt, t, x, y, s, dev, args)
    return [v.cpu().numpy() for v in (gA, gb, gc, jx, jy, js)], ia.cpu().numpy(), ij.cpu().numpy(), eng, B


def _same(ref, got, what):
    (o0, ia0, ij0), (o1, ia1, ij1) = ref, got
    assert (ia0 == ia1).all() and (ij0 == ij1).all(), what
    for a, b in zip(o1, o0):
        assert _rel(a, b) <= 1e-12, (what, _rel(a, b))


@pytest.mark.parametrize("name,B", [("C3", 64), ("C5", 32), ("EXP", 32), ("C2SOC", 8)])
def test_every_tier_gives_the_default_result(name, B, cuda_device, monkeypatch):
    dev = cuda_device
    bt = pr.CONFIGS[name](B=B) if name != "C2SOC" else pr.qp_as_socp(pr.dense_qp(B, 100, 200, 50, seed=0), factor="eigen")
    st = bt.structure
    eng = Engine(st, dev)
    sol = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings({"eps": 1e-9, "max_iters": 200000}))
    assert int((sol.status == 1).sum()) == B
    x, y, s = (v.cpu().numpy() for v in (sol.x, sol.y, sol.s))
    rng = np.random.default_rng(4)
    dx, dy, t = rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m)), random_tangents(bt, rng)
    for pc in (0, 1):
        args = {**LSMR, "lsqr_precond": pc}
        for k in ("BCONE_VALUES_GLOBAL", "BCONE_SMALL_CTA"):
            monkeypatch.delenv(k, raising=False)
        o, ia, ij, eng0, _ = _tier_outputs(bt, x, y, s, dx, dy, t, dev, args)
        ref = (o, ia, ij)
        assert (ia > 0).all() and (ij > 0).all()
        if name == "C2SOC":   # the eigen form runs values off chip by default
            assert "values off chip" in eng0.path_info()["bwd"]
        for env in (("BCONE_VALUES_GLOBAL", "1"), ("BCONE_SMALL_CTA", "0"), ("BCONE_SMALL_CTA", "2")):
            for k in ("BCONE_VALUES_GLOBAL", "BCONE_SMALL_CTA"):
                monkeypatch.delenv(k, raising=False)
            monkeypatch.setenv(*env)
            o1, ia1, ij1, _, _ = _tier_outputs(bt, x, y, s, dx, dy, t, dev, args)
            _same(ref, (o1, ia1, ij1), (name, pc, env))


def test_vectors_in_the_global_slab(cuda_device):
    """C4's instances (n = 1000, m = 2000) keep the LSMR vectors in the per-CTA slab: the adjoint against SciPy at a fixed
    iteration count, and the adjoint identity with the forward mode."""
    dev = cuda_device
    bt = pr.CONFIGS["C4"](B=3)
    st = bt.structure
    eng = Engine(st, dev)
    # (any point will do for the derivatives: the solve is not held to its tolerance here)
    sol = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings({"eps": 1e-4, "max_iters": 5000}))
    x, y, s = (v.cpu().numpy() for v in (sol.x, sol.y, sol.s))
    rng = np.random.default_rng(6)
    dx, dy, t = rng.standard_normal((bt.B, st.n)), rng.standard_normal((bt.B, st.m)), random_tangents(bt, rng)
    args = {**LSMR, "lsqr_precond": 0, "lsqr_iter_lim": 10}
    _, _, gb, gc, its = _vjp(eng, bt, x, y, s, dx, dy, dev, args)
    assert (its.cpu().numpy() == 10).all()
    for i in range(bt.B):
        M, dz, _, piy = lsmr_ref.adjoint_system(*_instance(bt, i, x, y, s), dx[i], dy[i])
        (db, dc), _, sp = _scipy_with_spread(M.T, dz, 10, lambda r: lsmr_ref.adjoint_grads(r, x[i], piy, st.n)[1:], k=3)
        e = max(_rel(gb[i], db), _rel(gc[i], dc))
        assert e <= max(1e-9, 100 * sp), (i, e, sp)
    _adjoint_identity(eng, bt, x, y, s, t, dev, {**TIGHT, "lsqr_iter_lim": 20000})


# ----------------------------------------------------------------------------- forward mode: the adjoint identity
def _adjoint_identity(eng, bt, x, y, s, t, dev, args, pcs=(1,)):
    B, st = bt.B, bt.structure
    rng = np.random.default_rng(9)
    w = (rng.standard_normal((B, st.n)), rng.standard_normal((B, st.m)))
    jx, jy, _, its = _jvp(eng, bt, t, x, y, s, dev, args)
    jx, jy = jx.cpu().numpy(), jy.cpu().numpy()
    assert (its.cpu().numpy() > 0).all()
    lhs = (w[0] * jx).sum(1) + (w[1] * jy).sum(1)
    scale = np.sqrt((w[0] ** 2).sum(1) + (w[1] ** 2).sum(1)) * np.sqrt((jx ** 2).sum(1) + (jy ** 2).sum(1))
    for pc in pcs:
        gA, gP, gb, gc, _ = _vjp(eng, bt, x, y, s, w[0], w[1], dev, {**args, "lsqr_precond": pc})
        rhs = (gA.cpu().numpy() * t.A_vals).sum(1) + (gb.cpu().numpy() * t.b).sum(1) + (gc.cpu().numpy() * t.c).sum(1)
        if gP is not None:
            rhs += (gP.cpu().numpy() * t.P_vals).sum(1)
        e = np.abs(lhs - rhs) / scale
        assert e.max() < 1e-6, (pc, e.max(), int(e.argmax()))


@pytest.mark.parametrize("name,B", [("C1", 64), ("C2", 512), ("C3", 256), ("C5", 64), ("EXP", 64)])
def test_jvp_is_the_transpose_of_vjp(name, B, cuda_device):
    dev = cuda_device
    bt = pr.CONFIGS[name](B=B)
    eng = Engine(bt.structure, dev)
    if bt.x_star is not None:
        x, y, s = bt.x_star, bt.y_star, bt.s_star
    else:
        sol = eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), make_settings({"eps": 1e-9, "max_iters": 200000}))
        assert int((sol.status == 1).sum()) == B
        x, y, s = (v.cpu().numpy() for v in (sol.x, sol.y, sol.s))
    t = random_tangents(bt, np.random.default_rng(10))
    args = {**TIGHT, "lsqr_iter_lim": 40 * (bt.structure.n + bt.structure.m + 1)}
    _adjoint_identity(eng, bt, x, y, s, t, dev, args, pcs=(1, 2) if name in ("C1", "C2") else (1,))


@pytest.mark.parametrize("shape", [(10, 20, 0), (8, 14, 3)])
def test_tangent_on_inactive_rows_only(shape, cuda_device):
    """As test_gpu_jvp_inactive, with LSMR: a tangent in rows of inactive nonneg constraints only.  The equilibrated system's
    right-hand side is then exactly zero; the tangent must be finite and agree with the plain LSMR."""
    n, m, z = shape
    dev = cuda_device
    bt = pr.dense_qp(2, n, m, z, seed=12)
    eng = Engine(bt.structure, dev)
    T = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)  # noqa: E731
    A, P, b, c = T(bt.A_vals), T(bt.P_vals), T(bt.b), T(bt.c)
    sol = eng.solve(A, b, c, P, make_settings({"eps": 1e-11, "max_iters": 200000}))
    assert bool((sol.status == 1).all())
    inactive = [i for i in range(z, m) if float(sol.y[0, i]) == 0.0 and float(sol.y[1, i]) == 0.0]
    assert inactive
    zb, zc, zP = torch.zeros_like(b), torch.zeros_like(c), torch.zeros_like(P)
    for i in inactive[:4]:
        for j in (0, n - 1):
            tA = torch.zeros_like(A)
            tA[:, i * n + j] = 1.0
            outs = {pc: eng.jvp(A, b, c, sol.x, sol.y, sol.s, tA, zb, zc, P, zP,
                                make_settings({**LSMR, "lsqr_precond": pc, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12})) for pc in (0, 1)}
            for a_, b_ in zip(outs[1][:3], outs[0][:3]):
                assert bool(torch.isfinite(a_).all())
                assert float((a_ - b_).abs().max()) <= 1e-6 * max(1.0, float(b_.abs().max()))


@pytest.mark.parametrize("name", ["C1", "C3"])
def test_zero_tangent_takes_no_iterations(name, cuda_device):
    dev = cuda_device
    bt, xo, yo, so = _solved(name, 4)
    z = pr.Batch(bt.structure, np.zeros_like(bt.A_vals), np.zeros_like(bt.b), np.zeros_like(bt.c),
                 None if bt.P_vals is None else np.zeros_like(bt.P_vals))
    eng = Engine(bt.structure, dev)
    for pc in (0, 1):
        jx, jy, js, its = _jvp(eng, bt, z, xo, yo, so, dev, {**LSMR, "lsqr_precond": pc})
        assert (its.cpu().numpy() == 0).all()
        assert not any(bool(v.abs().max() > 0) for v in (jx, jy, js))


# ----------------------------------------------------------------------------- shared matrices
@pytest.mark.parametrize("name,pc", [("C1", 0), ("C1", 2), ("C2", 1), ("C2", 2), ("C3", 1), ("C5", 1), ("EXP", 0)])
def test_shared_matrix_adjoint_sums(name, pc, cuda_device):
    """test_gpu_shared's checks with LSMR: the shared adjoint's sums against the per-instance sums to 1e-12 of sum |dA_b|,
    db, dc and the iteration counts bit-identical, two runs bit-identical."""
    from tests.test_gpu_shared import _check_vjp, shared_batch

    eng = _check_vjp(shared_batch(name, 256 if name in ("C1", "C2") else 64, seed=9), cuda_device, {**LSMR, "lsqr_precond": pc})
    if name == "C2" and pc == 2:
        assert eng.path_info()["bwd"].startswith("bwd_block_kernel") and eng.fallback_count() == 0


def test_shared_matrix_adjoint_block_fallback(cuda_device):
    """A shared P with a zero row and column: every instance goes to the second LSMR pass, which writes the records."""
    from tests.test_gpu_shared import _check_vjp

    base = pr.CONFIGS["C2"](B=1, seed=11)
    n = base.structure.n
    Pd = base.P_dense(0)
    Pd[45, :] = 0.0
    Pd[:, 45] = 0.0
    iu = np.triu_indices(n)
    B = 64
    bt = pr.plant(base.structure, np.repeat(base.A_vals, B, 0), np.repeat(Pd[iu][None], B, 0), np.random.default_rng(12), active_frac=0.2)
    eng = _check_vjp(bt, cuda_device, {**LSMR, "lsqr_precond": 2})
    assert eng.fallback_count() == B


# ----------------------------------------------------------------------------- the layer
def _programs():
    from tests.test_gpu_jvp import _sdp_make, _soc_make

    return ((_sdp_make, np.array([2.0, 0.5, 0.1, 3.0, 0.2, 1.5])), (_soc_make, np.array([0.5, 0.3, -0.2, 2.0])))


LAYER_ARGS = {"eps": 1e-12, "max_iters": 400000, **TIGHT, "lsqr_iter_lim": 20000}


@pytest.mark.parametrize("prog", [0, 1])
def test_layer_gradcheck_with_forward_ad(prog, cuda_device):
    """The reference's PSD and SOC gradcheck programs through _CvxpyLayer with mode = "lsmr"."""
    from tests.test_gpu_jvp import _layer_fn

    make, p0 = _programs()[prog]
    bd, f = _layer_fn(make(p0[None]), cuda_device, LAYER_ARGS)
    A = _t(bd.A_eval, cuda_device).requires_grad_(True)
    q = _t(bd.q_eval, cuda_device).requires_grad_(True)
    if bd.P_eval is not None:
        fn, inputs = f, (_t(bd.P_eval, cuda_device).requires_grad_(True), q, A)
    else:
        fn, inputs = (lambda q_, A_: f(None, q_, A_)), (q, A)
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-4, rtol=1e-3, check_forward_ad=True, check_undefined_grad=False)


@pytest.mark.parametrize("prog", [0, 1])
def test_fused_layer_gradcheck_with_forward_ad(prog, cuda_device):
    """The same programs through _CvxpyLayerFused, mode = "lsmr" given per call."""
    from cvxpylayers_b200.interface import _CvxpyLayerFused
    from tests.test_gpu_shared import _fused

    make, p0 = _programs()[prog]
    _, cl, p_stack = _fused(make(p0[None]), cuda_device, {})

    def f(ps):
        return _CvxpyLayerFused.apply(ps, cl, LAYER_ARGS, True, None)[:2]

    assert torch.autograd.gradcheck(f, (p_stack.clone().requires_grad_(True),), eps=1e-6, atol=1e-4, rtol=1e-3,
                                    check_forward_ad=True, check_undefined_grad=False)
