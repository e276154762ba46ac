"""The register-tiled forward (fwd_fast.cu) and the dense adjoints (bwd_fast.cu, bwd_block.cu) across the shape classes of
tests/tiled_shapes.py, on batches with a planted, strictly complementary optimum: the forward (default, warm start, A / P one
double off 16-byte alignment), the cached and the batch-shared set-up against the planted optimum; the adjoint with
lsqr_precond 0, 1, 2 and LSMR through whichever kernel the shape selects, misaligned once, and the batch-shared adjoint's sums,
against dense least squares with the exact cone Jacobian (tests/cone_ref.py).  Every failure message names the shape.

Tolerances: TOL, with the worst errors measured on an H100 80GB HBM3 (700 W) over all cases below it.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cvxpylayers_b200.engine import Engine, make_settings
from cvxpylayers_b200.structure import ConeSpec
from tests import cone_ref as cr
from tests import tiled_shapes as ts

pytestmark = pytest.mark.gpu

KEYS = list(ts.CASES)
B = 4
FWD = {"eps_abs": 1e-10, "eps_rel": 1e-10, "max_iters": 400000}
TIGHT = {"lsqr_atol": 1e-14, "lsqr_btol": 1e-14, "lsqr_conlim": 1e14}
TOL = {
    # relative to max(1, |planted|_inf), as in test_gpu_cones; y is the least well determined (nch1_live_eq_n: n live rows)
    "x": 1e-7, "s": 1e-7, "y": 3e-6,
    # relative to the exact answer's largest entry
    "precond0": 1e-8, "precond1": 1e-10, "precond2": 1e-10, "lsmr1": 1e-10, "shared": 3e-10,
}
# worst measured (all on nch1_live_eq_n unless named): x 4.2e-9, y 1.8e-7, s 4.6e-9 (cached, new b and c); adjoint lsqr_precond
# 0 4.2e-10, 1 2.5e-12 (misaligned), 2 1.1e-12 (n_gt_m), LSMR 4.7e-12; shared adjoint sums 1.7e-11 (dP).  The whole file runs
# in 17-19 s on the H100 (112 tests).
MODES = {"precond0": {"lsqr_precond": 0}, "precond1": {"lsqr_precond": 1}, "precond2": {"lsqr_precond": 2},
         "lsmr1": {"lsqr_precond": 1, "mode": "lsmr"}}
_CACHE: dict = {}


def _batch(key, shared=False):
    k = (key, shared)
    if k not in _CACHE:
        _CACHE[k] = ts.planted(ts.CASES[key], B, seed=100 + 2 * KEYS.index(key) + shared, shared=shared)
    return _CACHE[k]


def _replant_seed(key):
    return 7 + KEYS.index(key)


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _misaligned(a, dev):
    """A contiguous copy of ``a`` that starts one double into a larger buffer: 8 bytes off 16-byte alignment."""
    if a is None:
        return None
    buf = torch.zeros(a.size + 1, dtype=torch.float64, device=dev)
    v = buf[1:].view(a.shape)
    v.copy_(torch.as_tensor(a))
    assert v.is_contiguous() and v.data_ptr() % 16 == 8
    return v


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _check_forward(bt, sol, what):
    st = sol.status.cpu().numpy()
    assert (st == 1).all(), (what, st, sol.iters.cpu().numpy(), sol.resid.cpu().numpy())
    x, y, s = (t.cpu().numpy() for t in (sol.x, sol.y, sol.s))
    errs = {k: max(_rel(got[i], ref[i]) for i in range(bt.B)) for k, got, ref in (("x", x, bt.x_star), ("y", y, bt.y_star), ("s", s, bt.s_star))}
    print(f"{what}: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()) + f" iters {sol.iters.cpu().numpy()}")
    assert all(errs[k] <= TOL[k] for k in errs), (what, errs)


def _engine(key, dev):
    c = ts.CASES[key]
    eng = Engine(_batch(key).structure, dev)
    path, info = eng.path_info(), eng.kernel_info()
    print(f"{c.id}: {path} {info}")
    assert "register-tiled" in path["fwd"], (c.id, path)
    assert info["fwd_smem"] == ts.smem_bytes(c.n, c.m), (c.id, info)
    return eng


@pytest.mark.parametrize("key", KEYS)
def test_kernel_paths(key, cuda_device):
    """The register-tiled forward with the shared memory bc_fwdf_smem_bytes names, and the adjoint kernel the case records."""
    c = ts.CASES[key]
    path = _engine(key, cuda_device).path_info()
    assert path["bwd"] == Engine.BWD_PATHS[c.bwd], (c.id, path["bwd"])


@pytest.mark.parametrize("key", KEYS)
def test_forward_matches_planted_optimum(key, cuda_device):
    """Default settings, warm start at the planted point, and A / P passed 8 bytes off 16-byte alignment (plain loads in
    place of the bulk copies)."""
    bt, dev, c = _batch(key), cuda_device, ts.CASES[key]
    eng = _engine(key, dev)
    A, b, cc, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    S = make_settings(FWD)
    default = eng.solve(A, b, cc, P, S)
    _check_forward(bt, default, f"{c.id} default")
    warm = tuple(_t(a, dev) for a in (bt.x_star, bt.y_star, bt.s_star))
    _check_forward(bt, eng.solve(A, b, cc, P, S, warm=warm), f"{c.id} warm")
    mis = eng.solve(_misaligned(bt.A_vals, dev), b, cc, _misaligned(bt.P_vals, dev), S)
    _check_forward(bt, mis, f"{c.id} misaligned A / P")
    # how the data reach shared memory does not change the arithmetic: the same bits (and a race would show here)
    assert all(_same(default, mis).values()), (c.id, _same(default, mis))


def _same(a, b, idx=None):
    pick = (lambda t: t) if idx is None else (lambda t: t[idx])  # noqa: E731
    return {k: torch.equal(pick(getattr(a, k)), pick(getattr(b, k))) for k in ("x", "y", "s", "status", "iters")}


@pytest.mark.parametrize("key", KEYS)
def test_cached_setup(key, cuda_device):
    """Filling the cache leaves the solve bit-identical; reusing it reproduces the uncached solve bit for bit where the record
    is at the initial scale and reaches the planted optimum everywhere; a call with a new planted b, c on the same A, P from the
    cache reaches the new optimum."""
    bt, dev, c = _batch(key), cuda_device, ts.CASES[key]
    eng = Engine(bt.structure, dev)
    A, b, cc, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    S = make_settings(FWD)
    cache = eng.new_cache(B)
    assert cache is not None and cache.numel() == B * ts.cache_doubles(c.n, c.m), c.id
    plain = eng.solve(A, b, cc, P, S)
    fill = eng.solve(A, b, cc, P, S, cache=cache, reuse=False)
    assert all(_same(plain, fill).values()), (c.id, _same(plain, fill))
    hdr = cache.view(B, -1)[:, :3].cpu().numpy()
    assert (hdr[:, 1] == 1.0).all() and (hdr[:, 2] == S.rho_x).all(), (c.id, hdr)
    again = eng.solve(A, b, cc, P, S, cache=cache, reuse=True)
    kept = np.nonzero(hdr[:, 0] == S.scale)[0]
    if kept.size:
        same = _same(plain, again, torch.as_tensor(kept, device=dev))
        assert all(same.values()), (c.id, kept, same)
    _check_forward(bt, again, f"{c.id} cached, reuse ({kept.size} records at the initial scale)")
    bt2 = ts.replant(bt, c, seed=_replant_seed(key))
    _check_forward(bt2, eng.solve(A, _t(bt2.b, dev), _t(bt2.c, dev), P, S, cache=cache, reuse=True), f"{c.id} cached, new b and c")


@pytest.mark.parametrize("key", KEYS)
def test_shared_setup(key, cuda_device):
    """bcone_solve_shared (one A and P for the batch, one set-up) against the planted optima, and bit-identical to the same
    batch with A and P replicated."""
    bt, dev, c = _batch(key, shared=True), cuda_device, ts.CASES[key]
    eng = Engine(bt.structure, dev)
    b, cc, S = _t(bt.b, dev), _t(bt.c, dev), make_settings(FWD)
    got = eng.solve(_t(bt.A_vals[0], dev), b, cc, _t(None if bt.P_vals is None else bt.P_vals[0], dev), S)
    _check_forward(bt, got, f"{c.id} shared A / P")
    rep = eng.solve(_t(bt.A_vals, dev), b, cc, _t(bt.P_vals, dev), S)
    assert all(_same(got, rep).values()), (c.id, _same(got, rep))


# ----------------------------------------------------------------------------- adjoint
def _exact(key, shared, i):
    """The exact adjoint's matrix at instance i's planted point (cached per batch)."""
    k = (key, shared, i)
    if k not in _CACHE:
        bt, c = _batch(key, shared), ts.CASES[key]
        _CACHE[k] = cr.dense_M(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i],
                               ConeSpec(z=c.z, l=c.m - c.z))
    return _CACHE[k]


def _exact_grads(key, shared, dx, dy):
    """-> per instance the exact (dA in CSR order, dP on the upper triangle or None, db, dc)."""
    bt, c = _batch(key, shared), ts.CASES[key]
    iu = np.triu_indices(c.n)
    out = []
    for i in range(bt.B):
        dA, dP, db, dc = cr.exact_adjoint(bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i], bt.x_star[i], bt.y_star[i], bt.s_star[i],
                                          dx[i], dy[i], ConeSpec(z=c.z, l=c.m - c.z), _exact(key, shared, i))
        dPu = np.where(iu[0] == iu[1], dP[iu], dP[iu] + dP.T[iu]) if c.P else None
        out.append((dA.ravel(), dPu, db, dc))
    return out


def _settings(bt, mode):
    st = bt.structure
    return make_settings({**TIGHT, **MODES[mode], "lsqr_iter_lim": 50 * (st.n + st.m + 1)})


def _adjoint_error(key, eng, dev, mode, misaligned=False):
    bt, c = _batch(key), ts.CASES[key]
    rng = np.random.default_rng(11)
    dx, dy = rng.standard_normal((B, c.n)), rng.standard_normal((B, c.m))
    put = _misaligned if misaligned else _t
    gA, gP, gb, gc, its = eng.vjp(put(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.x_star, dev), _t(bt.y_star, dev),
                                  _t(bt.s_star, dev), _t(dx, dev), _t(dy, dev), put(bt.P_vals, dev), _settings(bt, mode))
    got = [t.cpu().numpy() if t is not None else None for t in (gA, gP, gb, gc)]
    worst = 0.0
    for i, ref in enumerate(_exact_grads(key, False, dx, dy)):
        r = np.concatenate([a for a in ref if a is not None])
        g = np.concatenate([a[i] for a in got if a is not None])
        worst = max(worst, np.abs(g - r).max() / np.abs(r).max())
    return worst, its.cpu().numpy()


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("key", KEYS)
def test_adjoint_matches_exact_least_squares(key, mode, cuda_device):
    """Engine.vjp at the planted point against lstsq with the exact cone Jacobian: dA, dP, db, dc.  lsqr_precond = 2 runs the
    KKT-block kernel where the shape selects it; it must take every instance whose live rows it has room for (they are
    independent, P is positive definite) and hand on exactly the others."""
    dev, c = cuda_device, ts.CASES[key]
    eng = _engine(key, dev)
    worst, its = _adjoint_error(key, eng, dev, mode)
    print(f"{c.id} {mode} [{eng.path_info()['bwd']}]: adjoint worst {worst:.1e}, iterations {its}")
    if mode == "precond2" and c.bwd == 2:
        _check_fallbacks(eng, c)
    assert worst <= TOL[mode], (c.id, mode, worst)


def _check_fallbacks(eng, c):
    want = 0 if ts.block_takes(c.n, c.m, c.z + c.active) else B
    assert eng.fallback_count() == want, (c.id, eng.fallback_count(), want)


@pytest.mark.parametrize("mode", ["precond1", "precond2"])
@pytest.mark.parametrize("key", ["nch1_live_eq_n", "kr4"])
def test_adjoint_misaligned(key, mode, cuda_device):
    """A / P 8 bytes off 16-byte alignment: the fused kernel's plain loads of A and P (precond1) and the block kernel's plain
    loads of the live rows (precond2)."""
    dev, c = cuda_device, ts.CASES[key]
    eng = _engine(key, dev)
    worst, its = _adjoint_error(key, eng, dev, mode, misaligned=True)
    print(f"{c.id} {mode} misaligned: adjoint worst {worst:.1e}, iterations {its}")
    if mode == "precond2":
        _check_fallbacks(eng, c)
    assert worst <= TOL[mode], (c.id, mode, worst)


@pytest.mark.parametrize("key", KEYS)
def test_shared_adjoint_sums(key, cuda_device):
    """bcone_vjp_shared: dA_sum / dP_sum against the sum of the exact per-instance adjoints, db / dc per instance."""
    bt, dev, c = _batch(key, shared=True), cuda_device, ts.CASES[key]
    eng = Engine(bt.structure, dev)
    rng = np.random.default_rng(12)
    dx, dy = rng.standard_normal((B, c.n)), rng.standard_normal((B, c.m))
    gA, gP, gb, gc, its = eng.vjp(_t(bt.A_vals[0], dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.x_star, dev), _t(bt.y_star, dev),
                                  _t(bt.s_star, dev), _t(dx, dev), _t(dy, dev), _t(None if bt.P_vals is None else bt.P_vals[0], dev),
                                  _settings(bt, "precond1"))
    ref = _exact_grads(key, True, dx, dy)
    errs = {"dA_sum": np.abs(gA.cpu().numpy() - sum(r[0] for r in ref)).max() / np.abs(sum(r[0] for r in ref)).max(),
            "db": max(np.abs(gb[i].cpu().numpy() - r[2]).max() / np.abs(r[2]).max() for i, r in enumerate(ref)),
            "dc": max(np.abs(gc[i].cpu().numpy() - r[3]).max() / np.abs(r[3]).max() for i, r in enumerate(ref))}
    if c.P:
        sP = sum(r[1] for r in ref)
        errs["dP_sum"] = np.abs(gP.cpu().numpy() - sP).max() / np.abs(sP).max()
    print(f"{c.id} shared adjoint: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()) + f" iterations {its.cpu().numpy()}")
    assert max(errs.values()) <= TOL["shared"], (c.id, errs)
