"""Infeasible, unbounded and iteration-limited instances on the forward paths (batches of tests/infeas_planted.py), and the
warm start after a non-solved instance.

Every batch mixes primal-infeasible instances, unbounded ones (a general ray and a zero column) and controls with a planted
optimum, one of them with a small slack along a certificate.  On every path: each status equals the plant and the C oracle's,
certified instances stop before ``max_iters``, non-solved instances return NaN, and the controls are the same as in the batch
without the bad instances -- bit for bit where the arithmetic is deterministic (the register-tiled kernel, the dense generic
kernel), within the launch-to-launch spread where K is formed with atomics (CSR, direct).

Tolerances, with the worst errors measured on an H100 80GB HBM3 (700 W):
* controls against the planted optimum at eps 1e-8: x, s 1e3 eps, y 1e5 eps relative to max(1, |planted|); worst x 3.4e-7
  (exp), s 1.4e-7 (300 tiled instances), y 6.8e-5 (dense SOC); mixed_scales runs at eps 1e-5 (x 8.5e-4, y 7.3e-2);
* controls against the same controls solved without the bad instances, CSR direct: NEIGHBOUR_TOL relative; worst 2.7e-9
  (y of mixed_scales), same iteration counts;
* the iteration limit (1, 5, 37 iterations) against the oracle with the same settings: LIMIT_TOL relative; worst 3.6e-10
  (register-tiled), 2.4e-13 (generic).
The file runs in about 95 s, 17 s of it drawing the 300-instance batch.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings
from cvxpylayers_b200.interface import SolverError, _CvxpyLayer
from oracle import oracle as orc
from tests import cone_planted as cp
from tests import infeas_planted as ip
from tests import tiled_shapes as ts

pytestmark = pytest.mark.gpu

EPS, MAX_ITERS = 1e-8, 20000
NEIGHBOUR_TOL = 1e-7
LIMIT_TOL = 1e-8

_MEMO: dict = {}


def _tiled(case, kinds=ip.MIX, seed=5):
    return lambda: ip.mixed(ts.planted(case, len(kinds), seed), kinds, seed=seed + 1)


def _cone(name, kinds=ip.MIX, **kw):
    return lambda: ip.mixed(cp.make(name, B=len(kinds)), kinds, seed=1, **kw)


def _wave():
    """More instances than one wave of resident CTAs (132 on an H100): the persistent work queue hands out the rest."""
    kinds = (ip.MIX * 43)[:300]
    return ip.mixed(ts.planted(ts.Case(100, 200, 50, 40, True, 2), len(kinds), 11), kinds, seed=12)


# name -> (batch factory, environment, eps, forward path must contain, deterministic)
PATHS = {
    "tiled_compile_time": (_tiled(ts.CASES["compile_time_widest"]), {}, EPS, "register-tiled", True),
    "tiled_kr4": (_tiled(ts.CASES["kr4"]), {}, EPS, "register-tiled", True),
    "tiled_n_gt_m": (_tiled(ts.CASES["n_gt_m"]), {}, EPS, "register-tiled", True),
    "tiled_all_equality": (_tiled(ts.CASES["all_equality"], ip.MIX_NO_SLACK), {}, EPS, "register-tiled", True),
    "tiled_wave": (_wave, {}, EPS, "register-tiled", True),
    "dense_soc": (_cone("soc_sizes"), {}, EPS, "fwd_kernel", True),
    "exp": (_cone("exp"), {}, EPS, "fwd_kernel", True),
    "csr_psd_warm": (_cone("psd_warm"), {}, EPS, "fwd_kernel", False),
    "csr_psd_serial": (_cone("psd_serial"), {}, EPS, "fwd_kernel", False),
    "csr_mixed": (_cone("mixed"), {}, EPS, "fwd_kernel", False),
    "csr_mixed_scales": (_cone("mixed_scales", ip.MIX[:6]), {}, 1e-5, "fwd_kernel", False),
    # (at eps 1e-8 its small-slack control needs more than 20000 iterations)
    "csr_mixed_block_scales": (_cone("mixed", block_scale=(1e-6, 1e3)), {}, 1e-6, "fwd_kernel", False),
    "csr_mixed_x1e-4": (_cone("mixed", scale=1e-4), {}, EPS, "fwd_kernel", False),
    "csr_mixed_x1e3": (_cone("mixed", scale=1e3), {}, EPS, "fwd_kernel", False),
    "small_cta": (_cone("mixed"), {"BCONE_SMALL_CTA": "2"}, EPS, "fwd_kernel", False),
    "values_global": (_cone("mixed"), {"BCONE_VALUES_GLOBAL": "1"}, EPS, "values off chip", False),
}


def _batch(name):
    if name not in _MEMO:
        _MEMO[name] = PATHS[name][0]()
    return _MEMO[name]


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _engine(name, dev, monkeypatch):
    for k, v in PATHS[name][1].items():
        monkeypatch.setenv(k, v)
    bt = _batch(name)
    eng = Engine(bt.structure, dev)
    path = eng.path_info()["fwd"]
    assert PATHS[name][3] in path, (name, path)
    return eng


def _settings(eps, **kw):
    return make_settings({"eps": eps, "max_iters": MAX_ITERS, **kw})


def _solve(eng, bt, dev, st, **kw):
    return eng.solve(_t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev), st, **kw)


def _np(sol):
    return [t.cpu().numpy() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)]


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _check_outcomes(bt, got, eps, what):
    x, y, s, status, iters, _ = got
    plant = bt.aux["status"]
    print(f"{what}: status {status} iters {iters}")
    assert np.array_equal(status, plant), (what, status, plant, iters)
    assert (iters < MAX_ITERS).all(), (what, iters)
    bad = plant != 1
    assert np.isnan(x[bad]).all() and np.isnan(y[bad]).all() and np.isnan(s[bad]).all(), what
    ok = ip.controls(bt)
    errs = {k: _rel(g[ok], r[ok]) for k, g, r in (("x", x, bt.x_star), ("y", y, bt.y_star), ("s", s, bt.s_star))}
    print(f"{what}: controls against the planted optimum " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert errs["x"] <= 1e3 * eps and errs["s"] <= 1e3 * eps and errs["y"] <= 1e5 * eps, (what, errs)


@pytest.mark.parametrize("name", list(PATHS))
def test_outcomes_and_untouched_neighbours(name, cuda_device, monkeypatch):
    bt, dev = _batch(name), cuda_device
    eng = _engine(name, dev, monkeypatch)
    eps, det = PATHS[name][2], PATHS[name][4]
    st = _settings(eps)
    full = _np(_solve(eng, bt, dev, st))
    _check_outcomes(bt, full, eps, name)
    if bt.B <= 16:
        _, _, _, ost, oits = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=eps, max_iters=MAX_ITERS)
        assert np.array_equal(ost, full[3]), (ost, full[3], oits)
    ok = ip.controls(bt)
    alone = _np(_solve(eng, bt.select(ok), dev, st))
    for k, (a, b_) in enumerate(zip(alone, full)):
        if det or k in (3, 4):   # (status and iteration counts everywhere)
            assert np.array_equal(a, b_[ok], equal_nan=k == 5), (name, k)
        elif k < 3:
            print(f"{name}: controls alone against the mixed batch, {'xys'[k]} {_rel(a, b_[ok]):.1e}")
            assert _rel(a, b_[ok]) <= NEIGHBOUR_TOL, (name, k, _rel(a, b_[ok]))


SETUP_PATHS = {
    "tiled": lambda: ip.shared(ts.planted(ts.CASES["kr4"], len(ip.SHARED_MIX), 7, shared=True), seed=8),
    "generic": lambda: ip.shared(cp.make("mixed", B=len(ip.SHARED_MIX)), seed=4),
}


@pytest.mark.parametrize("which", list(SETUP_PATHS))
def test_batch_shared_setup(which, cuda_device):
    """One A and P for the batch, the outcome chosen through b and c: the shared solve (one set-up) against the plant and the
    replicated solve."""
    bt, dev = SETUP_PATHS[which](), cuda_device
    eng = Engine(bt.structure, dev)
    st = _settings(EPS)
    P0 = None if bt.P_vals is None else _t(bt.P_vals[0], dev)
    got = _np(eng.solve(_t(bt.A_vals[0], dev), _t(bt.b, dev), _t(bt.c, dev), P0, st))
    _check_outcomes(bt, got, EPS, f"shared {which}")
    rep = _np(_solve(eng, bt, dev, st))
    assert np.array_equal(rep[3], got[3])
    if which == "tiled":   # the shared set-up is the replicated arithmetic on the tiled kernel
        for a, b_ in zip(got[:5], rep[:5]):
            assert np.array_equal(a, b_, equal_nan=True)
    ok = ip.controls(bt)
    alone = _np(eng.solve(_t(bt.A_vals[0], dev), _t(bt.b[ok], dev), _t(bt.c[ok], dev), P0, st))
    assert np.array_equal(alone[4], got[4][ok])
    if which == "tiled":
        for a, b_ in zip(alone[:3], got[:3]):
            assert np.array_equal(a, b_[ok])


def test_cached_setup(cuda_device):
    """The cached set-up: filling the cache is the plain solve, bit for bit; the solve from it (reuse=1, which starts at the
    scale the filling solve ended with) reaches the same outcomes."""
    bt, dev = _batch("tiled_kr4"), cuda_device
    eng = Engine(bt.structure, dev)
    st = _settings(EPS)
    cache = eng.new_cache(bt.B)
    assert cache is not None
    fill = _np(_solve(eng, bt, dev, st, cache=cache))
    reuse = _np(_solve(eng, bt, dev, st, cache=cache, reuse=True))
    plain = _np(_solve(eng, bt, dev, st))
    _check_outcomes(bt, reuse, EPS, "cached")
    for a, c_ in zip(fill[:5], plain[:5]):
        assert np.array_equal(a, c_, equal_nan=True)


# ----------------------------------------------------------------------------- the iteration limit
@pytest.mark.parametrize("name", ["tiled_kr4", "dense_soc", "csr_mixed"])
def test_iteration_limit_matches_the_oracle(name, cuda_device, monkeypatch):
    bt, dev = _batch(name), cuda_device
    eng = _engine(name, dev, monkeypatch)
    sub = bt.select(ip.controls(bt))
    worst = 0.0
    for k in (1, 5, 37):
        st = make_settings({"eps": EPS, "max_iters": k})
        x, y, s, status, iters, _ = _np(_solve(eng, sub, dev, st))
        xo, yo, so, sto, ito = orc.solve_batch(sub.structure, sub.A_vals, sub.b, sub.c, sub.P_vals, eps=EPS, max_iters=k)
        assert np.array_equal(status, sto) and np.array_equal(iters, ito), (k, status, sto, iters, ito)
        fin = sto != -4
        for g, r in ((x, xo), (y, yo), (s, so)):
            assert np.array_equal(np.isnan(g), np.isnan(r))
            if fin.any():
                worst = max(worst, _rel(g[fin], r[fin]))
    print(f"{name}: iteration limit, worst against the oracle {worst:.1e}")
    assert worst <= LIMIT_TOL


@pytest.mark.parametrize("name", ["tiled_kr4", "csr_mixed"])
def test_no_positive_tau_is_failed(name, cuda_device, monkeypatch):
    """Certificates switched off (eps_infeas = 0): an infeasible instance reaches the limit with tau = 0 and comes back
    FAILED with NaN, not INACCURATE with values scaled by 1e12."""
    bt, dev = _batch(name), cuda_device
    eng = _engine(name, dev, monkeypatch)
    i = list(bt.aux["kinds"]).index("infeasible")
    sub = bt.select([i])
    args = {"eps": EPS, "max_iters": 2000, "eps_infeas": 0.0}
    x, y, s, status, iters, _ = _np(_solve(eng, sub, dev, make_settings(args)))
    _, _, _, sto, _ = orc.solve_batch(sub.structure, sub.A_vals, sub.b, sub.c, sub.P_vals, **args)
    assert status[0] == -4 and sto[0] == -4 and iters[0] == 2000, (status, sto, iters)
    assert np.isnan(x).all() and np.isnan(y).all() and np.isnan(s).all()


# ----------------------------------------------------------------------------- derivatives on a batch with NaN rows
BWD = {"lsqr_atol": 1e-12, "lsqr_btol": 1e-12, "lsqr_iter_lim": 2000}


@pytest.mark.parametrize("name,precond,kernel", [("tiled_nch1", 1, "fused"), ("tiled_nch1", 2, "block"), ("tiled_kr4", 2, "block"),
                                                 ("csr_mixed", 1, "generic")])
def test_derivatives_with_non_solved_rows(name, precond, kernel, cuda_device, monkeypatch):
    """vjp and jvp on the solve's own outputs, NaN rows included, finish; each solved instance's derivatives are the bits of
    the batch without the bad instances.  (The shared adjoint's batch sum is NaN by construction and is not checked.)"""
    if name == "tiled_nch1":
        bt = _MEMO.setdefault(name, _tiled(ts.CASES["nch1_live_eq_n"])())
    else:
        bt = _batch(name)
    dev = cuda_device
    eng = Engine(bt.structure, dev)
    print(name, kernel, eng.path_info()["bwd"])
    sol = _solve(eng, bt, dev, _settings(EPS))
    st_b = make_settings({**BWD, "lsqr_precond": precond})
    rng = np.random.default_rng(3)
    n, m = bt.structure.n, bt.structure.m
    dx, dy = _t(rng.standard_normal((bt.B, n)), dev), _t(rng.standard_normal((bt.B, m)), dev)
    tA, tb, tc = (_t(rng.standard_normal(a.shape), dev) for a in (bt.A_vals, bt.b, bt.c))
    tP = None if bt.P_vals is None else _t(rng.standard_normal(bt.P_vals.shape), dev)
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    g = eng.vjp(A, b, c, sol.x, sol.y, sol.s, dx, dy, P, st_b)
    j = eng.jvp(A, b, c, sol.x, sol.y, sol.s, tA, tb, tc, P, tP, st_b)
    torch.cuda.synchronize()
    ok = torch.as_tensor(ip.controls(bt), device=dev)
    sel = lambda t: None if t is None else t[ok].contiguous()  # noqa: E731
    g1 = eng.vjp(sel(A), sel(b), sel(c), sel(sol.x), sel(sol.y), sel(sol.s), sel(dx), sel(dy), sel(P), st_b)
    j1 = eng.jvp(sel(A), sel(b), sel(c), sel(sol.x), sel(sol.y), sel(sol.s), sel(tA), sel(tb), sel(tc), sel(P), sel(tP), st_b)
    for a, b_ in zip(g, g1):
        if a is not None:
            assert torch.equal(a[ok], b_), (name, kernel)
    for a, b_ in zip(j, j1):
        assert torch.equal(a[ok], b_), (name, kernel)
    assert all(bool(torch.isfinite(t[ok]).all()) for t in (*g[:4], *j[:3]) if t is not None)


# ----------------------------------------------------------------------------- warm start after a non-solved instance
@pytest.mark.parametrize("name", ["tiled_kr4", "dense_soc", "csr_mixed"])
def test_warm_start_with_a_non_finite_row_is_a_cold_start(name, cuda_device, monkeypatch):
    """An explicit warm start whose row k holds NaN (in x0, y0 or s0) or +-inf: instance k is solved as from cold (its bits on
    the deterministic paths, its status elsewhere); the other rows equal the all-finite warm call."""
    bt, dev = _batch(name), cuda_device
    eng = _engine(name, dev, monkeypatch)
    det = PATHS[name][4]
    sub = bt.select(ip.controls(bt))
    st = _settings(EPS)
    cold = _np(_solve(eng, sub, dev, st))
    w0 = [sub.x_star + 1e-3, sub.y_star.copy(), sub.s_star.copy()]
    warm = _np(_solve(eng, sub, dev, st, warm=tuple(_t(a, dev) for a in w0)))
    assert (cold[3] == 1).all() and (warm[3] == 1).all() and (warm[4] < cold[4]).all(), (cold[4], warm[4])
    k = 1
    for where, val in (("x", np.nan), ("y", np.nan), ("s", np.nan), ("x", np.inf), ("s", -np.inf)):
        w = [a.copy() for a in w0]
        w["xys".index(where)][k, 2] = val
        got = _np(_solve(eng, sub, dev, st, warm=tuple(_t(a, dev) for a in w)))
        assert got[3][k] == cold[3][k] and got[3][k] == 1, (where, val, got[3], got[4])
        rest = np.arange(sub.B) != k
        for q in range(6):
            if det:
                assert np.array_equal(got[q][k], cold[q][k]), (where, val, q)
                assert np.array_equal(got[q][rest], warm[q][rest]), (where, val, q)
            elif q < 3:
                assert _rel(got[q][k], cold[q][k]) <= 1e3 * EPS and _rel(got[q][rest], warm[q][rest]) <= NEIGHBOUR_TOL


def _layer_args(bt, **opts):
    from tests.test_gpu_boundary import _layer
    return _layer(bt, **opts)


@pytest.mark.parametrize("host_inputs", [False, True])
def test_layer_recovers_after_an_infeasible_call(host_inputs, cuda_device, monkeypatch):
    """{"warm_start": True}: the first call holds an infeasible instance and raises SolverError; the next call, same batch
    size, feasible data, succeeds and matches a cold call (the tolerance of
    test_warm_start_through_the_layer_matches_the_oracle).  host_inputs: pinned host tensors through the pipelined path."""
    import cvxpylayers_b200.interface as itf

    kinds = ("control", "infeasible", "control", "control")
    base = ts.planted(ts.CASES["kr4"], len(kinds), 21)
    bad = ip.mixed(base, kinds, seed=22)
    good = base.select(list(range(len(kinds))))
    if host_inputs:
        monkeypatch.setattr(itf, "PIPE_CHUNK", 2)
    args = {"eps": 1e-6, "max_iters": MAX_ITERS, "warm_start": True}
    ctx, _, cl = _layer_args(bad, **args)
    dev = cuda_device

    def call(bt_, cl_):
        bd = pr.to_boundary(bt_)
        if host_inputs:
            ctx.device = dev
            A, q, P = (torch.tensor(a).pin_memory() for a in (bd.A_eval, bd.q_eval, bd.P_eval))
        else:
            A, q, P = _t(bd.A_eval, dev), _t(bd.q_eval, dev), _t(bd.P_eval, dev)
        return _CvxpyLayer.apply(P, q, A, cl_, {}, False, None)

    with pytest.raises(SolverError):
        call(bad, cl)
    p2, d2, _, _ = call(good, cl)
    cctx, _, ccl = _layer_args(good, eps=1e-6, max_iters=MAX_ITERS)
    if host_inputs:
        cctx.device = dev
    pc, dc, _, _ = call(good, ccl)
    assert np.abs(p2.cpu().numpy() - pc.cpu().numpy()).max() < 1e-4
    assert np.abs(p2.cpu().numpy() - good.x_star).max() < 1e-4
