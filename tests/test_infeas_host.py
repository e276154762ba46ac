"""CPU checks of tests/infeas_planted.py -- what its batches promise -- and the C oracle's status on them, plus the
oracle's rule for a non-finite warm start."""
from __future__ import annotations

import numpy as np
import pytest

from cvxpylayers_b200.problems import svec_to_mat
from oracle import oracle as orc
from tests import cone_planted as cp
from tests import cone_ref as cr
from tests import infeas_planted as ip
from tests import tiled_shapes as ts

MARGIN = 1e-3   # every certificate and slack block lies this far inside its cone, relative to the block's norm
ORACLE = {"eps": 1e-6, "max_iters": 20000}


def _cases():
    """name -> (batch factory, oracle settings)."""
    out = {}
    for name in ("mixed", "soc_sizes", "psd_warm", "psd_serial", "exp"):
        out[name] = (lambda name=name: ip.mixed(cp.make(name, B=len(ip.MIX)), seed=1), ORACLE)
    # blocks of magnitudes 1e-6 ... 1e3 in one instance: the termination test is relative to the largest block (test_gpu_cones)
    # (its last control needs more than 20000 iterations even at eps 1e-5)
    out["mixed_scales"] = (lambda: ip.mixed(cp.make("mixed_scales", B=6), ip.MIX[:6], seed=1), {"eps": 1e-5, "max_iters": 20000})
    for sc in (1e-4, 1e3):
        out[f"mixed_x{sc:g}"] = (lambda sc=sc: ip.mixed(cp.make("mixed", B=len(ip.MIX)), seed=2, scale=sc), ORACLE)
    out["mixed_block_scales"] = (lambda: ip.mixed(cp.make("mixed", B=len(ip.MIX)), seed=3, block_scale=(1e-6, 1e3)), ORACLE)
    out["mixed_shared"] = (lambda: ip.shared(cp.make("mixed", B=len(ip.SHARED_MIX)), seed=4), ORACLE)
    for cname in ("kr4", "n_gt_m", "all_equality"):
        kinds = ip.MIX_NO_SLACK if cname == "all_equality" else ip.MIX
        out[f"tiled_{cname}"] = (lambda cname=cname, kinds=kinds: ip.mixed(ts.planted(ts.CASES[cname], len(kinds), 5), kinds, seed=6), ORACLE)
    out["tiled_shared"] = (lambda: ip.shared(ts.planted(ts.CASES["kr4"], len(ip.SHARED_MIX), 7, shared=True), seed=8), ORACLE)
    return out


CASES = _cases()
_MEMO: dict = {}


def _get(name):
    if name not in _MEMO:
        _MEMO[name] = CASES[name][0]()
    return _MEMO[name]


def _margin_in(kind, v, k, dual):
    """How far v lies inside its block's cone (K* if ``dual``), relative to |v|; +inf for the zero cone."""
    nv = max(np.linalg.norm(v), 1e-300)
    if kind == "z":
        return np.inf if dual else (np.inf if not v.any() else -np.inf)
    if kind == "l":
        return v[0] / nv
    if kind == "q":
        return (v[0] - np.linalg.norm(v[1:])) / nv
    if kind == "s":
        return np.linalg.eigvalsh(svec_to_mat(v, k)).min() / nv
    in_exp = (kind == "ep") != dual
    proj = cr.proj_exp(v) if in_exp else cr.proj_exp_dual(v)   # 120-digit reference: v must be its own projection
    assert np.abs(proj - v).max() <= 1e-14 * nv, (kind, v, proj)
    r, s, t = v
    if in_exp:    # s > 0, s e^{r/s} <= t
        return min(s, t - s * np.exp(r / s)) / nv
    return min(-r, np.e * t + r * np.exp(s / r)) / nv   # r < 0, -r e^{s/r} <= e t


def _blockwise_margin(cones, v, dual):
    return min(_margin_in(kind, v[r:r + rows], k, dual) for kind, r, rows, k in ip.blocks(cones))


@pytest.mark.parametrize("name", list(CASES))
def test_certificates_rays_and_pattern(name):
    bt = _get(name)
    st, aux = bt.structure, bt.aux
    for i, kind in enumerate(aux["kinds"]):
        A, P, b, c = bt.A_dense(i), bt.P_dense(i), bt.b[i], bt.c[i]
        nA = np.abs(A).max()
        if kind == "infeasible":
            y = aux["y_cert"][i]
            assert np.abs(A.T @ y).max() <= 1e-13 * nA * np.linalg.norm(y), (i, np.abs(A.T @ y).max())
            assert abs(b @ y + 1.0) <= 1e-13 * max(1.0, np.abs(b) @ np.abs(y)), (i, b @ y)   # (the dot product's rounding)
            assert _blockwise_margin(st.cones, y, True) >= MARGIN and (y != 0).all(), i
        elif kind.startswith("unbounded"):
            xd, sd = aux["x_ray"][i], aux["s_ray"][i]
            assert np.linalg.norm(A @ xd + sd) <= 1e-13 * nA * np.linalg.norm(xd), i
            assert np.linalg.norm(P @ xd) <= 1e-13 * max(1.0, np.abs(P).max()) * np.linalg.norm(xd), i
            assert abs(c @ xd + 1.0) <= 1e-13 * max(1.0, np.abs(c) @ np.abs(xd)), (i, c @ xd)
            if kind == "unbounded":   # (the zero-column ray has s_d = 0 and touches one variable)
                assert _blockwise_margin(st.cones, sd, False) >= MARGIN and (xd != 0).all(), i
            else:
                assert not sd.any() and np.count_nonzero(xd) == 1 and not A[:, xd != 0].any() and not P[:, xd != 0].any()
        else:   # a planted optimum: feasible, complementary, stationary
            x, y, s = bt.x_star[i], bt.y_star[i], bt.s_star[i]
            sc = max(1.0, np.abs(b).max(), np.abs(c).max())
            assert np.abs(A @ x + s - b).max() <= 1e-12 * sc and np.abs(P @ x + A.T @ y + c).max() <= 1e-12 * sc, i
            assert abs(s @ y) <= 1e-12 * sc * max(1.0, np.linalg.norm(y)), i
            if kind == "control_near":
                yc = aux["y_cert"][i]
                assert np.abs(A.T @ yc).max() <= 1e-13 * nA * np.linalg.norm(yc)
                ratio = (s @ yc) / (np.linalg.norm(b) * np.linalg.norm(yc))   # (per-block scales change the norms)
                assert 0.5 * ip.NEAR <= ratio <= 2 * ip.NEAR or aux["block_scale"], (i, ratio)
    # the sparsity pattern: only the structure's positions carry values (the CSR values are A's, in order)
    M = ip._mask(st)
    for i in range(bt.B):
        assert np.array_equal(bt.A_dense(i)[M], bt.A_vals[i]) and not bt.A_dense(i)[~M].any()
    if aux["shared"]:
        assert (bt.A_vals == bt.A_vals[0]).all() and (bt.P_vals is None or (bt.P_vals == bt.P_vals[0]).all())


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_returns_the_planted_status(name):
    bt = _get(name)
    args = CASES[name][1]
    x, y, s, status, iters = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, **args)
    assert np.array_equal(status, bt.aux["status"]), (status, iters)
    assert (iters < args["max_iters"]).all(), iters
    bad = bt.aux["status"] != 1
    assert np.isnan(x[bad]).all() and np.isnan(y[bad]).all() and np.isnan(s[bad]).all()
    ok = ip.controls(bt)
    tol = 1e3 * args["eps"]
    for got, ref in ((x, bt.x_star), (s, bt.s_star)):
        err = np.abs(got[ok] - ref[ok]).max() / max(1.0, np.abs(ref[ok]).max())
        assert err <= tol, (name, err)


def test_scaled_certificates_keep_their_normalisation():
    """(A, b) -> D (A, b) per block: the certificate becomes D^-1 y and still has b'y = -1."""
    base = cp.make("mixed", B=len(ip.MIX))
    a, d = ip.mixed(base, seed=3), ip.mixed(base, seed=3, block_scale=(1e-6, 1e3))
    i = ip.MIX.index("infeasible")
    D = d.b[i] / a.b[i]
    assert np.allclose(d.aux["y_cert"][i] * D, a.aux["y_cert"][i], rtol=1e-14, atol=0)


# ----------------------------------------------------------------------------- the oracle's warm start from a non-finite row
def test_oracle_warm_start_from_a_non_finite_row_is_a_cold_start():
    """A warm-start row with NaN (a non-solved instance's outputs) or +-inf starts that instance cold: the cold solve's bits;
    the other rows keep their warm start."""
    bt = ip.mixed(cp.make("mixed", B=len(ip.MIX)), seed=1)
    ok = ip.controls(bt)
    sub = bt.select(ok)
    st = bt.structure
    cold = orc.solve_batch(st, sub.A_vals, sub.b, sub.c, sub.P_vals, **ORACLE)
    warm0 = (sub.x_star + 1e-3, sub.y_star, sub.s_star)
    warm = orc.solve_batch(st, sub.A_vals, sub.b, sub.c, sub.P_vals, warm=warm0, **ORACLE)
    assert (warm[4] < cold[4]).all()
    for where, val in (("x", np.nan), ("y", np.nan), ("s", np.nan), ("x", np.inf), ("s", -np.inf)):
        w = [a.copy() for a in warm0]
        w["xys".index(where)][1, 3] = val
        got = orc.solve_batch(st, sub.A_vals, sub.b, sub.c, sub.P_vals, warm=tuple(w), **ORACLE)
        for k in range(5):
            assert np.array_equal(got[k][1], cold[k][1]), (where, val, k)
            assert np.array_equal(np.delete(got[k], 1, 0), np.delete(warm[k], 1, 0)), (where, val, k)


def test_oracle_warm_start_after_an_infeasible_solve():
    """The outputs of an infeasible solve (NaN) as the next call's warm start: the feasible data solves as from cold."""
    from cvxpylayers_b200.structure import ConeSpec, Structure
    st = Structure.dense(1, 2, ConeSpec(l=2))
    A, c = np.array([[1.0, -1.0]]), np.array([[0.0]])
    x, y, s, status, _ = orc.solve_batch(st, A, np.array([[-1.0, -1.0]]), c, eps=1e-6, max_iters=2000)
    assert status[0] == -2 and np.isnan(x).all()
    cold = orc.solve_batch(st, A, np.array([[1.0, 1.0]]), c, eps=1e-6, max_iters=2000)
    warm = orc.solve_batch(st, A, np.array([[1.0, 1.0]]), c, eps=1e-6, max_iters=2000, warm=(x, y, s))
    assert cold[3][0] == 1 and all(np.array_equal(a, b) for a, b in zip(cold, warm))
