"""diffcp's ``mode="lsmr"`` on the host: the settings mapping, and the NumPy restatement of the kernels' LSMR
(``tests/lsmr_ref.py``) against SciPy's ``lsmr`` on the explicit adjoint and forward-mode systems of small solved instances.
The GPU suite (``test_gpu_lsmr.py``) then holds the kernels to SciPy directly."""
import numpy as np
import pytest
from scipy.sparse.linalg import lsmr as scipy_lsmr

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import make_settings
from oracle import oracle as orc
from tests import lsmr_ref
from tests.jvp_ref import dense_M, jvp_rhs, random_tangents


def test_make_settings_maps_the_mode():
    assert make_settings(None).lsmr == 0
    assert make_settings({"mode": "lsqr"}).lsmr == 0
    st = make_settings({"mode": "lsmr", "lsqr_atol": 1e-10, "lsqr_precond": 1})
    assert st.lsmr == 1 and st.lsqr_atol == 1e-10 and st.lsqr_precond == 1
    for bad in ("dense", "LSMR", "cg", None):
        with pytest.raises(ValueError):
            make_settings({"mode": bad})


def _solved(name, B, seed=0):
    bt = pr.CONFIGS[name](B=B, seed=seed)
    xo, yo, so, sto, _ = orc.solve_batch(bt.structure, bt.A_vals, bt.b, bt.c, bt.P_vals, eps=1e-10, max_iters=400000)
    assert (sto == 1).all()
    return bt, xo, yo, so


def _systems(name):
    """(matrix, right-hand side) of the adjoint (M', dz) and the forward mode (M, g) of two solved instances."""
    bt, xo, yo, so = _solved(name, 2)
    st, rng = bt.structure, np.random.default_rng(3)
    t = random_tangents(bt, rng)
    out = []
    for i in range(bt.B):
        P = bt.P_dense(i) if bt.P_vals is not None else None
        args = (st, bt.A_dense(i), P, bt.b[i], bt.c[i], xo[i], yo[i], so[i])
        M, dz, _, _ = lsmr_ref.adjoint_system(*args, rng.standard_normal(st.n), rng.standard_normal(st.m))
        out.append((M.T, dz))
        _, _, piy = dense_M(*args)
        dP = t.P_dense(i) if t.P_vals is not None else None
        out.append((M, jvp_rhs(bt.A_dense(i), xo[i], piy, t.A_dense(i), dP, t.b[i], t.c[i])))
    return out


@pytest.mark.parametrize("name", ["C1", "C3", "EXP"])
def test_restatement_reproduces_scipy_iterates_and_stop(name):
    for Bm, rhs in _systems(name):
        N = Bm.shape[1]
        x, itn, its = lsmr_ref.lsmr(Bm, rhs, iter_lim=40)
        scale = np.abs(its[-1]).max()
        for k in (1, 3, 10, 40):
            if k > itn:
                continue
            xs = scipy_lsmr(Bm, rhs, atol=1e-8, btol=1e-8, conlim=1e8, maxiter=k)[0]
            assert np.abs(its[k - 1] - xs).max() <= 1e-10 * max(np.abs(xs).max(), scale), (name, k)
        # the default rules: the same stopping iteration and solution as SciPy at the engine's limit of 2N
        x, itn, _ = lsmr_ref.lsmr(Bm, rhs)
        xs, istop, itn_s = scipy_lsmr(Bm, rhs, atol=1e-8, btol=1e-8, conlim=1e8, maxiter=2 * N)[:3]
        assert itn == itn_s and istop in (1, 2, 3, 7), (name, itn, itn_s, istop)
        assert np.abs(x - xs).max() <= 1e-9 * np.abs(xs).max()


def test_restatement_zero_right_hand_side_and_tight_tolerances():
    (Bm, rhs), _ = _systems("C1")[:2]
    x, itn, _ = lsmr_ref.lsmr(Bm, np.zeros_like(rhs))
    assert itn == 0 and not x.any()
    x, itn, _ = lsmr_ref.lsmr(Bm, rhs, atol=1e-12, btol=1e-12)
    xs, _, itn_s = scipy_lsmr(Bm, rhs, atol=1e-12, btol=1e-12, conlim=1e8, maxiter=2 * Bm.shape[1])[:3]
    assert itn == itn_s
    assert np.abs(x - xs).max() <= 1e-9 * np.abs(xs).max()
