"""Forward mode with the equilibrated LSQR (lsqr_precond = 1) when the data tangent lives only in rows of inactive nonneg
constraints: the equilibration drops those rows from the scaled system, so its right-hand side is exactly zero.  The solution of
the scaled system is then 0 and the dropped rows' unknowns come from their own equations; the tangent must be finite and agree
with the plain LSQR (lsqr_precond = 0), which keeps every row."""
import numpy as np
import pytest
import torch

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(10, 20, 0), (8, 14, 3)])   # C1's shape (inequality rows only), and one with equalities
def test_tangent_on_inactive_rows_only(shape, cuda_device):
    n, m, z = shape
    dev = cuda_device
    bt = pr.dense_qp(2, n, m, z, seed=12)
    st = bt.structure
    eng = Engine(st, dev)
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
            outs = {}
            for pc in (0, 1):
                S = make_settings({"lsqr_precond": pc, "lsqr_atol": 1e-12, "lsqr_btol": 1e-12})
                outs[pc] = eng.jvp(A, b, c, sol.x, sol.y, sol.s, tA, zb, zc, P, zP, S)
            for a_, b_ in zip(outs[1][:3], outs[0][:3]):
                assert bool(torch.isfinite(a_).all())
                assert float((a_ - b_).abs().max()) <= 1e-6 * max(1.0, float(b_.abs().max()))
