"""CPU tests of the host side of batch-shared matrices: the layer's ``shared_matrices`` option, its check that every parameter
feeding A or P is unbatched, and its exclusion of the cached set-up."""
import numpy as np
import pytest
import scipy.sparse as sp

from cvxpylayers_b200 import interface as itf
from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import make_settings


def _ctx():
    from tests.util import fake_param_prob

    bt = pr.dense_qp(2, 6, 9, 2, seed=3)
    problem, params = fake_param_prob(bt)
    pp = problem["param_prob"]
    ctx = itf.get_solver_ctx("B200", pp, problem["dims"], {}, None)
    sizes = [p.shape[1] for p in params]   # parameters, in order: A_cvx values + b, c, P (fake_param_prob)
    return bt, pp, ctx, sizes


def test_shared_matrices_is_a_layer_option_not_a_solver_setting():
    st = make_settings({"shared_matrices": True, "eps": 1e-6})
    assert st.eps_abs == 1e-6


def test_batched_matrix_parameter_is_refused_by_name():
    _, _, ctx, sizes = _ctx()
    order = [0, 1, 2]
    ctx.check_shared_matrices(sizes, [False, True, False], order)          # only c batched: fine
    with pytest.raises(ValueError, match="parameter 0"):
        ctx.check_shared_matrices(sizes, [True, True, False], order)       # A (and b) batched
    with pytest.raises(ValueError, match="parameter 2"):
        ctx.check_shared_matrices(sizes, [False, True, True], order)       # P batched
    # rows follow the column order, not the user order: user parameter 1 is A here
    ctx.check_shared_matrices([sizes[1], sizes[0], sizes[2]], [True, False, False], [1, 0, 2])
    with pytest.raises(ValueError, match="parameter 1"):
        ctx.check_shared_matrices([sizes[1], sizes[0], sizes[2]], [False, True, False], [1, 0, 2])


def test_parameter_feeding_only_b_may_be_batched():
    bt, pp, ctx, sizes = _ctx()
    A_map, q_map, P_map = pp.reduced_A.reduced_mat, pp.q, pp.reduced_P.reduced_mat
    nA, P1 = bt.structure.nnzA, A_map.shape[1]
    const = sp.csr_matrix((np.ones(nA), (np.arange(nA), np.full(nA, P1 - 1))), shape=(nA, P1))
    ctx.set_param_maps(sp.vstack([const, A_map.tocsr()[nA:]]).tocsr(), q_map, P_map)   # parameter 0 now feeds b only
    ctx.check_shared_matrices(sizes, [True, True, False], [0, 1, 2])
    with pytest.raises(ValueError, match="parameter 2"):
        ctx.check_shared_matrices(sizes, [True, True, True], [0, 1, 2])


def test_shared_matrices_and_the_cached_set_up_exclude_each_other():
    _, _, ctx, _ = _ctx()
    ctx.PA_is_constant = True   # would switch the cached set-up on by default
    assert ctx.setup_cache(None, "cpu", 2, {"shared_matrices": True}) is None
    with pytest.raises(ValueError, match="reuse_setup"):
        ctx.setup_cache(None, "cpu", 2, {"shared_matrices": True, "reuse_setup": True})


def test_registered_layer_refuses_a_batched_matrix_parameter(monkeypatch):
    """Through register() and the stand-in cvxpylayers package: the registered forward checks the parameters before any solve."""
    import torch

    from tests.util import fake_param_prob, install_fake_cvxpylayers

    fake = install_fake_cvxpylayers(monkeypatch)
    bt = pr.dense_qp(3, 6, 9, 2, seed=1)
    problem, params = fake_param_prob(bt)
    itf.register(fuse=True)
    th = [torch.tensor(p) for p in params]   # every parameter batched, A's and P's included
    layer = fake.tl.CvxpyLayer(problem, [], [], solver="B200", solver_args={"shared_matrices": True})
    with pytest.raises(ValueError, match="shared_matrices: parameter 0 feeds A or P but is batched"):
        layer(*th)
    layer = fake.tl.CvxpyLayer(problem, [], [], solver="B200")
    with pytest.raises(ValueError, match="shared_matrices: parameter 0"):   # the option per call, as solver_args
        layer(*th, solver_args={"shared_matrices": True})
