"""The shape classes of the register-tiled forward (tests/tiled_shapes.py) against libbcone.so's own eligibility and
shared-memory rules: a change to fwd_fast.cu's Geo that empties a class or moves a chosen shape out of the domain fails here,
on the CPU, instead of leaving tests/test_gpu_tiled_shapes.py to test other shapes than it names."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import tiled_shapes as ts


def test_domain_has_the_documented_size_and_ranges():
    dom = ts.domain()
    ns, ms = [n for n, _ in dom], [m for _, m in dom]
    assert len(dom) == ts.DOMAIN_SIZE
    assert (min(ns), max(ns)) == ts.N_RANGE and (min(ms), max(ms)) == ts.M_RANGE
    assert max(ts.smem_bytes(*s) for s in dom) <= ts.SMEM_OPTIN


@pytest.mark.parametrize("name", list(ts.CLASSES))
def test_class_is_not_empty_and_holds_its_representative(name):
    cls = ts.CLASSES[name]
    case = ts.CASES[cls.case]
    members = ts.class_members(name)
    print(f"{name}: {len(members)} shapes, representative {case.id}")
    assert members, f"class {name} ({cls.what}) is empty"
    assert cls.rule(case.n, case.m), f"{case.id} is not in class {name} ({cls.what})"
    assert cls.case_rule is None or cls.case_rule(case), f"{case.id} does not have what class {name} needs ({cls.what})"


@pytest.mark.parametrize("key", list(ts.CASES))
def test_chosen_shape_takes_the_tiled_forward(key):
    c = ts.CASES[key]
    assert ts.eligible(c.n, c.m), c.id
    assert ts.smem_bytes(c.n, c.m) <= ts.SMEM_OPTIN, (c.id, ts.smem_bytes(c.n, c.m))
    g = ts.Geo(c.n, c.m)
    assert ts.cache_doubles(c.n, c.m) >= 8 + g.npad + g.mpad + c.n * g.kst   # header, E, D and K^-1 at the stride restated here


def test_chosen_shapes_cover_the_issue_examples():
    """The explicit shapes, z = 0, z = m with m < n, an LP, two odd nnzP with P and the fused adjoint's NCH pair."""
    shapes = {(c.n, c.m) for c in ts.CASES.values()}
    for s in [(110, 136), (101, 93), (102, 100), (11, 509), (40, 512), (91, 197), (99, 199), (57, 333), (110, 93), (64, 160), (66, 160), (30, 341)]:
        assert s in shapes, s
    cases = list(ts.CASES.values())
    assert any(c.z == 0 for c in cases) and any(c.z == c.m < c.n for c in cases) and any(not c.P for c in cases)
    assert sum(c.P and c.nnzP % 2 == 1 for c in cases) >= 2
    assert ts.Geo(91, 197).kst == 106 and ts.Geo(110, 136).KR == 4 and ts.Geo(11, 509).CT * ts.Geo(11, 509).RTu == 256


@pytest.mark.parametrize("key", ["kr4", "lp_vertex", "nch1_live_eq_n", "all_equality"])
@pytest.mark.parametrize("shared", [False, True])
def test_planted_optimum_is_a_strictly_complementary_kkt_point(key, shared):
    """The generator's promise: KKT holds at (x*, y*, s*), exactly ``active`` nonneg rows are active, complementarity is
    strict and the live rows are independent (with n of them in an LP, so x* is the unique vertex)."""
    c = ts.CASES[key]
    bt = ts.planted(c, B=3, seed=5, shared=shared)
    for i in range(bt.B):
        A, P = bt.A_dense(i), bt.P_dense(i)
        x, y, s = bt.x_star[i], bt.y_star[i], bt.s_star[i]
        assert np.abs(A @ x + s - bt.b[i]).max() < 1e-12 and np.abs(P @ x + A.T @ y + bt.c[i]).max() < 1e-12
        assert (s[:c.z] == 0).all()
        l_y, l_s = y[c.z:], s[c.z:]
        assert (l_y >= 0).all() and (l_s >= 0).all() and (l_y * l_s == 0).all()
        assert int((l_y > 0).sum()) == c.active and ((l_y > 0.4) | (l_s > 0.4)).all()
        live = np.concatenate([np.arange(c.z), c.z + np.nonzero(l_y)[0]])
        assert np.linalg.matrix_rank(A[live]) == live.size
        if shared:
            assert np.array_equal(bt.A_vals[i], bt.A_vals[0]) and (bt.P_vals is None or np.array_equal(bt.P_vals[i], bt.P_vals[0]))


def test_oracle_solves_the_lp_batches_of_the_gpu_tests():
    """Operator splitting can crawl on an LP vertex: the C oracle (the same algorithm) reaches eps 1e-10 within the GPU tests'
    iteration limit on every LP batch they draw, and lands on the planted vertex."""
    from tests import test_gpu_tiled_shapes as T

    for key, c in ts.CASES.items():
        if c.P:
            continue
        bt = T._batch(key)
        for b in (bt, ts.replant(bt, c, seed=T._replant_seed(key)), T._batch(key, shared=True)):
            x, y, s, status, iters = orc.solve_batch(b.structure, b.A_vals, b.b, b.c, None, eps_abs=T.FWD["eps_abs"],
                                                     eps_rel=T.FWD["eps_rel"], max_iters=T.FWD["max_iters"])
            assert (status == 1).all(), (c.id, status, iters)
            assert np.abs(x - b.x_star).max() < 1e-6, c.id
