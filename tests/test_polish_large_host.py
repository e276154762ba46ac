"""Solution polishing past the on-chip limit (n > 128: csrc/polish_large.cu), on the CPU: the NumPy restatement
(tests/polish_ref.py) recovers the planted optimum at the sizes the slab tier polishes -- a sparse LP at a vertex (n = 300,
m = 600), a dense QP (n = 200), a sparse QP with a diagonal P (n = 300) and a CSR QP with a general sparse P (n = 160) --
starting from the planted optimum perturbed by 1e-3 on the planted active set.  The batch builders and the perturbation are
shared with tests/test_gpu_polish_large.py."""
from __future__ import annotations

import numpy as np
import pytest

from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.structure import ConeSpec, Structure
from tests import polish_ref as pref
from tests import tiled_shapes as ts


def csr_general_p_qp(B, n, m, z, seed):
    """A random CSR pattern for A (about a tenth of the entries, every row non-empty) and a sparse upper-triangular P pattern
    with off-diagonal entries (the diagonal plus about 5 % of the rest), P diagonally dominant, planted by problems.plant."""
    rng = np.random.default_rng(seed)
    mask = rng.random((m, n)) < 0.1
    mask[np.arange(m), rng.integers(0, n, m)] = True
    indptr = np.r_[0, np.cumsum(mask.sum(1))].astype(np.int32)
    indices = np.nonzero(mask)[1].astype(np.int32)
    pm = np.triu(rng.random((n, n)) < 0.05, 1) | np.eye(n, dtype=bool)
    p_indptr = np.r_[0, np.cumsum(pm.sum(1))].astype(np.int32)
    p_rows, p_cols = np.nonzero(pm)
    st = Structure(n, m, indptr, indices, ConeSpec(z=z, l=m - z), p_indptr, p_cols.astype(np.int32))
    A = rng.standard_normal((B, indices.size)) / np.sqrt(n * 0.1)
    P = np.zeros((B, p_cols.size))
    off = p_rows != p_cols
    P[:, off] = 0.3 * rng.standard_normal((B, int(off.sum())))
    for i in range(B):   # diagonal: 0.5 + the absolute row sum of the symmetric off-diagonal part
        rs = np.zeros(n)
        np.add.at(rs, p_rows[off], np.abs(P[i, off]))
        np.add.at(rs, p_cols[off], np.abs(P[i, off]))
        P[i, ~off] = 0.5 + rs[p_rows[~off]]
    return pr.plant(st, A, P, rng, name=f"csr_general_p_qp_n{n}", active_frac=0.2)


def large_batches():
    """name -> builder of the planted batches the slab tier is checked on (every one strictly complementary)."""
    return {
        "sparse_lp_300": lambda: pr.sparse_lp(3, 300, 600, density=0.05, seed=1),
        "dense_qp_200": lambda: ts.planted(ts.Case(200, 300, 50, 60, True, 0), 3, seed=2),
        "sparse_qp_300": lambda: pr.sparse_qp(3, 300, 600, seed=3),
        "csr_general_p_160": lambda: csr_general_p_qp(3, 160, 200, 20, seed=4),
    }


def perturbed_start(bt, seed, eps=1e-3):
    """The planted optimum moved by up to ``eps`` without changing the active set it names: x and the zero rows' y anywhere,
    y up on the active nonneg rows, s up on the inactive ones."""
    rng = np.random.default_rng(seed)
    z = bt.structure.cones.z
    x = bt.x_star + eps * rng.uniform(-1, 1, bt.x_star.shape)
    y, s = bt.y_star.copy(), bt.s_star.copy()
    y[:, :z] += eps * rng.uniform(-1, 1, (bt.B, z))
    act = bt.y_star[:, z:] > 0
    y[:, z:] += np.where(act, eps * rng.uniform(0.1, 1, act.shape), 0.0)
    s[:, z:] += np.where(act, 0.0, eps * rng.uniform(0.1, 1, act.shape))
    return x, y, s


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.mark.parametrize("key", list(large_batches()))
def test_restatement_recovers_the_planted_optimum_past_the_on_chip_limit(key):
    bt = large_batches()[key]()
    assert bt.structure.n > 128
    x, y, s = perturbed_start(bt, seed=7)
    flags, X, Y, S = pref.polish_batch(bt, x, y, s, np.ones(bt.B, dtype=np.int32))
    assert (flags == 1).all(), (key, flags)
    err = max(_rel(X, bt.x_star), _rel(Y, bt.y_star), _rel(S, bt.s_star))
    assert err < 1e-9, (key, err)
    assert _rel(x, bt.x_star) > 1e3 * err   # (the start really was inexact)


def test_perturbed_start_names_the_planted_active_set():
    bt = large_batches()["sparse_qp_300"]()
    x, y, s = perturbed_start(bt, seed=7)
    z = bt.structure.cones.z
    assert np.array_equal(y[:, z:] > s[:, z:], bt.y_star[:, z:] > 0)
