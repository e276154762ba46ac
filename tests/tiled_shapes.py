"""Shapes of the register-tiled forward (fwd_fast.cu) and planted dense batches for them -- TEST INFRASTRUCTURE.

The domain -- the (n, m) that take the register-tiled forward when A is dense and every row is a zero or nonneg row -- comes
from libbcone.so itself: ``bc_fwdf_eligible(n, m)`` and ``bc_fwdf_smem_bytes(n, m) <= SMEM_OPTIN``, the rule ``bcone_create``
applies.  The shape classes below restate ``Geo`` of fwd_fast.cu (CT, RTu, KR, the compile-time ``<10, 50>`` instantiation and
its padded K^-1 row stride); each names what only its shapes exercise.  tests/test_tiled_shapes_host.py checks on the CPU that
every class is non-empty, that every chosen shape is in the domain and in its class, and that the domain still has the size
and ranges written here, so a change to ``Geo`` that empties a class or moves a chosen shape out fails there, not silently in
the GPU tests (tests/test_gpu_tiled_shapes.py).

``planted`` draws dense QPs and LPs whose optimum is planted with an exact number of active rows, so the optimum is unique
and the solution map is differentiable there (see its docstring).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from functools import lru_cache

import numpy as np

from cvxpylayers_b200 import _lib
from cvxpylayers_b200.problems import Batch
from cvxpylayers_b200.structure import ConeSpec, Structure

SMEM_OPTIN = 232448   # H100: shared memory per CTA with the opt-in attribute (227 KB)
FT, TR, TC = 512, 4, 10   # fwd_fast.cu: threads per CTA, rows and columns of a thread's register tile of A

# the domain at SMEM_OPTIN, n, m <= 512 (re-derived from the library by tests/test_tiled_shapes_host.py)
DOMAIN_SIZE = 13520
N_RANGE = (11, 110)
M_RANGE = (93, 512)


@lru_cache(maxsize=None)
def _fns():
    lib = _lib.load()
    for name in ("bc_fwdf_eligible", "bc_fwdf_smem_bytes", "bc_fwdf_cache_doubles"):
        getattr(lib, name).argtypes = [C.c_int, C.c_int]
    lib.bc_fwdf_eligible.restype = C.c_int
    lib.bc_fwdf_smem_bytes.restype = C.c_size_t
    lib.bc_fwdf_cache_doubles.restype = C.c_size_t
    return lib


def eligible(n: int, m: int) -> bool:
    return bool(_fns().bc_fwdf_eligible(n, m))


def smem_bytes(n: int, m: int) -> int:
    return int(_fns().bc_fwdf_smem_bytes(n, m))


def cache_doubles(n: int, m: int) -> int:
    return int(_fns().bc_fwdf_cache_doubles(n, m))


def in_domain(n: int, m: int) -> bool:
    return eligible(n, m) and smem_bytes(n, m) <= SMEM_OPTIN


@lru_cache(maxsize=None)
def domain() -> tuple:
    """Every (n, m) with n, m <= 512 that takes the register-tiled forward on an H100."""
    return tuple((n, m) for n in range(1, FT + 1) for m in range(1, FT + 1) if in_domain(n, m))


# ----------------------------------------------------------------------------- Geo of fwd_fast.cu, restated
@dataclass(frozen=True)
class Geo:
    n: int
    m: int

    @property
    def CT(self):   # column tiles
        return -(-self.n // TC)

    @property
    def RTu(self):   # row tiles
        return -(-self.m // TR)

    @property
    def npad(self):
        return self.CT * TC

    @property
    def mpad(self):
        return self.RTu * TR

    @property
    def KR(self):   # rows per tile of the K^-1 product (kinv_rows<KR>)
        return 2 if (self.npad // 2) * self.CT <= FT else 4

    @property
    def compile_time(self):   # bc_fwdf_kernel: fwd_fast_kernel<10, 50>; every other shape runs <0, 0>
        return self.CT == 10 and self.RTu == 50

    @property
    def kst(self):   # K^-1 row stride: padded to a conflict-free stride in the compile-time instantiation only
        return self.npad + ((10 - (self.npad & 7)) & 7) if (self.compile_time and self.KR == 2) else self.npad


# ----------------------------------------------------------------------------- the chosen shapes
@dataclass(frozen=True)
class Case:
    """One planted batch: n variables, m rows of which z are equalities and ``active`` of the m - z nonneg rows active at
    the optimum; ``P``: a quadratic term; ``bwd``: the adjoint kernel bcone_create picks (``Engine.BWD_PATHS`` index:
    0 generic, 1 fused, 2 KKT-block with the fused kernel as fallback)."""
    n: int
    m: int
    z: int
    active: int
    P: bool
    bwd: int

    @property
    def id(self) -> str:
        return f"n{self.n}_m{self.m}_z{self.z}_a{self.active}" + ("" if self.P else "_lp")

    @property
    def nnzP(self) -> int:
        return self.n * (self.n + 1) // 2 if self.P else 0


# The fused adjoint needs an even n <= 128; the KKT-block one in addition a quadratic term.
CASES = {
    "kr4": Case(110, 136, 30, 60, True, 2),            # KR = 4 at the largest layout (232,304 B); nnzP odd
    "n_gt_m": Case(101, 93, 10, 50, True, 0),           # nnzP = 5151 odd; generic adjoint
    "n_gt_m_fused": Case(102, 100, 20, 50, True, 2),    # n > m with an even n: the fused and the KKT-block adjoint; nnzP odd
    "all_equality": Case(110, 93, 93, 0, True, 2),      # l = 0: the zero-cone metric on every row; S does not fit beside W
    "half_cta": Case(11, 509, 0, 10, True, 0),         # CT RTu = 256; z = 0
    "lp_vertex": Case(30, 341, 10, 20, False, 1),       # LP at a vertex: z + active = n, no P; the fused adjoint without P
    "full_cta": Case(40, 512, 10, 20, True, 2),         # every thread holds a tile; fused adjoint at m = 512
    "compile_time_widest": Case(91, 197, 20, 40, True, 0),
    "odd_mn_compile_time": Case(99, 199, 50, 30, True, 0),
    "odd_mn": Case(57, 333, 0, 40, True, 0),            # nnzP = 1653 odd
    "nch1_live_eq_n": Case(64, 160, 24, 40, True, 2),   # NCH = 1; z + active = n: the block adjoint's nl <= n at its edge
    "nch2": Case(66, 160, 16, 30, True, 2),             # NCH = 2; nnzP = 2211 odd: the fused adjoint loads P without TMA
}


@dataclass(frozen=True)
class ShapeClass:
    what: str             # what only this class exercises
    rule: object          # (n, m) -> bool, within the domain
    case: str             # key of CASES: the representative
    case_rule: object = None   # Case -> bool: what the representative's batch must have beyond its shape


CLASSES = {
    "kr4": ShapeClass("kinv_rows<4> and its 4-row thread map", lambda n, m: Geo(n, m).KR == 4, "kr4"),
    "n_gt_m": ShapeClass("rowsR = npad: K larger than A's row space", lambda n, m: n > m, "n_gt_m"),
    "n_gt_m_even": ShapeClass("n > m through the fused and the KKT-block adjoint (even n)", lambda n, m: n > m and n % 2 == 0,
                              "n_gt_m_fused"),
    "smem_edge": ShapeClass("the largest layout bcone_create accepts (within 144 B of the limit)",
                            lambda n, m: smem_bytes(n, m) >= SMEM_OPTIN - 144, "kr4"),
    "half_cta": ShapeClass("CT RTu = 256: the act = false threads in every product, n << m",
                           lambda n, m: Geo(n, m).CT * Geo(n, m).RTu == FT // 2, "half_cta"),
    "full_cta_m512": ShapeClass("CT RTu = 512 at m = 512: every thread holds a tile, 16 output warps",
                                lambda n, m: Geo(n, m).CT * Geo(n, m).RTu == FT and m == FT, "full_cta"),
    "odd_mn": ShapeClass("odd m n: A staged by plain loads instead of the TMA bulk copy", lambda n, m: (n * m) % 2 == 1, "odd_mn"),
    "compile_time_widest": ShapeClass("<10, 50> with 9 padding columns and 3 padding rows: kst = 106 with most padding live",
                                      lambda n, m: Geo(n, m).compile_time and Geo(n, m).npad - n == 9 and Geo(n, m).mpad - m == 3,
                                      "compile_time_widest"),
    "compile_time_odd_mn": ShapeClass("<10, 50> with plain-load staging", lambda n, m: Geo(n, m).compile_time and (n * m) % 2 == 1,
                                      "odd_mn_compile_time"),
    "all_equality": ShapeClass("l = 0: the zero-cone metric on every row (n > m keeps the rows independent)",
                               lambda n, m: n > m, "all_equality", lambda c: c.z == c.m),
    "lp": ShapeClass("no quadratic term: an LP at a vertex", lambda n, m: True, "lp_vertex",
                     lambda c: not c.P and c.z + c.active == c.n),
    "equality_free": ShapeClass("z = 0", lambda n, m: True, "odd_mn", lambda c: c.z == 0),
    "odd_nnzP": ShapeClass("odd nnzP with P: P scattered / loaded without the bulk copy", lambda n, m: n % 4 in (1, 2),
                           "odd_mn", lambda c: c.P and c.nnzP % 2 == 1),
    "odd_nnzP_fused": ShapeClass("odd nnzP in the fused adjoint (tmaP = 0)", lambda n, m: n % 4 == 2, "nch2",
                                 lambda c: c.P and c.nnzP % 2 == 1),
    "fused_nch1": ShapeClass("bwd_fast_kernel<1> (even n <= 64)", lambda n, m: n % 2 == 0 and n <= 64, "nch1_live_eq_n"),
    "fused_nch2": ShapeClass("bwd_fast_kernel<2> (even 64 < n <= 128)", lambda n, m: n % 2 == 0 and 64 < n <= 128, "nch2"),
    "fused_m256": ShapeClass("the fused adjoint at m >= 256", lambda n, m: n % 2 == 0 and m >= 256, "full_cta"),
    "block_s_overflow": ShapeClass("live rows <= n whose S does not fit beside W: the KKT-block adjoint hands them on",
                                   lambda n, m: n % 2 == 0 and not block_takes(n, m, min(n, m)), "all_equality",
                                   lambda c: c.P and not block_takes(c.n, c.m, c.z + c.active)),
    "block_live_eq_n": ShapeClass("exactly n live rows in the KKT-block adjoint", lambda n, m: n % 2 == 0 and m >= n, "nch1_live_eq_n",
                                  lambda c: c.P and c.z + c.active == c.n),
}


def block_takes(n: int, m: int, live: int) -> bool:
    """bwd_block.cu's blk_fits, restated: the KKT-block adjoint takes an instance with ``live`` live rows when they are at most
    n and W (live x n) and S (live x live, packed) fit in the m n doubles the rows are staged in; otherwise the fused kernel
    re-runs it (counted by ``Engine.fallback_count``)."""
    return live <= n and live * n + live * (live + 1) // 2 <= ((m * n + 1) & ~1)


def class_members(name: str) -> list:
    rule = CLASSES[name].rule
    return [s for s in domain() if rule(*s)]


# ----------------------------------------------------------------------------- planted batches
def _plant_one(A, P, z, active, rng):
    """(b, c, x, y, s) for one dense A (m x n) and P (n x n or None) with exactly ``active`` nonneg rows active, chosen so that
    the live rows have a condition number below 100 (LICQ with margin: they determine y and, at a vertex, x; operator
    splitting slows down with it -- at 1e3 one planted LP vertex took the C oracle more than 4e5 iterations too)."""
    m, n = A.shape
    for _ in range(100):
        act = z + np.sort(rng.choice(m - z, active, replace=False))
        live = np.concatenate([np.arange(z), act])
        sv = np.linalg.svd(A[live], compute_uv=False) if live.size else np.ones(1)
        if sv[-1] > 1e-2 * sv[0]:
            break
    else:
        raise AssertionError(("no well-conditioned set of live rows", z, active, sv[-1] / sv[0]))
    x = rng.standard_normal(n)
    y, s = np.zeros(m), np.zeros(m)
    y[:z] = rng.standard_normal(z)
    y[act] = rng.uniform(0.5, 2.0, active)
    dead = np.setdiff1d(np.arange(z, m), act)
    s[dead] = rng.uniform(0.5, 2.0, dead.size)
    c = -A.T @ y - (P @ x if P is not None else 0.0)
    return A @ x + s, c, x, y, s


def _draw_AP(n, m, with_P, rng):
    A = rng.standard_normal((m, n)) / np.sqrt(n)
    if not with_P:
        return A, None
    L = rng.standard_normal((n, n))
    return A, L @ L.T / n + 0.1 * np.eye(n)


def planted(case: Case, B: int, seed: int, shared: bool = False) -> Batch:
    """B dense instances of ``case`` in the distribution of ``problems.dense_qp`` (A ~ N(0, 1) / sqrt(n), P = L L' / n + 0.1 I),
    each with a planted optimum: x ~ N(0, 1); y ~ N(0, 1) on the z zero rows; exactly ``case.active`` nonneg rows active with
    y in [0.5, 2] and s = 0, the others with s in [0.5, 2] and y = 0.  With z + active <= n the live rows are independent
    (checked), P is positive definite or, in an LP, z + active = n: the planted (x, y, s) is the unique optimum, strictly
    complementary, and the solution map is differentiable there.  ``shared``: every instance has instance 0's A and P (own
    b and c).  x_star / y_star / s_star hold the planted point."""
    assert case.z + case.active <= case.n and case.active <= case.m - case.z
    assert case.P or case.z + case.active == case.n, "an LP needs n live rows for a unique x"
    n, m = case.n, case.m
    rng = np.random.default_rng(seed)
    st = Structure.dense(n, m, ConeSpec(z=case.z, l=m - case.z), with_P=case.P)
    iu = np.triu_indices(n)
    A_vals, P_vals, b, c, X, Y, S = [], [], [], [], [], [], []
    A, P = _draw_AP(n, m, case.P, rng)
    for i in range(B):
        if i and not shared:
            A, P = _draw_AP(n, m, case.P, rng)
        bi, ci, x, y, s = _plant_one(A, P, case.z, case.active, rng)
        A_vals.append(A.ravel()); b.append(bi); c.append(ci); X.append(x); Y.append(y); S.append(s)
        if case.P:
            P_vals.append(P[iu])
    arr = lambda a: np.ascontiguousarray(np.stack(a))  # noqa: E731
    return Batch(st, arr(A_vals), arr(b), arr(c), arr(P_vals) if case.P else None, arr(X), arr(Y), arr(S), f"planted_{case.id}")


def replant(bt: Batch, case: Case, seed: int) -> Batch:
    """The same A and P per instance with a new planted optimum (new b, c, x*, y*, s* and active set)."""
    rng = np.random.default_rng(seed)
    out = [_plant_one(bt.A_dense(i), bt.P_dense(i) if case.P else None, case.z, case.active, rng) for i in range(bt.B)]
    b, c, X, Y, S = (np.ascontiguousarray(np.stack([o[k] for o in out])) for k in range(5))
    return Batch(bt.structure, bt.A_vals, b, c, bt.P_vals, X, Y, S, bt.name + "_replanted")
