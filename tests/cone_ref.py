"""Independent reference of every cone the engine accepts -- TEST INFRASTRUCTURE.

* Exponential cone K_exp = cl{(x, y, z): y > 0, y e^{x/y} <= z}: projection in mpmath at 120 digits and its Jacobian by
  central differences of that projection.  The iterative case solves the stationarity condition in rho = x / y by plain
  bisection on a bracket found by a float64 scan; whatever finds the root, a point is accepted only when its Moreau
  certificate (p in K, v - p in the polar cone, p'(v - p) = 0) holds to 1e-40 relative, which is what makes the reference
  independent of the device's and the C oracle's scheme (Newton starts, absolute thresholds).
* Zero, nonnegative, second-order and PSD cones: the float64 closed forms of ``problems.proj_dual_cone`` and
  ``oracle.np_ref.dproj_matrix``.
* ``exact_adjoint`` / ``exact_jvp``: diffcp's adjoint and forward-mode derivative with a dense ``M`` built from that
  Jacobian, solved by ``numpy.linalg.lstsq`` (no oracle call).
"""
from __future__ import annotations

from functools import lru_cache

import mpmath as mp
import numpy as np

from cvxpylayers_b200.problems import proj_dual_cone as _proj_dual_polyhedral_soc_psd
from cvxpylayers_b200.structure import ConeSpec
from oracle.np_ref import dproj_matrix as _dproj_polyhedral_soc_psd
from tests.jvp_ref import jvp_rhs

_DPS = 120   # 60 digits lose up to 30 to cancellation in v - p near the rays (rho ~ -66: r - y rho ~ 1e-29 r)
_CERT = mp.mpf("1e-40")
# bracket scan in rho: near the (0, 0, t) ray the root lies far out on the positive side, near the (x < 0, 0, 0) ray on the
# negative side (rho ~ x / y with y -> 0)
_GRID = np.concatenate([-np.geomspace(1e12, 60.0, 4000, endpoint=False), np.linspace(-60.0, 700.0, 76001),
                        np.geomspace(700.0, 1e15, 4000)[1:]])


def _h(r, s, t, rho):
    """Stationarity residual in rho: p = y (rho, 1, e^rho), v - p = mu (e^rho, (1 - rho) e^rho, -1)."""
    E = mp.exp(rho)
    den = rho + E * E
    y = (r + t * E) / den
    mu = (r * E - t * rho) / den
    return y + mu * E * (1 - rho) - s, y, mu


def certificate(v, p):
    """Largest violation of the Moreau conditions of p = Pi_{K_exp}(v), relative to ||v|| (||v||^2 for p'(v - p))."""
    r, s, t = v
    d = [v[i] - p[i] for i in range(3)]
    sc = max(mp.mpf(1) * 1e-300, mp.sqrt(r * r + s * s + t * t))
    if p[1] > 0:
        in_k = max(0, p[1] * mp.exp(p[0] / p[1]) - p[2])
    else:
        in_k = max(abs(p[1]), max(0, p[0]), max(0, -p[2]))
    if d[0] > 0:   # -d in K* = {(u, w, z): u < 0, -u e^{w/u} <= e z}
        in_polar = max(0, d[0] * mp.exp(d[1] / d[0]) + mp.e * d[2])
    else:
        in_polar = max(abs(d[0]), max(0, d[1]), max(0, d[2]))
    comp = abs(sum(p[i] * d[i] for i in range(3)))
    return max(in_k / sc, in_polar / sc, comp / (sc * sc))


def _bisect(r, s, t, a, b):
    """Bisection down to 1e-12 of the bracket, then the bracketing Illinois iteration (bisection again if it fails)."""
    ha = _h(r, s, t, a)[0]
    for k in range(420):
        if k == 40:
            try:
                return mp.findroot(lambda x: _h(r, s, t, x)[0], (a, b), solver="illinois", maxsteps=200)
            except (ValueError, ZeroDivisionError):
                pass
        c = (a + b) / 2
        hc = _h(r, s, t, c)[0]
        if (hc > 0) == (ha > 0):
            a, ha = c, hc
        else:
            b = c
    return (a + b) / 2


def _brackets(r, s, t):
    rho, r, s, t = _GRID, float(r), float(s), float(t)
    with np.errstate(all="ignore"):   # _h in float64, divided through by e^{2 rho} where rho > 0 so that nothing overflows
        F = np.exp(-np.abs(rho))
        pos = rho > 0
        den = np.where(pos, rho * F * F + 1.0, rho + F * F)
        y = np.where(pos, r * F * F + t * F, r + t * F) / den
        muE = np.where(pos, r - t * rho * F, r * F * F - t * rho * F) / den
        h = y + muE * (1 - rho) - s
    ok = np.isfinite(h)   # y > 0 and mu >= 0 are left to the certificate: a root can sit where the grid's mu is still < 0
    idx = np.nonzero(ok[:-1] & ok[1:] & (np.sign(h[:-1]) != np.sign(h[1:])) & (np.sign(den[:-1]) == np.sign(den[1:])))[0]
    # a root can sit between the pole of h (rho + e^{2 rho} = 0) and the grid point next to it
    pole, eps = _pole(), mp.mpf("1e-50")
    k = int(np.searchsorted(rho, float(pole)))
    return [(mp.mpf(rho[i]), mp.mpf(rho[i + 1])) for i in idx] + [(mp.mpf(rho[k - 1]), pole - eps), (pole + eps, mp.mpf(rho[k]))]


@lru_cache(maxsize=None)
def _pole():
    return mp.findroot(lambda x: x + mp.exp(2 * x), mp.mpf("-0.4263"))


def exp_case(v) -> int:
    """The case of proj_exp's case split (0 inside, 1 polar, 2 r < 0 and s < 0, 3 iterative), decided exactly."""
    with mp.workdps(_DPS):
        r, s, t = (mp.mpf(float(a)) for a in v)
        if (s > 0 and s * mp.exp(r / s) <= t) or (r <= 0 and s == 0 and t >= 0):
            return 0
        if (r > 0 and r * mp.exp(s / r) <= -mp.e * t) or (r == 0 and s <= 0 and t <= 0):
            return 1
        if r < 0 and s < 0:
            return 2
        return 3


def _proj_exp_mp(v, hint=None):
    """-> (p as three mpf, case, rho or None); v: three mpf at the working precision."""
    r, s, t = v
    case = 0 if ((s > 0 and s * mp.exp(r / s) <= t) or (r <= 0 and s == 0 and t >= 0)) else \
        1 if ((r > 0 and r * mp.exp(s / r) <= -mp.e * t) or (r == 0 and s <= 0 and t <= 0)) else \
        2 if (r < 0 and s < 0) else 3
    if case == 0:
        return [r, s, t], 0, None
    if case == 1:
        return [mp.mpf(0)] * 3, 1, None
    if case == 2:
        return [r, mp.mpf(0), max(t, mp.mpf(0))], 2, None
    tries = []
    if hint is not None:
        w = mp.mpf("1e-12") * max(1, abs(hint))
        tries.append((hint - w, hint + w))
    tries += _brackets(r, s, t)
    for a, b in tries:
        if (_h(r, s, t, a)[0] > 0) == (_h(r, s, t, b)[0] > 0):
            continue
        rho = _bisect(r, s, t, a, b)
        _, y, _ = _h(r, s, t, rho)
        p = [y * rho, y, y * mp.exp(rho)]
        if y > 0 and certificate(v, p) <= _CERT:
            return p, 3, rho
    raise ArithmeticError(f"no certified exponential-cone projection of {[float(a) for a in v]}")


def proj_exp(v) -> np.ndarray:
    """Pi_{K_exp}(v) in float64."""
    with mp.workdps(_DPS):
        return np.array([float(a) for a in _proj_exp_mp([mp.mpf(float(a)) for a in v])[0]])


def dproj_exp(v) -> np.ndarray:
    """D Pi_{K_exp}(v) (3 x 3) by central differences of the 120-digit projection, step 1e-20 ||v||."""
    with mp.workdps(_DPS):
        v0 = [mp.mpf(float(a)) for a in v]
        _, _, rho = _proj_exp_mp(v0)
        h = mp.mpf("1e-20") * max(1, mp.sqrt(sum(a * a for a in v0)))
        J = np.zeros((3, 3))
        for j in range(3):
            vp, vm = list(v0), list(v0)
            vp[j] += h
            vm[j] -= h
            pp, pm = _proj_exp_mp(vp, rho)[0], _proj_exp_mp(vm, rho)[0]
            J[:, j] = [float((pp[i] - pm[i]) / (2 * h)) for i in range(3)]
        return J


def proj_exp_dual(v) -> np.ndarray:
    """Pi_{K*}(v) = v + Pi_K(-v) (Moreau) for the dual cone K* = K_exp*."""
    v = np.asarray(v, dtype=np.float64)
    return v + proj_exp(-v)


def dproj_exp_dual(v) -> np.ndarray:
    return np.eye(3) - dproj_exp(-np.asarray(v, dtype=np.float64))


def _split(cones: ConeSpec):
    head = ConeSpec(z=cones.z, l=cones.l, q=list(cones.q), s=list(cones.s))
    return head, head.m


def proj_dual(v: np.ndarray, cones: ConeSpec) -> np.ndarray:
    """Pi_{K*}(v) over a whole cone spec (SCS row order z, l, q, s, ep, ed): ep rows project onto K_exp*, ed rows onto K_exp."""
    head, mh = _split(cones)
    out = np.empty_like(v, dtype=np.float64)
    out[:mh] = _proj_dual_polyhedral_soc_psd(v[:mh], head)
    for e in range(cones.ep + cones.ed):
        blk = v[mh + 3 * e: mh + 3 * e + 3]
        out[mh + 3 * e: mh + 3 * e + 3] = proj_exp_dual(blk) if e < cones.ep else proj_exp(blk)
    return out


def dproj_dual(v: np.ndarray, cones: ConeSpec) -> np.ndarray:
    """Dense Jacobian of :func:`proj_dual` at v."""
    head, mh = _split(cones)
    D = np.zeros((v.size, v.size))
    D[:mh, :mh] = _dproj_polyhedral_soc_psd(v[:mh], head)
    for e in range(cones.ep + cones.ed):
        o = mh + 3 * e
        D[o:o + 3, o:o + 3] = dproj_exp_dual(v[o:o + 3]) if e < cones.ep else dproj_exp(v[o:o + 3])
    return D


def dense_M(A, P, b, c, x, y, s, cones: ConeSpec):
    """-> M (N x N), D (m x m), pi_y: diffcp's derivative matrix at (x, y, s) with the reference cone Jacobian."""
    m, n = A.shape
    N = n + m + 1
    v = y - s
    D = dproj_dual(v, cones)
    piy = proj_dual(v, cones)
    Pm = np.zeros((n, n)) if P is None else P
    Px = Pm @ x
    DQ = np.zeros((N, N))
    DQ[:n, :n] = Pm
    DQ[:n, n:n + m] = A.T
    DQ[:n, -1] = c
    DQ[n:n + m, :n] = -A
    DQ[n:n + m, -1] = b
    DQ[-1, :n] = -(2 * Px + c)
    DQ[-1, n:n + m] = -b
    DQ[-1, -1] = x @ Px
    Dpi = np.eye(N)
    Dpi[n:n + m, n:n + m] = D
    return (DQ - np.eye(N)) @ Dpi + np.eye(N), D, piy


def exact_adjoint(A, P, b, c, x, y, s, dx, dy, cones: ConeSpec, MDpi=None):
    """-> dA (dense m x n), dP (dense n x n, gradient wrt a full unsymmetric P), db, dc.  MDpi: dense_M's result, if at hand."""
    n = A.shape[1]
    M, D, piy = MDpi or dense_M(A, P, b, c, x, y, s, cones)
    dz = np.concatenate([dx, D.T @ dy, [-(x @ dx + y @ dy)]])
    r = np.linalg.lstsq(M.T, dz, rcond=None)[0]
    rx, ry, rt = r[:n], r[n:-1], r[-1]
    return np.outer(ry, x) - np.outer(piy, rx), np.outer(rt * x - rx, x), piy * rt - ry, x * rt - rx


def exact_jvp(A, P, b, c, x, y, s, dA, dP, db, dc, cones: ConeSpec, MDpi=None):
    """-> dx, dy, ds for dense tangents (dP: the full symmetric tangent of P, or None).  MDpi: dense_M's result, if at hand."""
    n = A.shape[1]
    M, D, piy = MDpi or dense_M(A, P, b, c, x, y, s, cones)
    z = np.linalg.lstsq(M, jvp_rhs(A, x, piy, dA, dP, db, dc), rcond=None)[0]
    zx, zy, zt = z[:n], z[n:-1], z[-1]
    Dzy = D @ zy
    return zx - x * zt, Dzy - y * zt, Dzy - zy - s * zt
