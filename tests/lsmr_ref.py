"""NumPy restatement of the engine's LSMR (``lsmr_block`` in cvxpylayers_b200/csrc/common.cuh) -- TEST INFRASTRUCTURE.

The same recurrences, in the same order, as the device routine: u and v normalised by multiplying with the reciprocal of
their norms, v's normalisation applied in the pass that updates h-bar, x and h, ||x|| taken after that pass, SciPy's
``scipy.sparse.linalg.lsmr`` stopping rules at damp = 0.  Returns every iterate so that the CPU suite can hold it to SciPy's
own iterates, and the GPU suite can hold the kernels to SciPy directly.

``adjoint_system`` builds the adjoint's explicit least-squares problem ``r = argmin ||M' r - dz||`` the way
``oracle.np_ref.vjp_dense`` does; ``tests.jvp_ref.dense_M`` / ``jvp_rhs`` give the forward mode's ``z = argmin ||M z - g||``.
"""
from __future__ import annotations

import numpy as np

from tests.jvp_ref import dense_M


def sym_ortho(a, b):
    """SciPy's stable Givens rotation: (c, s, r) with [c s; -s c] [a; b] = [r; 0]."""
    if b == 0:
        return np.sign(a), 0.0, abs(a)
    if a == 0:
        return 0.0, np.sign(b), abs(b)
    if abs(b) > abs(a):
        tau = a / b
        s = np.sign(b) / np.sqrt(1 + tau * tau)
        return s * tau, s, b / s
    tau = b / a
    c = np.sign(a) / np.sqrt(1 + tau * tau)
    return c, c * tau, a / c


def lsmr(B, rhs, atol=1e-8, btol=1e-8, conlim=1e8, iter_lim=None):
    """-> (x, itn, iterates): LSMR on the explicit matrix ``B`` as the kernels run it; ``iterates[k]`` is x after k + 1 steps."""
    N = B.shape[1]
    iter_lim = 2 * N if iter_lim is None or iter_lim < 0 else iter_lim
    ctol = 1.0 / conlim if conlim > 0 else 0.0
    u = np.array(rhs, dtype=np.float64)
    x = np.zeros(N)
    normb = np.sqrt(u @ u)
    beta, alpha, v = normb, 0.0, np.zeros(N)
    if beta > 0:
        u = u * (1.0 / beta)
        v = B.T @ u
        alpha = np.sqrt(v @ v)
    v = v * (1.0 / alpha if alpha > 0 else 1.0)
    h, hbar = v.copy(), np.zeros(N)
    if alpha * beta == 0:
        return x, 0, []
    zetabar, alphabar, rho, rhobar, cbar, sbar = alpha * beta, alpha, 1.0, 1.0, 1.0, 0.0
    betadd, betad, rhodold, tautildeold, thetatilde, zeta, d = beta, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0
    normA2, maxrbar, minrbar = alpha * alpha, 0.0, 1e100
    itn, iterates = 0, []
    while itn < iter_lim:
        itn += 1
        u = B @ v - alpha * u
        beta = np.sqrt(u @ u)
        vs = 1.0
        if beta > 0:
            u = u * (1.0 / beta)
            v = B.T @ u - beta * v
            alpha = np.sqrt(v @ v)
            if alpha > 0:
                vs = 1.0 / alpha
        chat, shat, alphahat = sym_ortho(alphabar, 0.0)
        rhoold = rho
        c, s, rho = sym_ortho(alphahat, beta)
        thetanew = s * alpha
        alphabar = c * alpha
        rhobarold, zetaold, thetabar, rhotemp = rhobar, zeta, sbar * rho, cbar * rho
        cbar, sbar, rhobar = sym_ortho(cbar * rho, thetanew)
        zeta = cbar * zetabar
        zetabar = -sbar * zetabar
        v = v * vs
        hbar = h - (thetabar * rho / (rhoold * rhobarold)) * hbar
        x = x + (zeta / (rho * rhobar)) * hbar
        h = v - (thetanew / rho) * h
        iterates.append(x.copy())
        normx = np.sqrt(x @ x)
        betaacute, betacheck = chat * betadd, -shat * betadd
        betahat = c * betaacute
        betadd = -s * betaacute
        thetatildeold = thetatilde
        ctildeold, stildeold, rhotildeold = sym_ortho(rhodold, thetabar)
        thetatilde = stildeold * rhobar
        rhodold = ctildeold * rhobar
        betad = -stildeold * betad + ctildeold * betahat
        tautildeold = (zetaold - thetatildeold * tautildeold) / rhotildeold
        taud = (zeta - thetatilde * tautildeold) / rhodold
        d += betacheck * betacheck
        normr = np.sqrt(d + (betad - taud) ** 2 + betadd * betadd)
        normA2 += beta * beta
        normA = np.sqrt(normA2)
        normA2 += alpha * alpha
        maxrbar = max(maxrbar, rhobarold)
        if itn > 1:
            minrbar = min(minrbar, rhobarold)
        condA = max(maxrbar, rhotemp) / min(minrbar, rhotemp)
        normar = abs(zetabar)
        test1 = normr / normb
        test2 = normar / (normA * normr) if normA * normr != 0 else np.inf
        test3 = 1.0 / condA
        t1 = test1 / (1 + normA * normx / normb)
        rtol = btol + atol * normA * normx / normb
        istop = 0
        if itn >= iter_lim:
            istop = 7
        if 1 + test3 <= 1:
            istop = 6
        if 1 + test2 <= 1:
            istop = 5
        if 1 + t1 <= 1:
            istop = 4
        if test3 <= ctol:
            istop = 3
        if test2 <= atol:
            istop = 2
        if test1 <= rtol:
            istop = 1
        if istop:
            break
    return x, itn, iterates


def adjoint_system(st, A, P, b, c, x, y, s, dx, dy):
    """-> (M, dz, D, pi_y): the adjoint solves r = argmin ||M' r - dz|| (diffcp's B3; np_ref.vjp_dense)."""
    M, D, piy = dense_M(st, A, P, b, c, x, y, s)
    dz = np.concatenate([dx, D.T @ dy, [-(x @ dx + y @ dy)]])
    return M, dz, D, piy


def adjoint_grads(r, x, piy, n):
    """-> dA (dense), db, dc of the adjoint from its least-squares solution r (np_ref.vjp_dense's assembly)."""
    rx, ry, rt = r[:n], r[n:-1], r[-1]
    return np.outer(ry, x) - np.outer(piy, rx), piy * rt - ry, x * rt - rx
