// refine.cu -- solution refinement (bcone_refine; NumPy twin: tests/refine_ref.py), compiled as a translation unit of its own so
// that the kernels of bwd.cu compile to the code they have without it.
//
// Gauss-Newton on the homogeneous embedding's residual map at tau = 1 (Busseti, Moursi & Boyd, "Solution refinement at regular
// points of conic problems", 2019).  At w = (x, v), v = y - s, pi = Pi_{K*}(v):
//   R(x, v) = [P x + A' pi + c ;  b - A x - (pi - v) ;  -(x'P x + c'x + b'pi)],
// whose Jacobian in (x, v) is the first n + m columns of the forward mode's M = (DQ - I) blkdiag(I, D, 1) + I.  A step solves
// min ||M[:, :n+m] z + R|| by the forward mode's LSQR with the tau column masked (fixing tau removes M's null vector at a
// solution, the homogeneity direction), then backtracks alpha = 1, 1/2, ..., 1/32 to the first trial with a smaller ||R||_2.
// Every trial is a full set-up (SOC projection, PSD Jacobi, exponential projection and Jacobians).  The candidate is
// (x, pi, pi - v), so y in K*, s in K and y's = 0 hold exactly; it replaces the input only if none of polishing's
// rp, rd, gap grows.
#define BC_REFINE 1
#include "bwd.cu"
