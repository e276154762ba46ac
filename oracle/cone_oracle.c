/*
 * cone_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 * See cone_oracle.h for scope, provenance and the parity-pin statement.
 *
 * What is restated (published algorithms; no upstream source was available):
 *  - forward : operator splitting on the homogeneous self-dual embedding with
 *    a quadratic objective (O'Donoghue, "Operator splitting for a homogeneous
 *    embedding of the linear complementarity problem", SIAM J. Optim. 2021) --
 *    the algorithm of SCS 3.x that diffcp calls for the reference at
 *    src/cvxpylayers/interfaces/diffcp_if.py:365 (F3-F6 in SURVEY.md 8a):
 *    Ruiz equilibration, reduced normalised KKT solve (dense Cholesky here),
 *    projection on R^n x K* x R_+, over-relaxation alpha, SCS termination
 *    criteria on the un-normalised data, adaptive scale heuristic.
 *  - backward: Agrawal et al., "Differentiating through a cone program" (2019),
 *    i.e. diffcp's adjoint_derivative (called at diffcp_if.py:86): dz from
 *    (dx,dy,ds=0), r = LSQR(M^T, dz) with M = (DQ - I) DPi(z) + I, gradient
 *    assembly on the sparsity pattern (B1-B4 in SURVEY.md 8a), extended with
 *    the quadratic-objective terms of the embedding so a native P is handled.
 *  - LSQR: Paige & Saunders, ACM TOMS 8(1) 1982, with the stopping rules of
 *    the SciPy implementation that diffcp's lsqr.cpp ports (atol, btol, conlim).
 */
#include "cone_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <malloc.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TAU_FACTOR 10.0
#define ZERO_CONE_FACTOR 1000.0
#define MIN_SCALE 1e-4
#define MAX_SCALE 1e4
#define RESCALE_MIN_ITERS 100
#define EQ_MIN 1e-4
#define EQ_MAX 1e4

void orc_default_settings(orc_settings *st) {
  st->eps_abs = 1e-4; st->eps_rel = 1e-4; st->eps_infeas = 1e-7;
  st->alpha = 1.5; st->rho_x = 1e-6; st->scale = 0.1;
  st->lsqr_atol = 1e-8; st->lsqr_btol = 1e-8; st->lsqr_conlim = 1e8;
  st->max_iters = 100000; st->normalize = 1; st->adaptive_scale = 1; st->check_interval = 25;
  st->ruiz_passes = 10; st->lsqr_iter_lim = -1; st->lsqr_precond = 0; st->adaptive_check = 0;
  st->acceleration_lookback = 10; st->acceleration_interval = 10;
}

int orc_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* ------------------------------------------------------------------ cones */
enum { CZERO = 0, CNONNEG = 1, CSOC = 2, CPSD = 3, CEXP = 4, CEXPD = 5 };
typedef struct { int type, start, size, order; } cblock;

static int cone_blocks(const orc_desc *d, cblock **out) {
  int nb = (d->z > 0) + (d->l > 0) + d->nq + d->ns + d->ep + d->ed;
  cblock *B = (cblock *)malloc(sizeof(cblock) * (nb > 0 ? nb : 1));
  int k = 0, off = 0;
  if (d->z > 0) { B[k++] = (cblock){CZERO, off, d->z, 0}; off += d->z; }
  if (d->l > 0) { B[k++] = (cblock){CNONNEG, off, d->l, 0}; off += d->l; }
  for (int i = 0; i < d->nq; i++) { B[k++] = (cblock){CSOC, off, d->q[i], 0}; off += d->q[i]; }
  for (int i = 0; i < d->ns; i++) {
    int o = d->s[i], sz = o * (o + 1) / 2;
    B[k++] = (cblock){CPSD, off, sz, o}; off += sz;
  }
  for (int i = 0; i < d->ep; i++) { B[k++] = (cblock){CEXP, off, 3, 0}; off += 3; }
  for (int i = 0; i < d->ed; i++) { B[k++] = (cblock){CEXPD, off, 3, 0}; off += 3; }
  *out = B;
  return k;
}

/* cyclic Jacobi eigen-decomposition of a symmetric k x k matrix (row-major).
 * On exit X holds eigenvalues on its diagonal, V the eigenvectors as columns. */
static void jacobi_eig(int k, double *X, double *V) {
  for (int i = 0; i < k; i++) for (int j = 0; j < k; j++) V[i * k + j] = (i == j);
  for (int sweep = 0; sweep < 30; sweep++) {
    int rotations = 0;
    for (int p = 0; p < k - 1; p++) for (int q = p + 1; q < k; q++) {
      double apq = X[p * k + q];
      if (fabs(apq) <= 1e-17 * (fabs(X[p * k + p]) + fabs(X[q * k + q])) || apq == 0.0) continue;
      rotations++;
      double app = X[p * k + p], aqq = X[q * k + q];
      double theta = (aqq - app) / (2.0 * apq);
      double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int r = 0; r < k; r++) { /* columns p,q */
        double xp = X[r * k + p], xq = X[r * k + q];
        X[r * k + p] = c * xp - s * xq; X[r * k + q] = s * xp + c * xq;
      }
      for (int r = 0; r < k; r++) { /* rows p,q */
        double xp = X[p * k + r], xq = X[q * k + r];
        X[p * k + r] = c * xp - s * xq; X[q * k + r] = s * xp + c * xq;
      }
      for (int r = 0; r < k; r++) {
        double vp = V[r * k + p], vq = V[r * k + q];
        V[r * k + p] = c * vp - s * vq; V[r * k + q] = s * vp + c * vq;
      }
    }
    if (rotations == 0) break;
  }
}

/* svec (lower-triangle column-major, off-diagonals * sqrt2) <-> symmetric matrix;
 * layout stated at reference src/cvxpylayers/torch/cvxpylayer.py:201-222. */
static void svec_to_mat(int k, const double *v, double *X) {
  int idx = 0; const double is2 = 0.70710678118654752440;
  for (int j = 0; j < k; j++) for (int i = j; i < k; i++) {
    double val = v[idx++];
    if (i == j) X[i * k + i] = val; else { X[i * k + j] = val * is2; X[j * k + i] = val * is2; }
  }
}
static void mat_to_svec(int k, const double *X, double *v) {
  int idx = 0; const double s2 = 1.41421356237309504880;
  for (int j = 0; j < k; j++) for (int i = j; i < k; i++)
    v[idx++] = (i == j) ? X[i * k + i] : 0.5 * (X[i * k + j] + X[j * k + i]) * s2;
}

static void proj_soc(int sz, double *v) {
  if (sz == 0) return;
  if (sz == 1) { if (v[0] < 0) v[0] = 0; return; }
  double t = v[0], nx = 0;
  for (int i = 1; i < sz; i++) nx += v[i] * v[i];
  nx = sqrt(nx);
  if (nx <= t) return;
  if (nx <= -t) { for (int i = 0; i < sz; i++) v[i] = 0; return; }
  double a = 0.5 * (1.0 + t / nx);
  v[0] = a * nx;
  for (int i = 1; i < sz; i++) v[i] *= a;
}

static void proj_psd(int k, double *v) {
  double *X = (double *)malloc(sizeof(double) * 2 * k * k), *V = X + k * k;
  svec_to_mat(k, v, X);
  jacobi_eig(k, X, V);
  double *lam = (double *)malloc(sizeof(double) * k);
  for (int i = 0; i < k; i++) lam[i] = X[i * k + i] > 0 ? X[i * k + i] : 0;
  for (int i = 0; i < k; i++) for (int j = 0; j < k; j++) {
    double acc = 0;
    for (int e = 0; e < k; e++) acc += V[i * k + e] * lam[e] * V[j * k + e];
    X[i * k + j] = acc;
  }
  mat_to_svec(k, X, v);
  free(lam); free(X);
}


/* ---- exponential cone K_exp = cl{(x,y,z): y > 0, y e^{x/y} <= z} ------------------------------
 * Projection: the three closed-form cases, otherwise bisection on the dual variable with an inner
 * 1-D Newton (Parikh & Boyd, "Proximal Algorithms" 6.3.4 -- the scheme of SCS's exp_cone.c), then a
 * Newton polish of the univariate optimality condition in rho = x/y (Friberg 2023) to full precision.
 * Jacobian: implicit differentiation of the projection's KKT system (the 4x4 solve of SURVEY.md 8a B1). */
static double exp_newton_one_d(double rho, double yh, double zh) {
  double t = fmax(-zh, 1e-6);
  for (int i = 0; i < 100; i++) {
    double f = t * (t + zh) / rho / rho - yh / rho + log(t / rho) + 1.0;
    double fp = (2.0 * t + zh) / rho / rho + 1.0 / t;
    t -= f / fp;
    if (t <= -zh) return 0.0;
    if (t <= 0.0) return zh;
    if (fabs(f) < 1e-13) break;
  }
  return t + zh;
}
static double exp_calc_grad(const double *v, double *x, double rho) {
  x[2] = exp_newton_one_d(rho, v[1], v[2]);
  x[1] = (x[2] - v[2]) * x[2] / rho;
  x[0] = v[0] - rho;
  if (x[1] <= 1e-12) return x[0];
  return x[0] + x[1] * log(x[1] / x[2]);
}
static double exp_h(double r, double s, double t, double rho, double *y, double *mu) {
  double E = exp(rho), id = 1.0 / (rho + E * E);
  *y = (r + t * E) * id;
  *mu = (r * E - t * rho) * id;   /* = y e^rho - t without its cancellation once y e^rho ~ t */
  return *y + *mu * E * (1.0 - rho) - s;
}
/* Newton on h(rho) = 0 (rho = x / y of the projection p = (rho y, y, y e^rho); h is the stationarity residual of the */
/* y-coordinate, exp_h above) with the analytic derivative, started from *rho0 (the previous iterate's root; the */
/* cone moves little between operator-splitting iterations) or from a crude guess.  Accepts only a root with y > 0, */
/* mu >= 0 and |h| at rounding level; anything else (no decrease, leaving the domain) returns false and the caller falls */
/* back to the bisection.  Typically 2-4 iterations warm, 5-8 cold. */
static int exp_newton_rho(double r, double s, double t, double *rho0, double *x) {
  double rho = (rho0 && *rho0 == *rho0) ? *rho0 : (s > 0 ? fmin(fmax(r / s, -20.0), 20.0) : (t > 0 && r > 0 ? fmin(log(fmax(t, 1e-300) / fmax(r, 1e-300)) , 20.0) : 0.0));
  const double scale = fmax(1.0, fmax(fabs(r), fmax(fabs(s), fabs(t))));
  double y, mu, hv = exp_h(r, s, t, rho, &y, &mu);
  for (int it = 0; it < 30; it++) {
    if (!(hv == hv)) return 0;
    if (fabs(hv) <= 1e-15 * scale) break;
    const double E = exp(rho), den = rho + E * E;
    const double yp = (t * E * den - (r + t * E) * (1.0 + 2.0 * E * E)) / (den * den);
    const double mup = (yp + y) * E;
    const double hp = yp + mup * E * (1.0 - rho) - mu * E * rho;
    if (hp == 0.0 || !(hp == hp)) return 0;
    double step = -hv / hp, rn, yn, mn, hn;
    int bt = 0;
    int stalled = 0;
    for (;; bt++) {   /* damping: accept the first step that reduces |h| inside the domain */
      rn = rho + step;
      hn = exp_h(r, s, t, rn, &yn, &mn);
      if (hn == hn && fabs(hn) < fabs(hv)) break;   /* (rho + e^{2 rho} may have either sign: roots exist on both sides of its zero) */
      if (bt == 12) { stalled = 1; break; }
      step *= 0.5;
    }
    if (stalled) {   /* no decrease left: at rounding level that is convergence, anywhere else a failure */
      if (fabs(hv) <= 1e-11 * scale) break;
      return 0;
    }
    const int tiny = fabs(step) <= 1e-15 * fmax(1.0, fabs(rn));
    rho = rn; hv = hn; y = yn; mu = mn;
    if (tiny) break;
  }
  if (!(fabs(hv) <= 1e-11 * scale) || !(y > 0)) return 0;
  /* Certificate (the projection is the unique point with p in K, v - p in the polar cone, p'(v - p) = 0): h = 0 alone can */
  /* be met by a spurious root where mu = y e^rho - t is pure cancellation, so the dual part is checked on d = v - p itself. */
  const double E = exp(rho);
  const double px = y * rho, py = y, pz = y * E;
  const double dx = r - px, dy = s - py, dz = t - pz;           /* must be mu (E, (1 - rho) E, -1), mu >= 0 */
  /* the normal divided by max(1, e^rho): mu2 = -dz would carry the rounding of t - y e^rho, times e^rho, into dx */
  const double na = E >= 1.0 ? 1.0 : E, n0 = na, n1 = na * (1.0 - rho), n2 = E >= 1.0 ? -1.0 / E : -1.0;
  const double nn = sqrt(n0 * n0 + n1 * n1 + n2 * n2), mu2 = (dx * n0 + dy * n1 + dz * n2) / nn;
  if (!(mu2 >= -1e-13 * scale)) return 0;
  if (fabs(dx - mu2 * n0 / nn) > 1e-9 * scale || fabs(dy - mu2 * n1 / nn) > 1e-9 * scale || fabs(dz - mu2 * n2 / nn) > 1e-9 * scale) return 0;
  if (fabs(px * dx + py * dy + pz * dz) > 1e-9 * scale * scale) return 0;
  x[0] = px; x[1] = py; x[2] = pz;
  if (rho0) *rho0 = rho;
  return 1;
}
static int exp_newton_multi(double r, double s, double t, double *x) {
  if (exp_newton_rho(r, s, t, NULL, x)) return 1;
  const double starts[6] = {0.0, -1.0, 1.0, -3.0, 3.0, 8.0};
  for (int k = 0; k < 6; k++) { double g = starts[k]; if (exp_newton_rho(r, s, t, &g, x)) return 1; }
  return 0;
}
/* returns the case: 0 in K, 1 in polar (-> 0), 2 analytic face, 3 iterative.  The iterative case first tries the Newton
 * iteration above (certified by the Moreau conditions, more accurate than the bisection near the y = 0 face) and only
 * then the bisection of Parikh & Boyd. */
static int proj_exp_unit(double *v) {
  const double r = v[0], s = v[1], t = v[2];
  if ((s > 0 && s * exp(fmin(r / s, 700.0)) - t <= 1e-13) || (r <= 0 && s == 0 && t >= 0)) return 0;
  if ((r > 0 && r * exp(fmin(s / r, 700.0)) + 2.718281828459045 * t <= 1e-13) || (r == 0 && s <= 0 && t <= 0)) { v[0] = v[1] = v[2] = 0; return 1; }
  if (r < 0 && s < 0) { v[1] = 0.0; v[2] = fmax(t, 0.0); return 2; }
  double x[3];
  if (exp_newton_multi(r, s, t, x)) { v[0] = x[0]; v[1] = x[1]; v[2] = x[2]; return 3; }
  double lb = 0.0, ub = 0.125;
  while (exp_calc_grad(v, x, ub) > 0 && ub < 1e300) { lb = ub; ub *= 2.0; }
  for (int i = 0; i < 200; i++) {
    double rho = 0.5 * (ub + lb), g = exp_calc_grad(v, x, rho);
    if (g > 0) lb = rho; else ub = rho;
    if (ub - lb < 1e-10 * fmax(1.0, rho)) break;
  }
  if (x[1] > 1e-12) { /* polish */
    double rr = x[0] / x[1], y, mu, hv = exp_h(r, s, t, rr, &y, &mu);
    for (int it = 0; it < 8; it++) {
      double d = 1e-7 * fmax(1.0, fabs(rr)), y2, m2;
      double dh = (exp_h(r, s, t, rr + d, &y2, &m2) - exp_h(r, s, t, rr - d, &y2, &m2)) / (2.0 * d);
      if (dh == 0.0) break;
      double rn = rr - hv / dh, yn, mn, hn = exp_h(r, s, t, rn, &yn, &mn);
      if (!(fabs(hn) < fabs(hv) && yn > 0 && mn >= 0)) break;
      rr = rn; hv = hn; y = yn; mu = mn;
    }
    if (y > 0 && mu >= 0) { x[0] = y * rr; x[1] = y; x[2] = y * exp(rr); }
  }
  v[0] = x[0]; v[1] = x[1]; v[2] = x[2];
  return 3;
}
/* The projection is positively homogeneous and its Jacobian homogeneous of degree 0: both work on v / 2^k with max|v_i| in
 * [1, 2), so that the absolute thresholds of proj_exp_unit (the 1e-13 case tests, the 1e-12 face test, the Newton and
 * bisection tolerances) are relative to |v|; a power of two keeps the scaling exact. */
static int exp_unit_scale(const double *v, double *u) {
  const double m = fmax(fabs(v[0]), fmax(fabs(v[1]), fabs(v[2])));
  const int k = m > 0.0 ? ilogb(m) : 0;
  for (int i = 0; i < 3; i++) u[i] = scalbn(v[i], -k);
  return k;
}
static int proj_exp(double *v) {
  double u[3];
  const int k = exp_unit_scale(v, u), cs = proj_exp_unit(u);
  for (int i = 0; i < 3; i++) v[i] = scalbn(u[i], k);
  return cs;
}
/* J (3x3 row-major) = D Pi_{K_exp}(v) */
static void dproj_exp_mat(const double *v0, double *J) {
  double v[3];
  exp_unit_scale(v0, v);
  double p[3] = {v[0], v[1], v[2]};
  int cs = proj_exp_unit(p);
  for (int i = 0; i < 9; i++) J[i] = 0;
  if (cs == 0) { J[0] = J[4] = J[8] = 1.0; return; }
  if (cs == 1) return;
  if (cs == 2) { J[0] = 1.0; J[8] = v[2] > 0 ? 1.0 : 0.0; return; }
  if (!(p[1] > 1e-12)) { J[0] = v[0] < 0 ? 1.0 : 0.0; J[8] = p[2] > 0 ? 1.0 : 0.0; return; } /* landed on the y = 0 face */
  const double rho = p[0] / p[1], E = exp(rho), mu = p[2] - v[2], a = mu * E / p[1];
  double K[4][7] = {{1.0 + a, -a * rho, 0.0, E, 1, 0, 0},
                    {-a * rho, 1.0 + a * rho * rho, 0.0, E * (1.0 - rho), 0, 1, 0},
                    {0.0, 0.0, 1.0, -1.0, 0, 0, 1},
                    {E, E * (1.0 - rho), -1.0, 0.0, 0, 0, 0}};
  for (int c = 0; c < 4; c++) { /* Gauss-Jordan with partial pivoting */
    int pv = c;
    for (int r2 = c + 1; r2 < 4; r2++) if (fabs(K[r2][c]) > fabs(K[pv][c])) pv = r2;
    if (pv != c) for (int k = 0; k < 7; k++) { double tmp = K[c][k]; K[c][k] = K[pv][k]; K[pv][k] = tmp; }
    double ip = 1.0 / K[c][c];
    for (int k = 0; k < 7; k++) K[c][k] *= ip;
    for (int r2 = 0; r2 < 4; r2++) if (r2 != c) { double f = K[r2][c]; if (f != 0) for (int k = 0; k < 7; k++) K[r2][k] -= f * K[c][k]; }
  }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) J[i * 3 + j] = K[i][4 + j];
}
/* dual-cone versions used on the y block: DUALK = 1 for rows whose primal cone K is the exp cone
 * (project onto K* by Moreau), 0 for rows whose primal cone is the dual exp cone (K* = K_exp). */
static void proj_exp_dualblock(double *v, int primal_is_exp) {
  if (primal_is_exp) { double w[3] = {-v[0], -v[1], -v[2]}; proj_exp(w); for (int i = 0; i < 3; i++) v[i] += w[i]; }
  else proj_exp(v);
}
static void dproj_exp_dualblock_mat(const double *v, int primal_is_exp, double *J) {
  if (primal_is_exp) { double w[3] = {-v[0], -v[1], -v[2]}; dproj_exp_mat(w, J); for (int i = 0; i < 9; i++) J[i] = ((i % 4 == 0) ? 1.0 : 0.0) - J[i]; }
  else dproj_exp_mat(v, J);
}

static void proj_dual_blocks(const cblock *B, int nb, double *v) {
  for (int k = 0; k < nb; k++) {
    double *vb = v + B[k].start;
    switch (B[k].type) {
      case CZERO: break; /* dual of the zero cone is free */
      case CNONNEG: for (int i = 0; i < B[k].size; i++) if (vb[i] < 0) vb[i] = 0; break;
      case CSOC: proj_soc(B[k].size, vb); break;
      case CPSD: proj_psd(B[k].order, vb); break;
      case CEXP: proj_exp_dualblock(vb, 1); break;
      case CEXPD: proj_exp_dualblock(vb, 0); break;
      default: break;
    }
  }
}
void orc_proj_dual_cone(const orc_desc *d, double *v) {
  cblock *B; int nb = cone_blocks(d, &B);
  proj_dual_blocks(B, nb, v);
  free(B);
}

/* out = DPi_{K*}(v)[dv]  (SURVEY.md 8a row B1) */
static void dproj_dual_blocks(const cblock *B, int nb, const double *v, const double *dv, double *out) {
  for (int k = 0; k < nb; k++) {
    const double *vb = v + B[k].start, *db = dv + B[k].start; double *ob = out + B[k].start;
    int sz = B[k].size;
    switch (B[k].type) {
      case CZERO: for (int i = 0; i < sz; i++) ob[i] = db[i]; break;
      case CNONNEG: for (int i = 0; i < sz; i++) ob[i] = vb[i] > 0 ? db[i] : 0.0; break;
      case CSOC: {
        if (sz == 1) { ob[0] = vb[0] > 0 ? db[0] : 0.0; break; }
        double t = vb[0], nx = 0;
        for (int i = 1; i < sz; i++) nx += vb[i] * vb[i];
        nx = sqrt(nx);
        if (nx <= t) { for (int i = 0; i < sz; i++) ob[i] = db[i]; break; }
        if (nx <= -t) { for (int i = 0; i < sz; i++) ob[i] = 0; break; }
        double xdx = 0;
        for (int i = 1; i < sz; i++) xdx += vb[i] * db[i];
        /* (1/(2nx)) [[nx, x'],[x, (t+nx) I - t xx'/nx^2]] */
        ob[0] = 0.5 * (db[0] + xdx / nx);
        for (int i = 1; i < sz; i++)
          ob[i] = (vb[i] * db[0] + (t + nx) * db[i] - t * vb[i] * xdx / (nx * nx)) / (2.0 * nx);
        break;
      }
      case CPSD: {
        int o = B[k].order;
        double *X = (double *)malloc(sizeof(double) * 4 * o * o);
        double *V = X + o * o, *Dm = V + o * o, *T = Dm + o * o;
        svec_to_mat(o, vb, X); jacobi_eig(o, X, V); svec_to_mat(o, db, Dm);
        /* T = V' Dm V */
        for (int i = 0; i < o; i++) for (int j = 0; j < o; j++) {
          double acc = 0;
          for (int a = 0; a < o; a++) { double va = V[a * o + i]; if (va == 0) continue;
            double in = 0; for (int b2 = 0; b2 < o; b2++) in += Dm[a * o + b2] * V[b2 * o + j];
            acc += va * in; }
          T[i * o + j] = acc;
        }
        for (int i = 0; i < o; i++) for (int j = 0; j < o; j++) {
          double li = X[i * o + i], lj = X[j * o + j], bij;
          if (li > 0 && lj > 0) bij = 1.0; else if (li <= 0 && lj <= 0) bij = 0.0;
          else { double lp = li > 0 ? li : lj, ln = li > 0 ? lj : li; bij = lp / (lp - ln); }
          T[i * o + j] *= bij;
        }
        /* Dm = V T V' */
        for (int i = 0; i < o; i++) for (int j = 0; j < o; j++) {
          double acc = 0;
          for (int a = 0; a < o; a++) { double in = 0;
            for (int b2 = 0; b2 < o; b2++) in += T[a * o + b2] * V[j * o + b2];
            acc += V[i * o + a] * in; }
          Dm[i * o + j] = acc;
        }
        mat_to_svec(o, Dm, ob);
        free(X);
        break;
      }
      case CEXP: case CEXPD: {
        double J[9]; dproj_exp_dualblock_mat(vb, B[k].type == CEXP, J);
        for (int i = 0; i < 3; i++) ob[i] = J[i * 3] * db[0] + J[i * 3 + 1] * db[1] + J[i * 3 + 2] * db[2];
        break;
      }
      default: for (int i = 0; i < sz; i++) ob[i] = 0; break;
    }
  }
}
void orc_dproj_dual_cone(const orc_desc *d, const double *v, const double *dv, double *out) {
  cblock *B; int nb = cone_blocks(d, &B);
  dproj_dual_blocks(B, nb, v, dv, out);
  free(B);
}

/* ------------------------------------------------------------- sparse ops */
static void csr_mv(int m, const int32_t *ip, const int32_t *ix, const double *v, const double *x, double *y) {
  for (int i = 0; i < m; i++) { double a = 0; for (int k = ip[i]; k < ip[i + 1]; k++) a += v[k] * x[ix[k]]; y[i] = a; }
}
static void csr_mtv(int m, int n, const int32_t *ip, const int32_t *ix, const double *v, const double *x, double *y) {
  for (int j = 0; j < n; j++) y[j] = 0;
  for (int i = 0; i < m; i++) { double xi = x[i]; if (xi == 0) continue;
    for (int k = ip[i]; k < ip[i + 1]; k++) y[ix[k]] += v[k] * xi; }
}
static void symu_mv(int n, const int32_t *ip, const int32_t *ix, const double *v, const double *x, double *y) {
  for (int j = 0; j < n; j++) y[j] = 0;
  if (!ip) return;
  for (int i = 0; i < n; i++) for (int k = ip[i]; k < ip[i + 1]; k++) {
    int j = ix[k]; y[i] += v[k] * x[j]; if (j != i) y[j] += v[k] * x[i];
  }
}
static double dot(int n, const double *a, const double *b) { double s = 0; for (int i = 0; i < n; i++) s += a[i] * b[i]; return s; }
static double nrm2(int n, const double *a) { return sqrt(dot(n, a, a)); }

/* ------------------------------------------------------ Anderson acceleration
 * Restatement of the safeguarded Anderson acceleration SCS 3 applies to its iterate v (our w) -- SCS default
 * acceleration_lookback = 10 (type-I; a negative lookback selects type-II), acceleration_interval = 10; the
 * reference's tests switch it off explicitly with {"acceleration_lookback": 0} (tests/test_torch.py:401-405), so it
 * is ON on the reference's default path.  Algorithm: Zhang, O'Donoghue, Boyd, "Globally convergent type-I Anderson
 * acceleration for non-smooth fixed-point iterations" (2020) in the simplified form of SCS's aa.c [recalled, not
 * vendored: UPSTREAM, unverified constants]: every `interval` iterations the pair (x = iterate before the last step,
 * f = iterate after it) is pushed into a window of `mem` difference columns
 *     s = x - x_prev,  d = f - f_prev,  y = (x - f) - (x_prev - f_prev),
 * and once the window is full (SCS fills the memory before the first solve) the iterate is replaced by
 *     f - D gamma,   (S'Y + r I) gamma = S'g   [type-I]   or   (Y'Y + r I) gamma = Y'g   [type-II],
 * r = reg * (||Y||_F^2 + ||S||_F^2), reg = 1e-6 (type-I) / 1e-10 (type-II).  A step with ||gamma|| >= 1e10 (or a
 * singular system) is dropped and the window reset.  Safeguard: after the next plain step from the accelerated
 * point, if its fixed-point residual exceeds the residual of the pair that produced it (factor 1.0), the
 * accelerated point is rejected, the un-accelerated f restored and the window reset. */
typedef struct {
  int type1, mem, dim, iter, success;
  double reg, norm_g;
  double *x, *f, *g_prev, *g, *Y, *S, *D, *M, *work;
} aa_work;
#define AA_SAFEGUARD_FACTOR 1.0
#define AA_MAX_WEIGHT_NORM 1e10
static aa_work *aa_init(int dim, int lookback) {
  if (lookback == 0) return NULL;
  aa_work *a = (aa_work *)calloc(1, sizeof(aa_work));
  a->type1 = lookback > 0; a->mem = abs(lookback); a->dim = dim; a->iter = 0; a->success = 0;
  a->reg = a->type1 ? 1e-6 : 1e-10;
  size_t l = (size_t)dim, M = (size_t)a->mem;
  a->x = (double *)calloc(4 * l + 3 * l * M + M * M + M, sizeof(double));
  a->f = a->x + l; a->g_prev = a->f + l; a->g = a->g_prev + l; a->Y = a->g + l; a->S = a->Y + l * M; a->D = a->S + l * M;
  a->M = a->D + l * M; a->work = a->M + M * M;
  return a;
}
static void aa_free(aa_work *a) { if (a) { free(a->x); free(a); } }
static void aa_reset(aa_work *a) { if (a) { a->iter = 0; a->success = 0; } }
/* dense solve by Gaussian elimination with partial pivoting (len <= mem); returns 0 if singular */
static int aa_gesv(int len, double *Mx, double *rhs) {
  for (int c = 0; c < len; c++) {
    int pv = c; double best = fabs(Mx[c * len + c]);
    for (int r = c + 1; r < len; r++) if (fabs(Mx[r * len + c]) > best) { best = fabs(Mx[r * len + c]); pv = r; }
    if (!(best > 0)) return 0;
    if (pv != c) { for (int k = 0; k < len; k++) { double t = Mx[c * len + k]; Mx[c * len + k] = Mx[pv * len + k]; Mx[pv * len + k] = t; }
                   double t = rhs[c]; rhs[c] = rhs[pv]; rhs[pv] = t; }
    for (int r = c + 1; r < len; r++) {
      double f = Mx[r * len + c] / Mx[c * len + c];
      if (f == 0) continue;
      for (int k = c; k < len; k++) Mx[r * len + k] -= f * Mx[c * len + k];
      rhs[r] -= f * rhs[c];
    }
  }
  for (int r = len - 1; r >= 0; r--) {
    double acc = rhs[r];
    for (int k = r + 1; k < len; k++) acc -= Mx[r * len + k] * rhs[k];
    rhs[r] = acc / Mx[r * len + r];
  }
  return 1;
}
/* f (the newest iterate) is overwritten with the accelerated point when a step is taken; x is the iterate the last
 * step started from.  Returns ||gamma|| (0: nothing done, < 0: step rejected). */
static double aa_apply(aa_work *a, double *f, const double *x) {
  if (!a) return 0.0;
  const int l = a->dim;
  if (a->iter == 0) {
    for (int i = 0; i < l; i++) { a->x[i] = x[i]; a->f[i] = f[i]; a->g_prev[i] = x[i] - f[i]; }
    a->iter++;
    return 0.0;
  }
  const int len = a->iter < a->mem ? a->iter : a->mem, idx = (a->iter - 1) % a->mem;
  double *Yc = a->Y + (size_t)idx * l, *Sc = a->S + (size_t)idx * l, *Dc = a->D + (size_t)idx * l;
  for (int i = 0; i < l; i++) {
    const double g = x[i] - f[i];
    Sc[i] = x[i] - a->x[i]; Dc[i] = f[i] - a->f[i]; Yc[i] = g - a->g_prev[i];
    a->g[i] = g; a->g_prev[i] = g; a->x[i] = x[i]; a->f[i] = f[i];
  }
  a->norm_g = nrm2(l, a->g);
  double aa_norm = 0.0;
  if (a->iter >= a->mem) {   /* the memory is filled before the first solve */
    double ny = 0, ns = 0;
    for (int c = 0; c < len; c++) { ny += dot(l, a->Y + (size_t)c * l, a->Y + (size_t)c * l); ns += dot(l, a->S + (size_t)c * l, a->S + (size_t)c * l); }
    const double r = a->reg * (ny + ns);
    const double *Lm = a->type1 ? a->S : a->Y;
    for (int i = 0; i < len; i++) {
      for (int j = 0; j < len; j++) a->M[i * len + j] = dot(l, Lm + (size_t)i * l, a->Y + (size_t)j * l) + (i == j ? r : 0.0);
      a->work[i] = dot(l, Lm + (size_t)i * l, a->g);
    }
    const int ok = aa_gesv(len, a->M, a->work);
    aa_norm = ok ? nrm2(len, a->work) : INFINITY;
    if (!ok || !(aa_norm < AA_MAX_WEIGHT_NORM)) { aa_reset(a); return -1.0; }
    for (int c = 0; c < len; c++) { const double gc = a->work[c]; const double *Dk = a->D + (size_t)c * l; for (int i = 0; i < l; i++) f[i] -= gc * Dk[i]; }
    a->success = 1;
  }
  a->iter++;
  return aa_norm;
}
/* x_new: the accelerated point, f_new: one plain step from it.  Returns 1 if the step was rejected (both restored). */
static int aa_safeguard(aa_work *a, double *f_new, double *x_new) {
  if (!a || !a->success) return 0;
  a->success = 0;
  double nd = 0;
  for (int i = 0; i < a->dim; i++) { const double q = x_new[i] - f_new[i]; nd += q * q; }
  if (sqrt(nd) > AA_SAFEGUARD_FACTOR * a->norm_g) {
    memcpy(f_new, a->f, sizeof(double) * a->dim); memcpy(x_new, a->x, sizeof(double) * a->dim);
    aa_reset(a);
    return 1;
  }
  return 0;
}

/* ----------------------------------------------------------- forward solve */
typedef struct {
  int n, m;
  const orc_desc *d;
  double *Ah, *Ph, *D, *E, *bh, *ch, *ry, *K, *g, *tn, *tm;
  double rho_x, gRg;
} fwd_ws;

static int chol_lower(int n, double *K) {
  for (int j = 0; j < n; j++) {
    double dj = K[j * n + j];
    for (int k = 0; k < j; k++) dj -= K[j * n + k] * K[j * n + k];
    if (!(dj > 0)) return -1;
    dj = sqrt(dj); K[j * n + j] = dj;
    for (int i = j + 1; i < n; i++) {
      double a = K[i * n + j];
      for (int k = 0; k < j; k++) a -= K[i * n + k] * K[j * n + k];
      K[i * n + j] = a / dj;
    }
  }
  return 0;
}
static void chol_solve(int n, const double *L, double *x) {
  for (int i = 0; i < n; i++) { double a = x[i]; for (int k = 0; k < i; k++) a -= L[i * n + k] * x[k]; x[i] = a / L[i * n + i]; }
  for (int i = n - 1; i >= 0; i--) { double a = x[i]; for (int k = i + 1; k < n; k++) a -= L[k * n + i] * x[k]; x[i] = a / L[i * n + i]; }
}

static int factor(fwd_ws *w) {
  const orc_desc *d = w->d; int n = w->n, m = w->m;
  memset(w->K, 0, sizeof(double) * n * n);
  for (int i = 0; i < n; i++) w->K[i * n + i] = w->rho_x;
  if (d->P_indptr) for (int i = 0; i < n; i++) for (int k = d->P_indptr[i]; k < d->P_indptr[i + 1]; k++) {
    int j = d->P_indices[k]; /* upper: j >= i -> lower slot (j,i) */
    w->K[j * n + i] += w->Ph[k];
  }
  for (int i = 0; i < m; i++) {
    double ir = 1.0 / w->ry[i];
    for (int a = d->A_indptr[i]; a < d->A_indptr[i + 1]; a++) {
      double va = w->Ah[a] * ir; int ja = d->A_indices[a];
      for (int b2 = d->A_indptr[i]; b2 < d->A_indptr[i + 1]; b2++) {
        int jb = d->A_indices[b2];
        if (jb <= ja) w->K[ja * n + jb] += va * w->Ah[b2];
      }
    }
  }
  if (chol_lower(n, w->K)) return -1;
  /* g = (R_z + M)^{-1} h, h = (c, b) */
  for (int i = 0; i < m; i++) w->tm[i] = w->bh[i] / w->ry[i];
  csr_mtv(m, n, d->A_indptr, d->A_indices, w->Ah, w->tm, w->tn);
  for (int j = 0; j < n; j++) w->g[j] = w->ch[j] - w->tn[j];
  chol_solve(n, w->K, w->g);
  csr_mv(m, d->A_indptr, d->A_indices, w->Ah, w->g, w->tm);
  for (int i = 0; i < m; i++) w->g[n + i] = (w->bh[i] + w->tm[i]) / w->ry[i];
  double s = 0;
  for (int j = 0; j < n; j++) s += w->rho_x * w->g[j] * w->g[j];
  for (int i = 0; i < m; i++) s += w->ry[i] * w->g[n + i] * w->g[n + i];
  w->gRg = s;
  return 0;
}

static void set_ry(fwd_ws *w, double scale) {
  for (int i = 0; i < w->m; i++) w->ry[i] = (i < w->d->z) ? 1.0 / (ZERO_CONE_FACTOR * scale) : 1.0 / scale;
}

static int solve_impl(const orc_desc *d, const double *Av, const double *Pv, const double *b, const double *c,
                      const double *x0, const double *y0, const double *s0,
                      double *x, double *y, double *s, int32_t *iters, double *resid, const orc_settings *st);
int orc_solve(const orc_desc *d, const double *Av, const double *Pv, const double *b, const double *c,
              double *x, double *y, double *s, int32_t *iters, double *resid, const orc_settings *st) {
  return solve_impl(d, Av, Pv, b, c, NULL, NULL, NULL, x, y, s, iters, resid, st);
}
/* x0, y0, s0: a solution of a nearby problem (all three or none): the splitting starts at the fixed point it would be,
 * w = u + R^{-1} v with u = (x0 sigma / E, y0 sigma / D, 1), v_y = s0 D sigma (the inverse of the final un-scaling at tau = 1). */
int orc_solve_warm(const orc_desc *d, const double *Av, const double *Pv, const double *b, const double *c,
                   const double *x0, const double *y0, const double *s0,
                   double *x, double *y, double *s, int32_t *iters, double *resid, const orc_settings *st) {
  return solve_impl(d, Av, Pv, b, c, x0, y0, s0, x, y, s, iters, resid, st);
}
static int solve_impl(const orc_desc *d, const double *Av, const double *Pv, const double *b, const double *c,
                      const double *x0, const double *y0, const double *s0,
                      double *x, double *y, double *s, int32_t *iters, double *resid, const orc_settings *st) {
  int n = d->n, m = d->m, N = n + m + 1, nnzA = d->nnzA, nnzP = d->P_indptr ? d->nnzP : 0;
  size_t tot = (size_t)nnzA + nnzP + 3 * m + 3 * n + (size_t)n * n + (n + m) + n + m + 6 * (size_t)N + 2 * m + 2 * n;
  double *buf = (double *)calloc(tot + 16, sizeof(double)), *q = buf;
  fwd_ws W; W.n = n; W.m = m; W.d = d; W.rho_x = st->rho_x;
  W.Ah = q; q += nnzA; W.Ph = q; q += nnzP; W.D = q; q += m; W.E = q; q += n; W.bh = q; q += m; W.ch = q; q += n;
  W.ry = q; q += m; W.K = q; q += (size_t)n * n; W.g = q; q += n + m; W.tn = q; q += n; W.tm = q; q += m;
  double *w = q; q += N; double *u = q; q += N; double *ut = q; q += N; double *p = q; q += N; double *t = q; q += N;
  double *rsk = q; q += N; double *Axv = q; q += m; double *ATy = q; q += n; double *Pxv = q; q += n; double *tm2 = q; q += m;
  cblock *CB; int ncb = cone_blocks(d, &CB);
  aa_work *aa = NULL; double *wprev = NULL;

  memcpy(W.Ah, Av, sizeof(double) * nnzA);
  if (nnzP) memcpy(W.Ph, Pv, sizeof(double) * nnzP);
  for (int i = 0; i < m; i++) W.D[i] = 1.0;
  for (int j = 0; j < n; j++) W.E[j] = 1.0;
  /* --- Ruiz equilibration (SCS normalize.c, SURVEY.md 8a F4): D A E, E P E --- */
  if (st->normalize) for (int pass = 0; pass < st->ruiz_passes; pass++) {
    double *rn = W.tm, *cn = W.tn;
    for (int i = 0; i < m; i++) rn[i] = 0;
    for (int j = 0; j < n; j++) cn[j] = 0;
    for (int i = 0; i < m; i++) for (int k = d->A_indptr[i]; k < d->A_indptr[i + 1]; k++) {
      double a = fabs(W.Ah[k]); int j = d->A_indices[k];
      if (a > rn[i]) rn[i] = a;
      if (a > cn[j]) cn[j] = a;
    }
    if (nnzP) for (int i = 0; i < n; i++) for (int k = d->P_indptr[i]; k < d->P_indptr[i + 1]; k++) {
      double a = fabs(W.Ph[k]); int j = d->P_indices[k];
      if (a > cn[i]) cn[i] = a;
      if (a > cn[j]) cn[j] = a;
    }
    for (int i = 0; i < m; i++) { double v = rn[i] < 1e-8 ? 1.0 : 1.0 / sqrt(rn[i]); rn[i] = fmin(fmax(v, EQ_MIN), EQ_MAX); }
    for (int j = 0; j < n; j++) { double v = cn[j] < 1e-8 ? 1.0 : 1.0 / sqrt(cn[j]); cn[j] = fmin(fmax(v, EQ_MIN), EQ_MAX); }
    for (int k = 0; k < ncb; k++) if (CB[k].type >= CSOC) { /* one scale per non-separable cone */
      double mean = 0;
      for (int i = 0; i < CB[k].size; i++) mean += rn[CB[k].start + i];
      mean /= CB[k].size;
      for (int i = 0; i < CB[k].size; i++) rn[CB[k].start + i] = mean;
    }
    for (int i = 0; i < m; i++) for (int k = d->A_indptr[i]; k < d->A_indptr[i + 1]; k++) W.Ah[k] *= rn[i] * cn[d->A_indices[k]];
    if (nnzP) for (int i = 0; i < n; i++) for (int k = d->P_indptr[i]; k < d->P_indptr[i + 1]; k++) W.Ph[k] *= cn[i] * cn[d->P_indices[k]];
    for (int i = 0; i < m; i++) W.D[i] *= rn[i];
    for (int j = 0; j < n; j++) W.E[j] *= cn[j];
  }
  double nbh = 0, nch = 0, nb0 = 0, nc0 = 0;
  for (int i = 0; i < m; i++) { W.bh[i] = W.D[i] * b[i]; nbh = fmax(nbh, fabs(W.bh[i])); nb0 = fmax(nb0, fabs(b[i])); }
  for (int j = 0; j < n; j++) { W.ch[j] = W.E[j] * c[j]; nch = fmax(nch, fabs(W.ch[j])); nc0 = fmax(nc0, fabs(c[j])); }
  double sigma = fmax(nbh, nch);
  sigma = (!st->normalize || sigma < 1e-6) ? 1.0 : 1.0 / sigma;
  for (int i = 0; i < m; i++) W.bh[i] *= sigma;
  for (int j = 0; j < n; j++) W.ch[j] *= sigma;

  double scale = st->scale, dtau = TAU_FACTOR, alpha = st->alpha;
  set_ry(&W, scale);
  int status = ORC_INACCURATE, it = 0;
  double rp = NAN, rd = NAN, gap = NAN;
  if (factor(&W)) { status = ORC_FAILED; goto done; }
  w[N - 1] = 1.0;
  /* a warm start with a non-finite value (the NaN outputs of a non-solved instance) starts cold: from it tau never turns positive */
  int warm_ok = x0 && y0 && s0;
  for (int j = 0; warm_ok && j < n; j++) warm_ok = isfinite(x0[j]);
  for (int i = 0; warm_ok && i < m; i++) warm_ok = isfinite(y0[i]) && isfinite(s0[i]);
  if (warm_ok) {
    for (int j = 0; j < n; j++) w[j] = x0[j] * sigma / W.E[j];
    for (int i = 0; i < m; i++) w[n + i] = y0[i] * sigma / W.D[i] + s0[i] * W.D[i] * sigma / W.ry[i];
  }
  aa = aa_init(N, st->acceleration_lookback);
  if (aa) wprev = (double *)calloc(N, sizeof(double));
  const int aa_iv = st->acceleration_interval > 0 ? st->acceleration_interval : 1;
  double sum_log = 0; int n_log = 0, last_up = 0;
  /* adaptive check schedule: the distance to the tolerance is extrapolated log-linearly from the last
   * two checks and the next check is placed where convergence is predicted (same criteria, fewer
   * wasted iterations than a fixed stride) */
  int next_check = st->check_interval < 10 ? st->check_interval : 10, prev_it = 0; double prev_lr = 0;
  for (it = 1; it <= st->max_iters; it++) {
    /* Anderson acceleration of the iterate w (SCS: "accelerate here so that the last step is always a
     * projection onto the cone"): i = it - 1 is SCS's 0-based iteration counter. */
    const int aa_now = aa && it > 1 && (it - 1) % aa_iv == 0;
    double aa_nrm = 0.0;
    if (aa_now) aa_nrm = aa_apply(aa, w, wprev);
    if (aa) memcpy(wprev, w, sizeof(double) * N);
    /* affine step: ut = (R + Q)^{-1} R w   (SURVEY.md Appendix A.2 step 1) */
    csr_mtv(m, n, d->A_indptr, d->A_indices, W.Ah, w + n, W.tn);
    for (int j = 0; j < n; j++) p[j] = W.rho_x * w[j] - W.tn[j];
    chol_solve(n, W.K, p);
    csr_mv(m, d->A_indptr, d->A_indices, W.Ah, p, W.tm);
    for (int i = 0; i < m; i++) p[n + i] = w[n + i] + W.tm[i] / W.ry[i];
    double mu_g = 0, pRg = 0, pRp = 0, p_mu = 0;
    for (int j = 0; j < n; j++) { double r = W.rho_x; mu_g += r * w[j] * W.g[j]; pRg += r * p[j] * W.g[j]; pRp += r * p[j] * p[j]; p_mu += r * p[j] * w[j]; }
    for (int i = 0; i < m; i++) { double r = W.ry[i]; int k = n + i; mu_g += r * w[k] * W.g[k]; pRg += r * p[k] * W.g[k]; pRp += r * p[k] * p[k]; p_mu += r * p[k] * w[k]; }
    double qa = dtau + W.gRg, qb = mu_g - 2.0 * pRg - dtau * w[N - 1], qc = pRp - p_mu;
    double disc = qb * qb - 4.0 * qa * qc; if (disc < 0) disc = 0;
    double tau_t = (-qb + sqrt(disc)) / (2.0 * qa);
    for (int k = 0; k < n + m; k++) ut[k] = p[k] - tau_t * W.g[k];
    ut[N - 1] = tau_t;
    /* cone step: u = Pi_C(2 ut - w) */
    for (int k = 0; k < N; k++) { t[k] = 2.0 * ut[k] - w[k]; u[k] = t[k]; }
    proj_dual_blocks(CB, ncb, u + n);
    if (u[N - 1] < 0) u[N - 1] = 0;

    int check = st->adaptive_check ? (it >= next_check || it == st->max_iters) : ((it % st->check_interval == 0) || it == st->max_iters);
    if (check) {
      /* termination on the un-normalised data (SURVEY.md 8a F6) */
      double tau = u[N - 1];
      for (int i = 0; i < m; i++) rsk[n + i] = W.ry[i] * (u[n + i] - t[n + i]);
      csr_mv(m, d->A_indptr, d->A_indices, W.Ah, u, Axv);
      csr_mtv(m, n, d->A_indptr, d->A_indices, W.Ah, u + n, ATy);
      symu_mv(n, nnzP ? d->P_indptr : NULL, d->P_indices, W.Ph, u, Pxv);
      double xPx_u = dot(n, u, Pxv), ctx_u = dot(n, W.ch, u), bty_u = dot(m, W.bh, u + n);
      double nAx = 0, nS = 0, nPx = 0, nATy = 0, nAxs = 0;
      rp = 0; rd = 0;
      for (int i = 0; i < m; i++) {
        double sc = 1.0 / (W.D[i] * sigma);
        rp = fmax(rp, fabs(Axv[i] + rsk[n + i] - W.bh[i] * tau) * sc);
        nAx = fmax(nAx, fabs(Axv[i]) * sc); nS = fmax(nS, fabs(rsk[n + i]) * sc);
        nAxs = fmax(nAxs, fabs(Axv[i] + rsk[n + i]) * sc);
      }
      for (int j = 0; j < n; j++) {
        double sc = 1.0 / (W.E[j] * sigma);
        rd = fmax(rd, fabs(Pxv[j] + ATy[j] + W.ch[j] * tau) * sc);
        nPx = fmax(nPx, fabs(Pxv[j]) * sc); nATy = fmax(nATy, fabs(ATy[j]) * sc);
      }
      double s2 = sigma * sigma;
      if (tau > 1e-12) {
        double it_ = 1.0 / tau;
        double xPx = xPx_u * it_ * it_ / s2, ctx = ctx_u * it_ / s2, bty = bty_u * it_ / s2;
        rp *= it_; rd *= it_; gap = fabs(xPx + ctx + bty);
        double tp = st->eps_abs + st->eps_rel * fmax(fmax(nAx * it_, nS * it_), nb0);
        double td = st->eps_abs + st->eps_rel * fmax(fmax(nPx * it_, nATy * it_), nc0);
        double tg = st->eps_abs + st->eps_rel * fmax(fmax(fabs(xPx), fabs(ctx)), fabs(bty));
        if (rp <= tp && rd <= td && gap <= tg) { status = ORC_SOLVED; break; }
        if (st->adaptive_check) {
          double lr = log(fmax(fmax(rp / tp, rd / td), gap / tg));   /* > 0 while not converged */
          int step = st->check_interval;
          if (prev_it > 0 && lr < prev_lr) { double need = lr * (it - prev_it) / (prev_lr - lr); step = (int)ceil(0.9 * need) + 1; }
          if (step < 3) step = 3;
          if (step > st->check_interval) step = st->check_interval;
          prev_it = it; prev_lr = lr; next_check = it + step;
        }
        if (st->adaptive_scale) {
          double relp = rp / fmax(fmax(fmax(nAx * it_, nS * it_), nb0), 1e-18);
          double reld = rd / fmax(fmax(fmax(nPx * it_, nATy * it_), nc0), 1e-18);
          if (relp > 0 && reld > 0) { sum_log += log(relp) - log(reld); n_log++; }
        }
      }
      if (st->adaptive_check && next_check <= it) next_check = it + st->check_interval;
      /* certificates (homogeneous in u, so no division by tau) */
      double bty_c = bty_u / s2, ctx_c = ctx_u / s2;
      if (bty_c < 0 && nATy / (-bty_c) <= st->eps_infeas) { status = ORC_INFEASIBLE; break; }
      if (ctx_c < 0 && fmax(nPx, nAxs) / (-ctx_c) <= st->eps_infeas) { status = ORC_UNBOUNDED; break; }
      if (st->adaptive_scale && n_log > 0 && it - last_up >= RESCALE_MIN_ITERS) {
        double fac = sqrt(exp(sum_log / n_log));
        if (fac > 3.1622776601683795 || fac < 0.31622776601683794) {
          double ns = fmin(fmax(scale * fac, MIN_SCALE), MAX_SCALE);
          if (ns != scale) {
            for (int i = 0; i < m; i++) tm2[i] = W.ry[i];
            scale = ns; set_ry(&W, scale);
            if (factor(&W)) { status = ORC_FAILED; break; }
            /* keep R(w + u - 2 ut) invariant across the metric change */
            for (int i = 0; i < m; i++) { int k = n + i; w[k] = (tm2[i] / W.ry[i]) * (w[k] + u[k] - 2.0 * ut[k]) + 2.0 * ut[k] - u[k]; }
            sum_log = 0; n_log = 0; last_up = it;
            aa_reset(aa);   /* the fixed-point map changed */
            aa_nrm = 0.0;
          }
        }
      }
    }
    for (int k = 0; k < N; k++) w[k] += alpha * (u[k] - ut[k]);
    /* safeguard after the convergence check (it acts on w, convergence is judged on u) */
    if (aa_now && aa_nrm > 0) aa_safeguard(aa, w, wprev);
  }
  if (it > st->max_iters) it = st->max_iters;
  {
    double tau = u[N - 1];
    if (status == ORC_INACCURATE && !(tau > 1e-12)) status = ORC_FAILED;   /* iteration limit without a positive tau: no usable point */
    if (status == ORC_SOLVED || status == ORC_INACCURATE) {
      if (!(tau > 1e-12)) tau = 1e-12;
      for (int i = 0; i < m; i++) rsk[n + i] = W.ry[i] * (u[n + i] - t[n + i]);
      for (int j = 0; j < n; j++) x[j] = W.E[j] * u[j] / (sigma * tau);
      for (int i = 0; i < m; i++) { y[i] = W.D[i] * u[n + i] / (sigma * tau); s[i] = rsk[n + i] / (W.D[i] * sigma * tau); }
    } else {
      for (int j = 0; j < n; j++) x[j] = NAN;
      for (int i = 0; i < m; i++) { y[i] = NAN; s[i] = NAN; }
    }
  }
done:
  if (iters) *iters = it;
  if (resid) { resid[0] = rp; resid[1] = rd; resid[2] = gap; }
  aa_free(aa); free(wprev);
  free(CB); free(buf);
  return status;
}

/* ------------------------------------------------------------------- LSQR */
typedef void (*lin_fn)(void *ctx, const double *in, double *out);

/* Solve min ||B r - rhs|| for a square/rectangular operator: mv = B, mtv = B'.
 * Paige & Saunders LSQR with the SciPy stopping rules (damp = 0). */
static int lsqr_core(int rows, int cols, lin_fn mv, lin_fn mtv, void *ctx, const double *rhs, double *xs,
                     double atol, double btol, double conlim, int iter_lim) {
  double *u = (double *)calloc((size_t)2 * rows + 3 * cols, sizeof(double));
  double *tu = u + rows, *v = tu + rows, *w = v + cols, *tv = w + cols;
  const double eps = 2.220446049250313e-16;
  double ctol = conlim > 0 ? 1.0 / conlim : 0.0;
  if (iter_lim < 0) iter_lim = 2 * cols;
  int itn = 0;
  for (int j = 0; j < cols; j++) xs[j] = 0;
  memcpy(u, rhs, sizeof(double) * rows);
  double bnorm = nrm2(rows, rhs), beta = bnorm, alfa = 0;
  if (beta > 0) { for (int i = 0; i < rows; i++) u[i] /= beta; mtv(ctx, u, v); alfa = nrm2(cols, v); }
  if (alfa > 0) { for (int j = 0; j < cols; j++) { v[j] /= alfa; w[j] = v[j]; } }
  double rhobar = alfa, phibar = beta, anorm = 0, ddnorm = 0, xxnorm = 0, z = 0, cs2 = -1, sn2 = 0;
  double arnorm = alfa * beta;
  if (arnorm == 0) { free(u); return 0; }
  while (itn < iter_lim) {
    itn++;
    mv(ctx, v, tu);
    for (int i = 0; i < rows; i++) u[i] = tu[i] - alfa * u[i];
    beta = nrm2(rows, u);
    if (beta > 0) {
      for (int i = 0; i < rows; i++) u[i] /= beta;
      anorm = sqrt(anorm * anorm + alfa * alfa + beta * beta);
      mtv(ctx, u, tv);
      for (int j = 0; j < cols; j++) v[j] = tv[j] - beta * v[j];
      alfa = nrm2(cols, v);
      if (alfa > 0) for (int j = 0; j < cols; j++) v[j] /= alfa;
    }
    double rho = hypot(rhobar, beta), cs = rhobar / rho, sn = beta / rho;
    double theta = sn * alfa; rhobar = -cs * alfa;
    double phi = cs * phibar; phibar = sn * phibar;
    double tau = sn * phi;
    double t1 = phi / rho, t2 = -theta / rho, dd = 0;
    for (int j = 0; j < cols; j++) { double dk = w[j] / rho; dd += dk * dk; xs[j] += t1 * w[j]; w[j] = v[j] + t2 * w[j]; }
    ddnorm += dd;
    double delta = sn2 * rho, gambar = -cs2 * rho, rhs_ = phi - delta * z, zbar = rhs_ / gambar;
    double xnorm = sqrt(xxnorm + zbar * zbar);
    double gamma = hypot(gambar, theta); cs2 = gambar / gamma; sn2 = theta / gamma; z = rhs_ / gamma; xxnorm += z * z;
    double acond = anorm * sqrt(ddnorm), rnorm = phibar;
    arnorm = alfa * fabs(tau);
    double test1 = rnorm / bnorm, test2 = arnorm / (anorm * rnorm + eps), test3 = 1.0 / (acond + eps);
    double tt1 = test1 / (1.0 + anorm * xnorm / bnorm), rtol = btol + atol * anorm * xnorm / bnorm;
    int istop = 0;
    if (itn >= iter_lim) istop = 7;
    if (1.0 + test3 <= 1.0) istop = 6;
    if (1.0 + test2 <= 1.0) istop = 5;
    if (1.0 + tt1 <= 1.0) istop = 4;
    if (test3 <= ctol) istop = 3;
    if (test2 <= atol) istop = 2;
    if (test1 <= rtol) istop = 1;
    if (istop) break;
  }
  free(u);
  return itn;
}

typedef struct { int r, c; const double *M; } dense_ctx;
static void dense_mv(void *c_, const double *in, double *out) {
  dense_ctx *c = (dense_ctx *)c_;
  for (int i = 0; i < c->r; i++) { double a = 0; for (int j = 0; j < c->c; j++) a += c->M[(size_t)i * c->c + j] * in[j]; out[i] = a; }
}
static void dense_mtv(void *c_, const double *in, double *out) {
  dense_ctx *c = (dense_ctx *)c_;
  for (int j = 0; j < c->c; j++) out[j] = 0;
  for (int i = 0; i < c->r; i++) for (int j = 0; j < c->c; j++) out[j] += c->M[(size_t)i * c->c + j] * in[i];
}
int orc_lsqr_dense(int32_t rows, int32_t cols, const double *Mrow, const double *rhs, double *sol,
                   double atol, double btol, double conlim, int32_t iter_lim) {
  dense_ctx c = {rows, cols, Mrow};
  return lsqr_core(rows, cols, dense_mv, dense_mtv, &c, rhs, sol, atol, btol, conlim, iter_lim);
}

/* --------------------------------------------------------------- backward */
typedef struct {
  const orc_desc *d; int n, m;
  const double *Av, *Pv, *b, *c, *v, *x;
  double xPx; double *Px2c; /* 2 P x + c */
  const cblock *CB; int ncb;
  double *Ls, *Rs, *t4; /* diagonal equilibration of the LSQR system (lsqr_precond) */
  double *t1, *t2, *t3;
} bwd_ctx;

/* DQ(pi_z) at pi_z = (x, y, 1):  [[P, A', c], [-A, 0, b], [-(2Px + c)', -b', x'Px]] */
static void apply_DQ(bwd_ctx *k, const double *in, double *out) {
  int n = k->n, m = k->m; const orc_desc *d = k->d;
  csr_mtv(m, n, d->A_indptr, d->A_indices, k->Av, in + n, out);
  if (d->P_indptr) { symu_mv(n, d->P_indptr, d->P_indices, k->Pv, in, k->t3); for (int j = 0; j < n; j++) out[j] += k->t3[j]; }
  for (int j = 0; j < n; j++) out[j] += k->c[j] * in[n + m];
  csr_mv(m, d->A_indptr, d->A_indices, k->Av, in, out + n);
  for (int i = 0; i < m; i++) out[n + i] = -out[n + i] + k->b[i] * in[n + m];
  out[n + m] = -dot(n, k->Px2c, in) - dot(m, k->b, in + n) + k->xPx * in[n + m];
}
static void apply_DQT(bwd_ctx *k, const double *in, double *out) {
  int n = k->n, m = k->m; const orc_desc *d = k->d;
  /* DQ' = [[P, -A', -(2Px + c)], [A, 0, -b], [c', b', x'Px]] */
  csr_mtv(m, n, d->A_indptr, d->A_indices, k->Av, in + n, out);
  for (int j = 0; j < n; j++) out[j] = -out[j];
  if (d->P_indptr) { symu_mv(n, d->P_indptr, d->P_indices, k->Pv, in, k->t3); for (int j = 0; j < n; j++) out[j] += k->t3[j]; }
  for (int j = 0; j < n; j++) out[j] -= k->Px2c[j] * in[n + m];
  csr_mv(m, d->A_indptr, d->A_indices, k->Av, in, out + n);
  for (int i = 0; i < m; i++) out[n + i] -= k->b[i] * in[n + m];
  out[n + m] = dot(n, k->c, in) + dot(m, k->b, in + n) + k->xPx * in[n + m];
}
/* M = (DQ - I) Dpi + I  (SURVEY.md 8a row B2) */
static void op_M(void *c_, const double *in, double *out) {
  bwd_ctx *k = (bwd_ctx *)c_; int n = k->n, m = k->m, N = n + m + 1;
  memcpy(k->t1, in, sizeof(double) * N);
  dproj_dual_blocks(k->CB, k->ncb, k->v, in + n, k->t1 + n);
  apply_DQ(k, k->t1, out);
  for (int i = 0; i < N; i++) out[i] += in[i] - k->t1[i];
}
static void op_MT(void *c_, const double *in, double *out) {
  bwd_ctx *k = (bwd_ctx *)c_; int n = k->n, m = k->m, N = n + m + 1;
  apply_DQT(k, in, k->t1);
  for (int i = 0; i < N; i++) k->t1[i] -= in[i];
  memcpy(k->t2, k->t1, sizeof(double) * N);
  dproj_dual_blocks(k->CB, k->ncb, k->v, k->t1 + n, k->t2 + n); /* Dpi is symmetric for every cone handled */
  for (int i = 0; i < N; i++) out[i] = k->t2[i] + in[i];
}

/* B' = diag(Ls) M' diag(Rs) and its transpose */
static void op_Bs(void *c_, const double *in, double *out) {
  bwd_ctx *k = (bwd_ctx *)c_; int N = k->n + k->m + 1;
  for (int i = 0; i < N; i++) k->t4[i] = k->Rs[i] * in[i];
  op_MT(c_, k->t4, out);
  for (int i = 0; i < N; i++) out[i] *= k->Ls[i];
}
static void op_BsT(void *c_, const double *in, double *out) {
  bwd_ctx *k = (bwd_ctx *)c_; int N = k->n + k->m + 1;
  for (int i = 0; i < N; i++) k->t4[i] = k->Ls[i] * in[i];
  op_M(c_, k->t4, out);
  for (int i = 0; i < N; i++) out[i] *= k->Rs[i];
}

/* 2-norm Ruiz scaling of a surrogate of M' (cone Jacobian replaced by its 0/1 skeleton:
 * zero rows and active nonneg rows 1, inactive nonneg rows dropped -- their unknown is exactly
 * dz_i = 0 --, SOC/PSD rows 1 with a unit diagonal standing in for I - D).  A diagonally
 * rescaled system has the same solution wherever the solution map is differentiable. */
static void lsqr_equilibrate(bwd_ctx *k, const double *piy_unused, int passes) {
  const orc_desc *d = k->d; int n = k->n, m = k->m, N = n + m + 1;
  double *L = k->Ls, *R = k->Rs;
  double *rs = (double *)calloc(2 * (size_t)N + m, sizeof(double)), *cs = rs + N, *dg = cs + N;
  int lo = d->z, hi = d->z + d->l;
  for (int i = 0; i < N; i++) { L[i] = 1.0; R[i] = 1.0; }
  for (int i = 0; i < m; i++) {
    int live = !(i >= lo && i < hi) || k->v[i] > 0;
    if (!live) { L[n + i] = 0.0; R[n + i] = 0.0; }
    dg[i] = (i >= hi) ? 1.0 : 0.0; /* surrogate of (I - D) on non-polyhedral rows */
  }
  for (int pass = 0; pass < passes; pass++) {
    for (int i = 0; i < 2 * N; i++) rs[i] = 0;
    /* A block: x-row j / y-col i carry -A_ij ; y-row i / x-col j carry A_ij */
    for (int i = 0; i < m; i++) for (int a = d->A_indptr[i]; a < d->A_indptr[i + 1]; a++) {
      int j = d->A_indices[a]; double v2 = k->Av[a] * k->Av[a];
      double e1 = v2 * L[j] * L[j] * R[n + i] * R[n + i];       /* (x-row j, y-col i) */
      double e2 = v2 * L[n + i] * L[n + i] * R[j] * R[j];       /* (y-row i, x-col j) */
      rs[j] += e1; cs[n + i] += e1; rs[n + i] += e2; cs[j] += e2;
    }
    if (d->P_indptr) for (int i = 0; i < n; i++) for (int a = d->P_indptr[i]; a < d->P_indptr[i + 1]; a++) {
      int j = d->P_indices[a]; double v2 = k->Pv[a] * k->Pv[a];
      double e1 = v2 * L[i] * L[i] * R[j] * R[j];
      rs[i] += e1; cs[j] += e1;
      if (i != j) { double e2 = v2 * L[j] * L[j] * R[i] * R[i]; rs[j] += e2; cs[i] += e2; }
    }
    for (int j = 0; j < n; j++) {
      double e1 = k->Px2c[j] * k->Px2c[j] * L[j] * L[j] * R[N - 1] * R[N - 1]; rs[j] += e1; cs[N - 1] += e1;
      double e2 = k->c[j] * k->c[j] * L[N - 1] * L[N - 1] * R[j] * R[j]; rs[N - 1] += e2; cs[j] += e2;
    }
    for (int i = 0; i < m; i++) {
      double b2 = k->b[i] * k->b[i];
      double e1 = b2 * L[n + i] * L[n + i] * R[N - 1] * R[N - 1]; rs[n + i] += e1; cs[N - 1] += e1;
      double e2 = b2 * L[N - 1] * L[N - 1] * R[n + i] * R[n + i]; rs[N - 1] += e2; cs[n + i] += e2;
      double e3 = dg[i] * L[n + i] * L[n + i] * R[n + i] * R[n + i]; rs[n + i] += e3; cs[n + i] += e3;
    }
    { double e = k->xPx * k->xPx * L[N - 1] * L[N - 1] * R[N - 1] * R[N - 1]; rs[N - 1] += e; cs[N - 1] += e; }
    for (int i = 0; i < N; i++) {
      if (L[i] > 0 && rs[i] > 1e-300) L[i] /= sqrt(sqrt(rs[i]));
      if (R[i] > 0 && cs[i] > 1e-300) R[i] /= sqrt(sqrt(cs[i]));
    }
  }
  free(rs);
}

/* ---- lsqr_precond = 2: LSQR right-preconditioned by the exact block factorisation of the KKT part
 * of the reduced system.  With live rows L (zero rows + active nonneg rows), the reduced matrix is
 *     B = [[G, -h'], [g', x'Px]],   G = [[P, -A_L'], [A_L, 0]],  h' = (2Px + c ; b_L),  g = (c ; b_L),
 * and B blkdiag(G,1)^{-1} = [[I, -h'], [(G^{-T} g)', x'Px]] is the identity plus a rank-2 term, so LSQR
 * converges in a handful of O(N) iterations; the singular homogeneity direction is still resolved by
 * LSQR's minimum-norm property.  Needs P > 0 and A_L of full row rank (both checked by the Cholesky
 * factorisations of P and of S = A_L P^{-1} A_L'); otherwise the caller falls back to lsqr_precond = 1.
 * Returns LSQR iterations, or -1 if the factorisation is not applicable. */
typedef struct { int nr; const double *hp, *q; double xPx; } border_ctx;
static void border_mv(void *c_, const double *in, double *out) {   /* C z */
  border_ctx *c = (border_ctx *)c_; int nr = c->nr; double zt = in[nr], acc = 0;
  for (int i = 0; i < nr; i++) { out[i] = in[i] - c->hp[i] * zt; acc += c->q[i] * in[i]; }
  out[nr] = acc + c->xPx * zt;
}
static void border_mtv(void *c_, const double *in, double *out) {  /* C' u */
  border_ctx *c = (border_ctx *)c_; int nr = c->nr; double ut = in[nr], acc = 0;
  for (int i = 0; i < nr; i++) { out[i] = in[i] + c->q[i] * ut; acc += c->hp[i] * in[i]; }
  out[nr] = -acc + c->xPx * ut;
}
static int vjp_block_precond(const orc_desc *d, bwd_ctx *K, const double *piy, const double *dz, double *r, const orc_settings *st) {
  int n = d->n, m = d->m, N = n + m + 1, lo = d->z, hi = d->z + d->l;
  if (!d->P_indptr || d->nq || d->ns || d->ep || d->ed) return -1;
  int *live = (int *)malloc(sizeof(int) * (m + 1)), nl = 0;
  for (int i = 0; i < m; i++) if (i < lo || i >= hi || piy[i] > 0) live[nl++] = i;
  if (nl > n) { free(live); return -1; }
  int nr = n + nl;
  double *Lp = (double *)calloc((size_t)n * n + (size_t)nl * n + (size_t)nl * nl + 6 * (size_t)(nr + 1) + 2 * n, sizeof(double));
  double *W = Lp + (size_t)n * n, *S = W + (size_t)nl * n, *hp = S + (size_t)nl * nl, *q = hp + nr + 1, *rhs = q + nr + 1, *z = rhs + nr + 1,
         *t1 = z + nr + 1, *t2 = t1 + nr + 1, *tn = t2 + nr + 1;
  int ok = 1;
  for (int i = 0; i < n; i++) for (int k = d->P_indptr[i]; k < d->P_indptr[i + 1]; k++) Lp[(size_t)d->P_indices[k] * n + i] += K->Pv[k];  /* lower */
  if (chol_lower(n, Lp)) ok = 0;
  if (ok) {
    for (int l = 0; l < nl; l++) {                       /* W_l = L^{-1} a_l */
      double *w = W + (size_t)l * n; int i0 = live[l];
      for (int j = 0; j < n; j++) w[j] = 0;
      for (int k = d->A_indptr[i0]; k < d->A_indptr[i0 + 1]; k++) w[d->A_indices[k]] = K->Av[k];
      for (int i = 0; i < n; i++) { double a = w[i]; for (int k = 0; k < i; k++) a -= Lp[(size_t)i * n + k] * w[k]; w[i] = a / Lp[(size_t)i * n + i]; }
    }
    for (int a = 0; a < nl; a++) for (int b2 = 0; b2 <= a; b2++) S[(size_t)a * nl + b2] = dot(n, W + (size_t)a * n, W + (size_t)b2 * n);
    if (nl > 0 && chol_lower(nl, S)) ok = 0;
  }
  if (!ok) { free(Lp); free(live); return -1; }
  /* G^{-1}(f, g) and G^{-T}(f, g); tr = +1 for G, -1 for G' (sign of the A_L coupling) */
#define GSOLVE(f, g, ox, oL, tr)                                                                          \
  do {                                                                                                    \
    for (int i = 0; i < n; i++) { double a = (f)[i]; for (int k = 0; k < i; k++) a -= Lp[(size_t)i * n + k] * tn[k]; tn[i] = a / Lp[(size_t)i * n + i]; } \
    for (int l = 0; l < nl; l++) (oL)[l] = (tr) * ((g)[l] - (tr) * dot(n, W + (size_t)l * n, tn));      \
    if (nl > 0) chol_solve(nl, S, (oL));                                                                  \
    for (int i = 0; i < n; i++) { double a = tn[i]; for (int l = 0; l < nl; l++) a += (tr) * W[(size_t)l * n + i] * (oL)[l]; (ox)[i] = a; } \
    for (int i = n - 1; i >= 0; i--) { double a = (ox)[i]; for (int k = i + 1; k < n; k++) a -= Lp[(size_t)k * n + i] * (ox)[k]; (ox)[i] = a / Lp[(size_t)i * n + i]; } \
  } while (0)
  /* G  : P rx - A_L' rL = f,  A_L rx = g  ->  S rL = g - A_L P^{-1} f,          rx = P^{-1}(f + A_L' rL)
     G' : P rx + A_L' rL = f, -A_L rx = g  ->  S rL = -(g) ... = -(g + ... ) see tr handling: rL = -(g - (-1) A_L P^{-1} f)... */
  for (int i = 0; i < n; i++) { hp[i] = K->Px2c[i]; q[i] = K->c[i]; }
  for (int l = 0; l < nl; l++) { hp[n + l] = K->b[live[l]]; q[n + l] = K->b[live[l]]; }
  /* q <- G^{-T} g:  P qx + A_L' qL = c ; -A_L qx = b_L */
  {
    double *gx = t1, *gL = t1 + n; memcpy(gx, q, sizeof(double) * n); memcpy(gL, q + n, sizeof(double) * nl);
    /* S qL = -(b_L + A_L P^{-1} c) ... derive: qx = P^{-1}(c - A_L' qL); -A_L P^{-1}(c - A_L' qL) = b_L -> S qL = b_L + A_L P^{-1} c */
    for (int i = 0; i < n; i++) { double a = gx[i]; for (int k = 0; k < i; k++) a -= Lp[(size_t)i * n + k] * tn[k]; tn[i] = a / Lp[(size_t)i * n + i]; }
    for (int l = 0; l < nl; l++) q[n + l] = gL[l] + dot(n, W + (size_t)l * n, tn);
    if (nl > 0) chol_solve(nl, S, q + n);
    for (int i = 0; i < n; i++) { double a = tn[i]; for (int l = 0; l < nl; l++) a -= W[(size_t)l * n + i] * q[n + l]; q[i] = a; }
    for (int i = n - 1; i >= 0; i--) { double a = q[i]; for (int k = i + 1; k < n; k++) a -= Lp[(size_t)k * n + i] * q[k]; q[i] = a / Lp[(size_t)i * n + i]; }
  }
  for (int i = 0; i < n; i++) rhs[i] = dz[i];
  for (int l = 0; l < nl; l++) rhs[n + l] = dz[n + live[l]];
  rhs[nr] = dz[N - 1];
  border_ctx bc = {nr, hp, q, K->xPx};
  int its = lsqr_core(nr + 1, nr + 1, border_mv, border_mtv, &bc, rhs, z, st->lsqr_atol, st->lsqr_btol, st->lsqr_conlim, st->lsqr_iter_lim);
  /* r = blkdiag(G,1)^{-1} z */
  for (int i = 0; i < N; i++) r[i] = 0;
  {
    double *ox = t2, *oL = t2 + n;
    GSOLVE(z, z + n, ox, oL, 1.0);
    for (int i = 0; i < n; i++) r[i] = ox[i];
    for (int l = 0; l < nl; l++) r[n + live[l]] = oL[l];
  }
  r[N - 1] = z[nr];
#undef GSOLVE
  free(Lp); free(live);
  return its;
}

int orc_vjp(const orc_desc *d, const double *Av, const double *Pv, const double *b, const double *c,
            const double *x, const double *y, const double *s, const double *dx, const double *dy,
            double *dAv, double *dPv, double *db, double *dc, const orc_settings *st) {
  int n = d->n, m = d->m, N = n + m + 1;
  double *buf = (double *)calloc((size_t)12 * N + 4 * n + 2 * m, sizeof(double)), *q = buf;
  double *v = q; q += m; double *piy = q; q += m; double *dz = q; q += N; double *r = q; q += N;
  bwd_ctx K; K.d = d; K.n = n; K.m = m; K.Av = Av; K.Pv = Pv; K.b = b; K.c = c; K.v = v; K.x = x;
  K.t1 = q; q += N; K.t2 = q; q += N; K.t3 = q; q += N; K.Px2c = q; q += n;
  K.Ls = q; q += N; K.Rs = q; q += N; K.t4 = q; q += N;
  cblock *CB; K.ncb = cone_blocks(d, &CB); K.CB = CB;
  for (int i = 0; i < m; i++) { v[i] = y[i] - s[i]; piy[i] = v[i]; }
  orc_proj_dual_cone(d, piy);
  if (d->P_indptr) { symu_mv(n, d->P_indptr, d->P_indices, Pv, x, K.t3); K.xPx = dot(n, x, K.t3); for (int j = 0; j < n; j++) K.Px2c[j] = 2.0 * K.t3[j] + c[j]; }
  else { K.xPx = 0; for (int j = 0; j < n; j++) K.Px2c[j] = c[j]; }
  /* dz = [dx ; DPi'(dy + ds) - ds ; -(x'dx + y'dy + s'ds)], ds = 0 (diffcp_if.py:84) */
  memcpy(dz, dx, sizeof(double) * n);
  orc_dproj_dual_cone(d, v, dy, dz + n);
  dz[N - 1] = -(dot(n, x, dx) + dot(m, y, dy));
  int its = 0, allz = 1;
  for (int i = 0; i < N; i++) if (fabs(dz[i]) > 1e-8) { allz = 0; break; }
  int done = 0;
  if (!allz && st->lsqr_precond == 2) { int k2 = vjp_block_precond(d, &K, piy, dz, r, st); if (k2 >= 0) { its = k2; done = 1; } }
  if (done) { /* solved with the block preconditioner */ }
  else if (!allz && st->lsqr_precond) {
    lsqr_equilibrate(&K, piy, st->ruiz_passes > 0 ? st->ruiz_passes : 10);
    for (int i = 0; i < N; i++) dz[i] *= K.Ls[i];
    its = lsqr_core(N, N, op_Bs, op_BsT, &K, dz, r, st->lsqr_atol, st->lsqr_btol, st->lsqr_conlim, st->lsqr_iter_lim);
    for (int i = 0; i < N; i++) r[i] *= K.Rs[i];
  } else if (!allz)
    its = lsqr_core(N, N, op_MT, op_M, &K, dz, r, st->lsqr_atol, st->lsqr_btol, st->lsqr_conlim, st->lsqr_iter_lim);
  /* gradient assembly on EVERY structural entry (SURVEY.md 8a row B4 and the A.nonzero() hazard note) */
  double rt = r[N - 1];
  for (int i = 0; i < m; i++) for (int k = d->A_indptr[i]; k < d->A_indptr[i + 1]; k++) {
    int j = d->A_indices[k];
    dAv[k] = x[j] * r[n + i] - piy[i] * r[j];
  }
  for (int i = 0; i < m; i++) db[i] = piy[i] * rt - r[n + i];
  for (int j = 0; j < n; j++) dc[j] = x[j] * rt - r[j];
  if (dPv && d->P_indptr) for (int i = 0; i < n; i++) for (int k = d->P_indptr[i]; k < d->P_indptr[i + 1]; k++) {
    int j = d->P_indices[k];
    double gij = (rt * x[i] - r[i]) * x[j], gji = (rt * x[j] - r[j]) * x[i];
    dPv[k] = (i == j) ? gij : gij + gji;
  }
  free(buf); free(CB);
  return its;
}

/* ------------------------------------------------------------ batch drivers */
/* Every instance allocates and frees a few hundred KB of scratch.  Above glibc's default mmap threshold each of those
 * is an mmap / munmap pair, and with ~128 threads doing that concurrently the kernel's address-space lock decides the
 * run time (the same batch took between 0.5 and 2.9 s on otherwise identical hosts).  Keep the scratch in the
 * per-thread malloc arenas instead. */
static void tune_malloc(void) {
  static int done = 0;
  if (done) return;
  done = 1;
  mallopt(M_MMAP_THRESHOLD, 1 << 29);
  mallopt(M_TRIM_THRESHOLD, 1 << 29);
  mallopt(M_TOP_PAD, 1 << 24);
}
void orc_solve_batch(const orc_desc *d, int32_t B, const double *Av, const double *Pv, const double *b,
                     const double *c, double *x, double *y, double *s, int32_t *status, int32_t *iters,
                     const orc_settings *st, int32_t nthreads) {
  int n = d->n, m = d->m; size_t nA = d->nnzA, nP = d->P_indptr ? d->nnzP : 0;
  tune_malloc();
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads)
#endif
  for (int i = 0; i < B; i++) {
    int32_t itc = 0;
    int stt = orc_solve(d, Av + i * nA, nP ? Pv + i * nP : NULL, b + (size_t)i * m, c + (size_t)i * n,
                        x + (size_t)i * n, y + (size_t)i * m, s + (size_t)i * m, &itc, NULL, st);
    if (status) status[i] = stt;
    if (iters) iters[i] = itc;
  }
}

void orc_solve_batch_warm(const orc_desc *d, int32_t B, const double *Av, const double *Pv, const double *b,
                          const double *c, const double *x0, const double *y0, const double *s0, double *x, double *y, double *s,
                          int32_t *status, int32_t *iters, const orc_settings *st, int32_t nthreads) {
  int n = d->n, m = d->m; size_t nA = d->nnzA, nP = d->P_indptr ? d->nnzP : 0;
  tune_malloc();
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads)
#endif
  for (int i = 0; i < B; i++) {
    int32_t itc = 0;
    int stt = solve_impl(d, Av + i * nA, nP ? Pv + i * nP : NULL, b + (size_t)i * m, c + (size_t)i * n,
                         x0 ? x0 + (size_t)i * n : NULL, y0 ? y0 + (size_t)i * m : NULL, s0 ? s0 + (size_t)i * m : NULL,
                         x + (size_t)i * n, y + (size_t)i * m, s + (size_t)i * m, &itc, NULL, st);
    if (status) status[i] = stt;
    if (iters) iters[i] = itc;
  }
}

void orc_vjp_batch(const orc_desc *d, int32_t B, const double *Av, const double *Pv, const double *b,
                   const double *c, const double *x, const double *y, const double *s, const double *dx,
                   const double *dy, double *dAv, double *dPv, double *db, double *dc, int32_t *lsqr_iters,
                   const orc_settings *st, int32_t nthreads) {
  int n = d->n, m = d->m; size_t nA = d->nnzA, nP = d->P_indptr ? d->nnzP : 0;
  tune_malloc();
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads)
#endif
  for (int i = 0; i < B; i++) {
    int its = orc_vjp(d, Av + i * nA, nP ? Pv + i * nP : NULL, b + (size_t)i * m, c + (size_t)i * n,
                      x + (size_t)i * n, y + (size_t)i * m, s + (size_t)i * m, dx + (size_t)i * n,
                      dy + (size_t)i * m, dAv + i * nA, (dPv && nP) ? dPv + i * nP : NULL,
                      db + (size_t)i * m, dc + (size_t)i * n, st);
    if (lsqr_iters) lsqr_iters[i] = its;
  }
}
