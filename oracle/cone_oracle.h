/*
 * cone_oracle.h -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * Plain-C, fp64 restatement of the hot path the reference delegates to
 * diffcp 1.1.4 + SCS 3.2.9 (neither is vendored in the reference nor
 * installable here, see DESIGN.md "Oracle"):
 *   forward : diffcp.solve_and_derivative_batch  (reference call site
 *             src/cvxpylayers/interfaces/diffcp_if.py:365, :369)
 *   backward: the adjoint closure adj_batch        (diffcp_if.py:86)
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library.  The product path
 * (cvxpylayers_b200/) never does.
 *
 * PARITY PIN STATUS: the reference holds no golden vectors for this path
 * (SURVEY.md section 8c).  This oracle is pinned against the analytic known
 * answers of the reference's own tests (closed-form ridge regression
 * tests/test_torch.py:90-118, x*=[1,1] tests/test_diffcp_optional_deps.py:29-57),
 * against SciPy's LSQR (the routine diffcp's lsqr.cpp ports), HiGHS on LPs,
 * central finite differences and solver-independent KKT certificates.
 * Iteration-level / bit-level parity with diffcp+SCS binaries: UNPINNED.
 */
#ifndef CONE_ORACLE_H
#define CONE_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Structure shared by the whole batch (same layout as include/bcone.h). */
typedef struct {
  int32_t n, m, nnzA, nnzP;
  const int32_t *A_indptr, *A_indices; /* CSR, m+1 / nnzA                  */
  const int32_t *P_indptr, *P_indices; /* CSR upper triangle incl. diag, or NULL */
  int32_t z, l, nq, ns, ep, ed;        /* cone spec in SCS row order z,l,q,s,ep,ed */
  const int32_t *q, *s;                /* SOC sizes [nq], PSD matrix orders [ns]   */
} orc_desc;

typedef struct {
  double eps_abs, eps_rel, eps_infeas;
  double alpha, rho_x, scale;
  double lsqr_atol, lsqr_btol, lsqr_conlim;
  int32_t max_iters, normalize, adaptive_scale, check_interval;
  int32_t ruiz_passes, lsqr_iter_lim, lsqr_precond, adaptive_check;
  int32_t acceleration_lookback;  /* SCS: Anderson acceleration window, 10 (type-I); < 0 type-II; 0 off */
  int32_t acceleration_interval;  /* SCS: accelerate every this many iterations, 10 */
} orc_settings;

enum { ORC_SOLVED = 1, ORC_INACCURATE = 2, ORC_UNBOUNDED = -1, ORC_INFEASIBLE = -2, ORC_FAILED = -4 };

void orc_default_settings(orc_settings *st);

/* One instance.  Solver form: min 1/2 x'Px + c'x  s.t. Ax + s = b, s in K.
 * resid[0..2] = final primal / dual residual inf-norms and |gap| on the
 * un-normalised data (SCS termination quantities). Returns status. */
int orc_solve(const orc_desc *d, const double *Av, const double *Pv, const double *b,
              const double *c, double *x, double *y, double *s, int32_t *iters,
              double *resid, const orc_settings *st);

/* Warm-started variants (a previous solution x0, y0, s0 of a nearby problem; SURVEY.md 8f.2). */
int orc_solve_warm(const orc_desc *d, const double *Av, const double *Pv, const double *b, const double *c,
                   const double *x0, const double *y0, const double *s0,
                   double *x, double *y, double *s, int32_t *iters, double *resid, const orc_settings *st);
void orc_solve_batch_warm(const orc_desc *d, int32_t B, const double *Av, const double *Pv, const double *b,
                          const double *c, const double *x0, const double *y0, const double *s0, double *x, double *y,
                          double *s, int32_t *status, int32_t *iters, const orc_settings *st, int32_t nthreads);

/* Adjoint of the solution map at (x,y,s): given dx,dy (ds = 0, as the reference
 * always passes, diffcp_if.py:84) produce dA (all nnzA structural entries),
 * dP (nnzP upper-tri entries, may be NULL), db, dc. Returns LSQR iterations. */
int orc_vjp(const orc_desc *d, const double *Av, const double *Pv, const double *b,
            const double *c, const double *x, const double *y, const double *s,
            const double *dx, const double *dy, double *dAv, double *dPv, double *db,
            double *dc, const orc_settings *st);

/* Batch drivers: instance-contiguous ("batch-major") arrays [B, .]; one OpenMP
 * task per instance -- mirrors diffcp's ThreadPool over instances. */
void orc_solve_batch(const orc_desc *d, int32_t B, const double *Av, const double *Pv,
                     const double *b, const double *c, double *x, double *y, double *s,
                     int32_t *status, int32_t *iters, const orc_settings *st, int32_t nthreads);
void orc_vjp_batch(const orc_desc *d, int32_t B, const double *Av, const double *Pv,
                   const double *b, const double *c, const double *x, const double *y,
                   const double *s, const double *dx, const double *dy, double *dAv,
                   double *dPv, double *db, double *dc, int32_t *lsqr_iters,
                   const orc_settings *st, int32_t nthreads);

/* Building blocks exposed for unit tests. */
void orc_proj_dual_cone(const orc_desc *d, double *v);                 /* v <- Pi_{K*}(v) */
void orc_dproj_dual_cone(const orc_desc *d, const double *v, const double *dv, double *out);
int orc_lsqr_dense(int32_t rows, int32_t cols, const double *Mrow, const double *rhs,
                   double *sol, double atol, double btol, double conlim, int32_t iter_lim);
int orc_max_threads(void);

#ifdef __cplusplus
}
#endif
#endif
