/*
 * bcone.h -- C ABI of the H100-native batched cone-program solve-and-differentiate
 * engine (libbcone.so).  Plain pointers and sizes only; every data pointer is the
 * CALLER'S DEVICE MEMORY unless stated, every call is asynchronous on the given
 * CUDA stream, every function returns 0 on success and a negative code on error
 * (message via bcone_last_error); nothing throws across this boundary.
 *
 * What each entry point replaces in the reference (cvxpy/cvxpylayers @ f0b1c15):
 *   bcone_create   <- DIFFCP_ctx.__init__            src/cvxpylayers/interfaces/diffcp_if.py:105-120
 *                     (captures the sparsity structure + cone dims once per layer;
 *                      CSR twin: MOREAU_ctx.__init__ moreau_if.py:181-222)
 *   bcone_ingest   <- _build_diffcp_matrices         diffcp_if.py:46-70   (per-instance Python loop
 *                     turning the [nnz,B] boundary tensors into solver data A=-A_cvx, b, c)
 *   bcone_solve    <- diffcp.solve_and_derivative_batch / solve_only_batch
 *                                                    diffcp_if.py:365, :369 (SCS forward solve)
 *   bcone_vjp      <- the adjoint closure adj_batch  diffcp_if.py:86      (diffcp adjoint_derivative)
 *   bcone_jvp      <- diffcp's forward derivative D  (second output of solve_and_derivative; the reference never calls it)
 *   bcone_emit     <- _compute_gradients re-packing  diffcp_if.py:88-94 + stacks :396-397
 *                     (dA_eval = [-dA ; db[b_idx]], dq_eval = [dc ; 0])
 *
 * Solver form (SCS / diffcp convention):  min 1/2 x'Px + c'x  s.t.  Ax + s = b, s in K,
 * dual y in K*.  K = zero(z) x nonneg(l) x SOC(q[0..nq)) x PSD(s[0..ns)) x exp(ep) x exp*(ed) in that
 * row order (exp triples (x,y,z): y e^{x/y} <= z).
 * All floating point data is fp64.
 */
#ifndef BCONE_H
#define BCONE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int32_t n, m, nnzA, nnzP;
  const int32_t *A_indptr, *A_indices; /* HOST pointers, CSR of A (m+1 / nnzA); copied        */
  const int32_t *P_indptr, *P_indices; /* HOST pointers, CSR upper triangle of P, or NULL     */
  int32_t z, l, nq, ns, ep, ed;        /* cone spec in SCS row order z, l, q, s, ep, ed        */
  const int32_t *q, *s;                /* HOST: SOC sizes [nq], PSD orders [ns]               */
  int32_t device;                      /* CUDA device ordinal                                 */
  int32_t max_batch;                   /* workspace is sized for this many instances          */
} bcone_desc;

typedef struct {
  double eps_abs, eps_rel, eps_infeas; /* SCS termination (defaults 1e-4, 1e-4, 1e-7)         */
  double alpha, rho_x, scale;          /* over-relaxation 1.5, 1e-6, 0.1                      */
  double lsqr_atol, lsqr_btol, lsqr_conlim; /* 1e-8, 1e-8, 1e8 (diffcp / SciPy LSQR rules)    */
  int32_t max_iters, normalize, adaptive_scale, check_interval;
  int32_t ruiz_passes, lsqr_iter_lim;  /* lsqr_iter_lim < 0 -> 2N like diffcp                 */
  int32_t lsqr_precond;                /* 0 plain LSQR (reference semantics), 1 diagonally equilibrated,
                                          2 KKT-block preconditioned where applicable (else 1) */
  int32_t adaptive_check;              /* 0: test termination every check_interval iterations (SCS);
                                          1: place the checks by log-linear extrapolation (<= check_interval apart) */
  int32_t acceleration_lookback;       /* SCS: Anderson acceleration window; 10 (type-I), < 0 type-II, 0 off
                                          (what the reference's tests pass, tests/test_torch.py:401-405); |.| <= 16 */
  int32_t acceleration_interval;       /* SCS: accelerate every this many iterations (10)                    */
} bcone_settings;

enum { BCONE_SOLVED = 1, BCONE_INACCURATE = 2, BCONE_UNBOUNDED = -1, BCONE_INFEASIBLE = -2, BCONE_FAILED = -4 };
enum { BCONE_OK = 0, BCONE_EINVAL = -1, BCONE_ECUDA = -2, BCONE_ENOMEM = -3, BCONE_EUNSUPPORTED = -4 };

void bcone_default_settings(bcone_settings *st);

/* Uploads the structure and picks the kernels (bcone_path_info).  The generic kernels keep an instance's CSR values in shared
 * memory; when they do not fit next to the rest of a CTA's working set, the values stay in global memory (L2 when the grid's
 * working set fits, HBM otherwise): the forward copies each instance's values into a per-CTA slab, the adjoint and the forward
 * mode read them in place from A_vals.  That tier is tried only after every on-chip option has failed;
 * BCONE_VALUES_GLOBAL=1 in the environment selects it for every generic kernel of a structure that would fit on chip (a test
 * hook).  BCONE_EUNSUPPORTED: even then the on-chip scratch (per-warp PSD scratch and persistent eigenvectors, exp-cone slots,
 * 8 n column partials) does not fit; the message names the largest PSD order that would have fit. */
int bcone_create(const bcone_desc *desc, void **handle);
void bcone_destroy(void *handle);
const char *bcone_last_error(void *handle); /* handle may be NULL: last create() error */

/* Boundary layout -> engine layout.  A_eval[nnz_aug, B], q_eval[n+1, B], P_eval[nnzP, B] are the
 * reference's batch-contiguous value matrices; gather[k] (HOST int32 [nnzA], given once at
 * bcone_set_boundary) is the row of A_eval feeding CSR slot k.  Outputs: A_vals[B,nnzA] = -A_eval,
 * b[B,m] (zeros off b_idx), c[B,n], P_vals[B,nnzP]. */
int bcone_set_boundary(void *handle, int32_t nnz_aug, const int32_t *gather, int32_t nb, const int32_t *b_idx);
/* Optional: P_eval[nnzP_boundary, B] rows in the reference's order for ANY symmetric pattern cvxpy emits (upper, lower or
 * full); gatherP[k] (HOST int32 [nnzP]) is the row feeding the engine's upper-triangular CSR slot k.  Rows that feed no
 * slot (the mirror entries of a full pattern) receive a zero gradient in bcone_emit.  Default: identity. */
int bcone_set_boundary_quad(void *handle, int32_t nnzP_boundary, const int32_t *gatherP);
int bcone_ingest(void *handle, int32_t B, const double *A_eval, const double *q_eval, const double *P_eval,
                 double *A_vals, double *P_vals, double *b, double *c, void *cuda_stream);
/* Engine gradients -> boundary layout: dA_eval[nnz_aug,B] = [-dA (boundary order) ; db[b_idx]],
 * dq_eval[n+1,B] = [dc ; 0], dP_eval[nnzP,B]. */
int bcone_emit(void *handle, int32_t B, const double *dA_vals, const double *dP_vals, const double *db,
               const double *dc, double *dA_eval, double *dq_eval, double *dP_eval, void *cuda_stream);

/* Same as bcone_ingest / bcone_emit on a COLUMN SLICE of the boundary tensors: the pointers address column lo of tensors whose
 * rows are ldb doubles apart (ldb = the full batch), B = hi - lo instances.  A sharded or pipelined caller reads its slice of
 * A_eval in place and writes its slice of dA_eval straight into the full gradient tensor (no staging copy, no concatenation). */
int bcone_ingest_pitched(void *handle, int32_t B, int64_t ldb, const double *A_eval, const double *q_eval, const double *P_eval,
                         double *A_vals, double *P_vals, double *b, double *c, void *cuda_stream);
int bcone_emit_pitched(void *handle, int32_t B, int64_t ldb, const double *dA_vals, const double *dP_vals, const double *db,
                       const double *dc, double *dA_eval, double *dq_eval, double *dP_eval, void *cuda_stream);

/* Peer exchange for a batch sharded over the GPUs of one node (SURVEY.md 8e: one exchange of solutions + gradients).  The
 * rank that owns the autograd graph allocates the destination with bcone_peer_alloc and passes the 64-byte CUDA IPC handle
 * to the other ranks (any host channel: torch.distributed, MPI, a pipe); they map it with bcone_peer_open and push their
 * shard with bcone_copy2d_async -- peer-to-peer over NVLink on the copy engines, chunk by chunk behind the solve, so the
 * transfer takes no SM and hides behind the next chunk's kernels.  bcone_copy2d_async also serves local strided copies. */
int bcone_peer_alloc(int32_t device, int64_t bytes, void **ptr, void *ipc_handle64);
int bcone_peer_open(int32_t device, const void *ipc_handle64, void **ptr);
int bcone_peer_close(void *ptr);
int bcone_peer_free(void *ptr);
int bcone_copy2d_async(void *dst, int64_t dpitch, const void *src, int64_t spitch, int64_t width, int64_t height, void *cuda_stream);

/* Parameter -> matrix affine map fused into the load stage (replaces the reference's sparse x dense products around
 * the solver interface: forward  A_eval = A_param @ p_stack etc. at src/cvxpylayers/torch/cvxpylayer.py:443-451,
 * transposes at :33-37).  The three maps are HOST CSR matrices [rows x P1] (P1 = total parameter size + 1; the last row
 * of p_stack is the constant 1, torch/cvxpylayer.py:84-141), rows in BOUNDARY order: A map nnz_aug rows ([A_cvx values ; b
 * entries], exactly the rows of A_eval), q map n + 1 rows, P map nnzP rows or NULL.  Call after bcone_set_boundary.
 * bcone_ingest_params: p_stack[P1, B] (device, batch axis contiguous) -> A_vals[B,nnzA] = -A_eval, b, c, P_vals without
 *   materialising A_eval.  bcone_emit_params: engine gradients -> dp_stack[P1, B] = (the three maps)' applied to
 *   [-dA ; db[b_idx]], [dc ; 0], dP; the row of the constant is left 0.  Only parameters and parameter gradients have
 *   to cross PCIe (or NVLink, for a sharded batch) on this path. */
int bcone_set_param_maps(void *handle, int32_t P1, const int32_t *A_ptr, const int32_t *A_col, const double *A_val,
                         const int32_t *q_ptr, const int32_t *q_col, const double *q_val,
                         const int32_t *P_ptr, const int32_t *P_col, const double *P_val);
int bcone_ingest_params(void *handle, int32_t B, const double *p_stack, double *A_vals, double *P_vals, double *b,
                        double *c, void *cuda_stream);
int bcone_emit_params(void *handle, int32_t B, const double *dA_vals, const double *dP_vals, const double *db,
                      const double *dc, double *dp_stack, void *cuda_stream);

/* Layer prologue / epilogue on the device (SURVEY.md 8f.3): what the reference does per call with expand / permute / reshape /
 * cat / transpose chains (_flatten_and_batch_params, src/cvxpylayers/torch/cvxpylayer.py:84-141) and with slices, Fortran
 * reshapes and a symmetric scatter (_recover_results, :225-282) are index maps, one launch each.  DEVICE pointers throughout
 * (maps int32, scales fp64), no handle.  op: 0 identity, 1 exp (GP variables), 2 log (GP parameters).
 *   rows_from_param: rows[k, b] = f(param[b * stride + map[k]]), k < K -- the K rows of p_stack[.., B] that one parameter owns
 *                    (stride 0 broadcasts an unbatched parameter; map = Fortran-order flattening, NULL = identity)
 *   param_from_rows: the adjoint (batch-sum for stride 0, x 1/p for log); gparam must be zeroed by the caller when stride = 0
 *   gather_cols    : out[b, k] = f(scale[k] * in[b * ld + map[k]]) -- one requested variable out of primal[B, n] / dual[B, m]
 *   scatter_cols   : the adjoint, accumulated into gin (zeroed by the caller) */
int bcone_rows_from_param(const double *param, int64_t stride, const int32_t *map, int32_t K, int32_t B, int32_t op, double *rows,
                          void *cuda_stream);
int bcone_param_from_rows(const double *grows, const double *param, int64_t stride, const int32_t *map, int32_t K, int32_t B,
                          int32_t op, double *gparam, void *cuda_stream);
int bcone_gather_cols(const double *in, int64_t ld, const int32_t *map, const double *scale, int32_t K, int32_t B, int32_t op,
                      double *out, void *cuda_stream);
int bcone_scatter_cols(const double *gout, const double *out, int64_t ld, const int32_t *map, const double *scale, int32_t K,
                       int32_t B, int32_t op, double *gin, void *cuda_stream);

/* Forward: instance-contiguous inputs A_vals[B,nnzA] (CSR order), P_vals[B,nnzP] or NULL, b[B,m], c[B,n];
 * outputs x[B,n], y[B,m], s[B,m], status[B], iters[B] (int32), resid[B,3] or NULL. */
int bcone_solve(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b,
                const double *c, double *x, double *y, double *s, int32_t *status, int32_t *iters,
                double *resid, const bcone_settings *st, void *cuda_stream);

/* Warm-started forward (SURVEY.md 8f.2; the reference has the API for one backend only, torch/cvxpylayer.py:464-487,
 * interfaces/moreau_if.py:237-256): x0[B,n], y0[B,m], s0[B,m] = a solution of a nearby problem (typically the previous call of
 * a training loop); the operator splitting starts at the fixed point that solution would be.  All three NULL = bcone_solve. */
int bcone_solve_warm(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                     const double *x0, const double *y0, const double *s0, double *x, double *y, double *s,
                     int32_t *status, int32_t *iters, double *resid, const bcone_settings *st, void *cuda_stream);

/* Forward with a cached set-up (SURVEY.md 8f.2, second half; the reference's template is the one-time `setup()` of
 * interfaces/moreau_if.py:237-256, `PA_is_constant`): the equilibration (D, E) and the factorisation (K^-1 at its final scale)
 * of every instance are kept in `cache` -- caller-owned device memory of bcone_cache_bytes(handle, B) bytes, 16-byte aligned.
 *   reuse = 0: solve as bcone_solve_warm and write the set-up;
 *   reuse = 1: the caller states that A_vals and P_vals are the ones of the call that wrote `cache` (same B, same order; b and c
 *              are free to change): the kernel skips the Ruiz passes, the formation of K, its Cholesky factorisation and
 *              inverse, and starts at the cached scale.  A record that was never completed (or was written with another
 *              rho_x) is rebuilt in place, so reuse = 1 on a fresh zero-filled buffer is safe.
 * An adaptive re-scaling inside a solve re-factorises as usual and refreshes the record.  Only the register-tiled dense kernel
 * (dense A, zero + nonneg rows, direct mode) has this path: bcone_cache_bytes returns 0 for every other structure, and
 * bcone_solve_cached then requires cache = NULL (it is bcone_solve_warm). */
size_t bcone_cache_bytes(void *handle, int32_t B);
int bcone_solve_cached(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                       const double *x0, const double *y0, const double *s0, double *x, double *y, double *s,
                       int32_t *status, int32_t *iters, double *resid, void *cache, int32_t reuse,
                       const bcone_settings *st, void *cuda_stream);

/* Backward (stateless): adjoint of the solution map at (x,y,s) applied to (dx,dy), ds = 0.
 * Outputs dA_vals[B,nnzA] (every structural entry), dP_vals[B,nnzP] or NULL, db[B,m], dc[B,n],
 * lsqr_iters[B] or NULL. */
int bcone_vjp(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b,
              const double *c, const double *x, const double *y, const double *s, const double *dx,
              const double *dy, double *dA_vals, double *dP_vals, double *db, double *dc,
              int32_t *lsqr_iters, const bcone_settings *st, void *cuda_stream);

/* Forward mode (stateless): derivative of the solution map at (x,y,s) applied to tangents of the data -- diffcp's
 * solve_and_derivative `D` (the reference's backend returns it next to the adjoint `DT` that bcone_vjp provides).  Exactly the
 * transpose of bcone_vjp: <(dx,dy), bcone_jvp(dA,dP,db,dc)> = <bcone_vjp(dx,dy), (dA,dP,db,dc)>.  Tangents in engine layout:
 * dA_vals[B,nnzA], dP_vals[B,nnzP] (upper-triangular values, an off-diagonal one perturbs P_ij and P_ji) or NULL = 0, db[B,m],
 * dc[B,n].  Outputs dx[B,n], dy[B,m], ds[B,m] or NULL, lsqr_iters[B] or NULL (0 where the tangent is zero).  Boundary-layout
 * tangents go through bcone_ingest / bcone_ingest_params first (both are linear; a tangent's constant row is 0).  Always the
 * generic LSQR kernel; lsqr_precond = 2 runs as 1.  BCONE_EUNSUPPORTED when the instance does not fit that kernel. */
int bcone_jvp(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
              const double *x, const double *y, const double *s, const double *dA_vals, const double *dP_vals,
              const double *db, const double *dc, double *dx, double *dy, double *ds, int32_t *lsqr_iters,
              const bcone_settings *st, void *cuda_stream);

/* Batch-shared matrices (OptNet-style layers: A and P are learned weights, every instance brings its own b and c).  The
 * replicated entry points above take A_vals[B,nnzA] / P_vals[B,nnzP] and return dA[B,nnzA] / dP[B,nnzP], which a layer then
 * sums over the batch; these take ONE copy of the values and return the batch sums, with the same kernels reading the one copy
 * (batch stride 0; it stays in L2).  Every structure bcone_create accepts works on them.  Results equal the replicated entry
 * points' on A_vals.expand(B, nnzA): bit for bit where the solve builds K without atomics, up to their launch-to-launch
 * variation where it does (generic direct forward with SOC / PSD / exp cones or CSR A).
 *   bcone_solve_shared: A_vals[nnzA], P_vals[nnzP] or NULL, b[B,m], c[B,n], x0 / y0 / s0 as bcone_solve_warm (all NULL = cold),
 *     outputs as bcone_solve.  On the register-tiled kernel (bcone_path_info fwd 2) the batch also shares ONE set-up: a one-CTA
 *     launch equilibrates A and P and factorises K at the initial scale into a record the handle keeps per stream, and every
 *     instance starts from it (as bcone_solve_cached with reuse = 1).  An instance whose adaptive scale changes
 *     re-factorises privately.
 *   bcone_vjp_shared: as bcone_vjp, with A_vals[nnzA], P_vals[nnzP]; dA_sum[nnzA] and dP_sum[nnzP] (or NULL) receive
 *     sum_b of what bcone_vjp returns for instance b; db[B,m], dc[B,n], lsqr_iters[B] stay per instance.  The kernels write
 *     r and pi_y per instance (n + 2m + 1 doubles, scratch kept by the handle per stream) and a two-stage reduction with a
 *     fixed order and no floating-point atomics forms the sums: two calls give identical bits.
 *   bcone_jvp_shared: as bcone_jvp, with A_vals[nnzA], P_vals[nnzP] and the shared tangents dA[nnzA], dP[nnzP] or NULL;
 *     db[B,m], dc[B,n] and the outputs per instance.
 *   bcone_ingest_params_shared: as bcone_ingest_params, but A_vals[nnzA] / P_vals[nnzP] are evaluated from column 0 of
 *     p_stack[P1,B] only (the parameters feeding A and P are unbatched); b and c from every column.
 *   bcone_emit_params_shared: as bcone_emit_params from dA_sum[nnzA] / dP_sum[nnzP] (or NULL): their contribution goes into
 *     column 0 of dp_stack[P1,B], that of db / dc into every column.  By linearity the batch sum of dp_stack over the rows of
 *     an unbatched parameter equals that of the replicated path, and that sum is all a layer's backward consumes. */
int bcone_solve_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                       const double *x0, const double *y0, const double *s0, double *x, double *y, double *s,
                       int32_t *status, int32_t *iters, double *resid, const bcone_settings *st, void *cuda_stream);
int bcone_vjp_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b,
                     const double *c, const double *x, const double *y, const double *s, const double *dx,
                     const double *dy, double *dA_sum, double *dP_sum, double *db, double *dc,
                     int32_t *lsqr_iters, const bcone_settings *st, void *cuda_stream);
int bcone_jvp_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                     const double *x, const double *y, const double *s, const double *dA, const double *dP,
                     const double *db, const double *dc, double *dx, double *dy, double *ds, int32_t *lsqr_iters,
                     const bcone_settings *st, void *cuda_stream);
int bcone_ingest_params_shared(void *handle, int32_t B, const double *p_stack, double *A_vals, double *P_vals, double *b,
                               double *c, void *cuda_stream);
int bcone_emit_params_shared(void *handle, int32_t B, const double *dA_sum, const double *dP_sum, const double *db,
                             const double *dc, double *dp_stack, void *cuda_stream);

/* Pitched host<->device copy on the caller's stream (bytes): moves a batch slice [rows, lo:hi] of a
 * boundary tensor directly between pinned host memory and a contiguous device chunk. */
int bcone_memcpy2d(void *dst, int64_t dpitch, const void *src, int64_t spitch, int64_t width, int64_t height,
                   int32_t to_device, void *cuda_stream);

/* Debug: per-phase cycle counters of the forward / block-backward kernels (see csrc/api.cu). */
int bcone_set_profile(void *handle, int32_t on, uint64_t *out16);

/* Introspection for benchmarks/tests: kernel launches issued by this handle so far, and the
 * launch geometry chosen for the forward / backward kernels. */
int64_t bcone_launch_count(void *handle);
/* instances of the last lsqr_precond = 2 bcone_vjp that fell back from the block factorisation to the equilibrated LSQR
 * (device synchronising; -1 before the first such call) */
int bcone_fallback_count(void *handle, int32_t *out);
int bcone_kernel_info(void *handle, int32_t *fwd_threads, int32_t *fwd_smem, int32_t *fwd_ctas_per_sm,
                      int32_t *bwd_threads, int32_t *bwd_smem, int32_t *bwd_ctas_per_sm);
/* Which kernels the structure selected.  fwd_path: 0 generic on-chip Cholesky (fwd.cu), 1 generic indirect (CG),
 * 2 register-tiled dense/polyhedral (fwd_fast.cu), 3 generic with the values on chip and the Cholesky factor + vectors in a
 * per-CTA slab of global memory (instances between the two; BCONE_FWD_MODE=indirect in the environment forces 1 instead).
 * Values off chip (see bcone_create): 4 values in the slab, Cholesky factor + vectors on chip; 5 values, Cholesky factor and
 * vectors in the slab (n <= 512); 6 values + vectors in the slab, indirect (CG).  bwd_path: 0 generic LSQR (bwd.cu), 1 fused
 * single-pass LSQR (bwd_fast.cu), 2 KKT-block preconditioned (bwd_block.cu, used when lsqr_precond = 2; falls back to 1 per
 * instance), 3 generic LSQR with the values read in place from A_vals (values off chip; bcone_jvp then runs the same way). */
int bcone_path_info(void *handle, int32_t *fwd_path, int32_t *bwd_path);
/* CTAs per SM of the generic forward's and adjoint's 4-CTA/SM build, 0 where the structure has none (more than 256 threads,
 * more than 56 KB of shared memory, or no gain in resident CTAs).  With BCONE_SMALL_CTA=2 every launch of a kernel that has
 * that build takes it. */
int bcone_small_cta_info(void *handle, int32_t *fwd_small_ctas, int32_t *bwd_small_ctas);

#ifdef __cplusplus
}
#endif
#endif
