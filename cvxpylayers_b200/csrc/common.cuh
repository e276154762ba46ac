// common.cuh -- device-side building blocks shared by the forward (fwd.cu) and backward
// (bwd.cu) kernels of the batched cone engine.  sm_90a (H100) only.
//
// Execution model: ONE CTA PER PROBLEM INSTANCE, persistent CTAs pulling instance ids from a
// global atomic counter (iteration counts vary 10x across a batch, a static grid would leave
// SMs idle in the tail).  All per-instance state lives in shared memory for the whole solve;
// HBM is touched once on the way in (TMA bulk copy of the instance's CSR values) and once on
// the way out.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "../../include/bcone.h"

#define BC_TAU_FACTOR 10.0
#define BC_ZERO_CONE_FACTOR 1000.0
#define BC_MIN_SCALE 1e-4
#define BC_MAX_SCALE 1e4
#define BC_RESCALE_MIN_ITERS 100
#define BC_EQ_MIN 1e-4
#define BC_EQ_MAX 1e4

enum { BC_CZERO = 0, BC_CNONNEG = 1, BC_CSOC = 2, BC_CPSD = 3 };

// Structure of the batch, device-resident (built once in bcone_create).
struct DevStruct {
  int n, m, nnzA, nnzP;
  int z, l, nq, ns;
  int ep, ed, exp_start;     // exponential cones: ep primal + ed dual triples starting at row exp_start
  int dense;                 // A pattern is the full m x n rectangle, row-major
  int ncones;                // non-polyhedral cone blocks (SOC + PSD)
  int max_psd;               // largest PSD order
  const int *A_indptr, *A_indices;         // CSR
  const int *At_colptr, *At_rowidx, *At_perm; // CSC view: value k of column j is A_vals[At_perm[k]]
  const int *A_rowof;        // row of each CSR slot [nnzA]
  const int *P_indptr, *P_indices, *P_rowof; // upper-tri CSR (+ row of each slot)
  const int *Pt_colptr, *Pt_rowidx, *Pt_perm; // CSC view of the upper triangle
  int p_dense;               // P pattern is the full upper triangle in row-major order
  const int *cone_type, *cone_start, *cone_size, *cone_order; // [ncones], rows are offsets in y
};

// The settings the kernels read: bcone_settings without its trailing lsmr field, which the host turns into the choice of
// kernel (so the argument blocks below keep their layout, and the LSQR kernels their code).  Field for field the same.
struct bc_settings {
  double eps_abs, eps_rel, eps_infeas, alpha, rho_x, scale, lsqr_atol, lsqr_btol, lsqr_conlim;
  int32_t max_iters, normalize, adaptive_scale, check_interval, ruiz_passes, lsqr_iter_lim, lsqr_precond, adaptive_check;
  int32_t acceleration_lookback, acceleration_interval;
};
static_assert(sizeof(bc_settings) == offsetof(bcone_settings, lsmr) && offsetof(bc_settings, lsqr_conlim) == offsetof(bcone_settings, lsqr_conlim) &&
                  offsetof(bc_settings, acceleration_interval) == offsetof(bcone_settings, acceleration_interval),
              "bc_settings must be bcone_settings up to its lsmr field");
inline bc_settings kernel_settings(const bcone_settings &s) {
  return {s.eps_abs, s.eps_rel, s.eps_infeas, s.alpha, s.rho_x, s.scale, s.lsqr_atol, s.lsqr_btol, s.lsqr_conlim,
          s.max_iters, s.normalize, s.adaptive_scale, s.check_interval, s.ruiz_passes, s.lsqr_iter_lim, s.lsqr_precond, s.adaptive_check,
          s.acceleration_lookback, s.acceleration_interval};
}

// Kernel argument blocks (passed by value as __grid_constant__).
struct FwdArgs {
  DevStruct S;
  int B;
  const double *A_vals, *P_vals, *b, *c;
  double *x, *y, *s;
  int *status, *iters;
  double *resid;
  bc_settings st;
  int *counter;
  int use_tma;
  double *ws;            // INDIRECT mode: per-CTA slab of global memory holding the iterate vectors
  long long ws_stride;   // doubles per CTA
  unsigned long long *prof;  // optional: [16] phase cycle counters (debug, bcone_set_profile)
  double *aa_ws;         // Anderson acceleration: per-CTA slab of global memory (L2-resident), or NULL when off
  long long aa_stride;   // doubles per CTA
  const double *x0, *y0, *s0;   // warm start [B, n] / [B, m] / [B, m] (a previous solution of a nearby problem), or NULL
  // cached set-up (register-tiled kernel only): per instance [8 header | E npad | D mpad | Kinv n x npad], see bc_fwdf_cache_doubles
  double *cache;         // NULL = off
  long long cache_stride;  // doubles per instance
  double *park;          // register-tiled kernel: per-CTA slab (4 x 8 x 512 doubles, L2) where the A tile waits out heavy cold calls
  int cache_reuse;       // 0: write the set-up of this solve; 1: A and P are unchanged since the solve that wrote it -> skip it
  int slab_vectors;      // values-off-chip build (fwd_kernel<.., VG = true>): the vectors (and a direct solve's factor) follow the
                         // values in the slab; 0 = they stay in shared memory
  // batch stride (doubles) of A_vals / P_vals: nnzA / nnzP, or 0 when one copy is shared by the batch (bcone_solve_shared).
  // cache_stride = 0 likewise marks a set-up record shared by the batch: read only, an instance that re-scales re-factorises
  // privately and leaves the record alone (other CTAs are reading it).
  long long sA, sP;
};

struct BwdArgs {
  DevStruct S;
  int B;
  const double *A_vals, *P_vals, *b, *c, *x, *y, *s, *dx, *dy;
  double *dA, *dP, *db, *dc;
  int *lsqr_iters;
  bc_settings st;
  int *counter;
  int use_tma;
  int psd_total;  // sum over PSD blocks of k^2 + k
  int p_in_smem;  // P values staged in shared memory (they fit) instead of read from L2
  const int *inst_list;  // optional: work item k is instance inst_list[k] (fallback pass of the block solver)
  const int *B_dev;      // optional: number of work items read from device memory
  int *fail_list, *fail_count;  // block solver: instances it could not handle, for the fallback pass
  unsigned long long *prof;     // optional: [16] phase cycle counters (debug, bcone_set_profile)
  double *ws;            // large instances: LSQR vectors live in a per-CTA slab of global memory (L2)
  long long ws_stride;
  // forward-mode derivative (bcone_jvp, bwd_kernel<.., .., true>): tangents of the data in (tP may be NULL = 0),
  // tangents of the solution out (ts may be NULL).  Unused by the adjoint kernels.
  const double *tA, *tP, *tb, *tc;
  double *tx, *ty, *ts;
  // batch stride (doubles) of A_vals / P_vals and of the tangents tA / tP: nnzA / nnzP, or 0 = one copy shared by the batch
  long long sA, sP;
  // shared matrices (bcone_vjp_shared): instead of dA / dP, each instance writes r and pi_y here (bc_srec_doubles apart,
  // layout at put_srec) for the batch-summing reduction of shared.cu.  NULL = assemble dA / dP per instance.
  double *srec;
};

// Solution polishing (polish.cu, bcone_polish): x, y, s are read and, for an accepted instance, overwritten in place.
struct PolishArgs {
  DevStruct S;
  int B;
  const double *A_vals, *P_vals, *b, *c;
  double *x, *y, *s;
  const int *status;
  int *polished;         // [B]: 1 accepted, 0 rejected (input kept), -1 not attempted
  double *resid;         // [B,3] or NULL: rp, rd, gap of an accepted instance
  long long sA, sP;      // batch strides of A_vals / P_vals (0: one copy shared by the batch)
  int *counter;
  int use_tma;           // dense A, n even, A_vals 16-byte aligned: live rows staged by TMA bulk copies
  long long stage_cap;   // doubles of the buffer the live rows, W and S share
  double delta;          // regularisation, relative to the largest absolute entry of P and A_L
  int refine;            // iterative refinement steps
};

// Solution polishing, slab tier (polish_large.cu): polishing's arguments (stage_cap and use_tma unused), each CTA's slab of global
// memory and the P layout decided at bcone_create.
struct PolishLargeArgs {
  PolishArgs a;
  double *ws;            // per-CTA slabs, ws_stride doubles apart (bc_polish_large_slab_doubles)
  long long ws_stride;
  int p_diag;            // no P, or only diagonal entries: L_P is the vector sqrt(P_jj + d), W is A_L with its columns scaled
};

// Solution refinement (refine.cu, bcone_refine): the forward-mode kernel's arguments (x, y, s read through a.x / a.y / a.s and, for
// an accepted instance, written through a.tx / a.ty / a.ts: the same arrays) and the refinement's own.
struct RefineArgs {
  BwdArgs a;
  const int *status;
  int *flags;            // [B]: 1 accepted, 0 rejected (input kept), -1 not attempted
  double *resid;         // [B,3] or NULL: rp, rd, gap of an accepted instance
  int steps;             // at most this many Newton steps
};

// Per-instance record of the shared-matrix adjoint: [r_x n | r_y m | r_tau | pi_y m].
__host__ __device__ inline long long bc_srec_doubles(int n, int m) { return (long long)n + 2LL * m + 1; }
// Written by the whole block; rx / ry / piy in shared memory (rx and ry may be one vector X = [r_x ; r_y ; r_tau]).
static __device__ __noinline__ void put_srec(double *rec, const double *rx, const double *ry, double rt, const double *piy, int n, int m) {
  for (int j = threadIdx.x; j < n; j += blockDim.x) rec[j] = rx[j];
  for (int i = threadIdx.x; i < m; i += blockDim.x) { rec[n + i] = ry[i]; rec[n + m + 1 + i] = piy[i]; }
  if (threadIdx.x == 0) rec[n + m] = rt;
}

// Phase timing (debug): thread 0 of every CTA adds the cycles since the previous stamp to prof[phase].
struct PhaseTimer {
  unsigned long long *p; long long t0;
  __device__ __forceinline__ void start(unsigned long long *prof) { p = prof; if (p && threadIdx.x == 0) t0 = clock64(); }
  __device__ __forceinline__ void stamp(int phase) {
    if (p && threadIdx.x == 0) { const long long t1 = clock64(); atomicAdd(p + phase, (unsigned long long)(t1 - t0)); t0 = t1; }
  }
  __device__ __forceinline__ void skip() { if (p && threadIdx.x == 0) t0 = clock64(); }   // restart without charging
};

// ----------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// ----------------------------------------------------------------------------- reductions
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide reduction of K values at once; every thread returns the same bits (fixed order).
// red must hold K * 32 doubles.  Contains two __syncthreads().
template <int K, bool MAX>
__device__ __forceinline__ void block_reduce(double (&v)[K], double *red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int k = 0; k < K; k++) v[k] = MAX ? warp_max(v[k]) : warp_sum(v[k]);
  __syncthreads();  // protects red against readers of a previous reduction
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) red[k * 32 + warp] = v[k];
  }
  __syncthreads();
  // second stage: every warp combines the per-warp partials with the same shuffle tree,
  // so all threads end with identical bits
#pragma unroll
  for (int k = 0; k < K; k++) {
    const double a = lane < nw ? red[k * 32 + lane] : 0.0;
    v[k] = MAX ? warp_max(a) : warp_sum(a);
  }
}

// ----------------------------------------------------------------------------- Anderson acceleration
// Safeguarded Anderson acceleration of the iterate w = (w_x, w_y, w_tau), the device twin of the oracle's
// aa_apply / aa_safeguard (oracle/cone_oracle.c; SCS 3 defaults: acceleration_lookback 10 = type-I,
// negative = type-II, acceleration_interval 10; the reference's tests switch it off with
// {"acceleration_lookback": 0}, tests/test_torch.py:401-405, i.e. it is on by default on that path).
// The window (three mem x N difference matrices + four N-vectors) does not fit next to the instance in shared
// memory, so it lives in a per-CTA slab of global memory that stays in L2 (85 KB per CTA for N = 301); it is
// touched once every `interval` iterations.  The mem x mem normal matrix is kept incrementally (only the row
// and column of the replaced difference pair are recomputed: 3 mem dot products per call instead of mem^2),
// the small solve runs on one warp with one matrix row per lane (partial pivoting through shuffles).
#define BC_AA_MAXMEM 16
#define BC_AA_HDR (8 + BC_AA_MAXMEM * BC_AA_MAXMEM + 3 * BC_AA_MAXMEM)
#define BC_AA_LU (BC_AA_MAXMEM * (BC_AA_MAXMEM + 1))
#define BC_AA_MAX_WEIGHT_NORM 1e10
#define BC_AA_SAFEGUARD_FACTOR 1.0
__host__ __device__ inline size_t aa_ws_doubles(int N, int mem) {
  const size_t Np = ((size_t)N + 1) & ~(size_t)1;
  return BC_AA_HDR + (4 + 3 * (size_t)mem) * Np;
}
struct AaIter {   // where the kernel keeps the iterate
  double *wx; int n; double *wy; int m; double *wtau;
  __device__ __forceinline__ double &at(int e) const { return e < n ? wx[e] : (e < n + m ? wy[e - n] : *wtau); }
};
// header: [0] pairs seen since the last reset, [1] a step was taken and awaits its safeguard, [2] ||g|| of that step,
// [3] the raw history of the fill phase has been turned into difference columns
__device__ __forceinline__ void aa_reset_dev(double *ws) { if (threadIdx.x == 0) { ws[0] = 0.0; ws[1] = 0.0; ws[2] = 0.0; ws[3] = 0.0; } }
// w_prev <- w (tau passed by value: the register-tiled kernel keeps it in a register)
static __device__ __noinline__ void aa_store_prev(double *ws, int mem, const AaIter w, double tau) {
  const int N = w.n + w.m + 1, Np = (N + 1) & ~1;
  double *wprev = ws + BC_AA_HDR + 3 * Np;
  for (int e = threadIdx.x; e < N; e += blockDim.x) wprev[e] = e == N - 1 ? tau : w.at(e);
}
// w (the newest iterate, reached by one step from w_prev) is overwritten with the accelerated point when a
// step is taken.  Block-uniform return value: ||gamma|| (0 nothing done, < 0 step dropped).  Starts and ends
// with a barrier; *w.wtau must have been written before the call (any thread).  sscr: BC_AA_MAXMEM + 1 doubles, lu:
// BC_AA_LU doubles of shared memory the call may use.
static __device__ __noinline__ double aa_apply_dev(double *ws, int lookback, const AaIter w, double *sscr, double *red, double *lu) {
  const int T = blockDim.x, t = threadIdx.x, N = w.n + w.m + 1, Np = (N + 1) & ~1;
  const int mem = lookback > 0 ? lookback : -lookback;
  const bool type1 = lookback > 0;
  double *hdr = ws, *Mm = ws + 8, *yn = Mm + BC_AA_MAXMEM * BC_AA_MAXMEM, *sn = yn + BC_AA_MAXMEM, *work = sn + BC_AA_MAXMEM;
  double *ax = ws + BC_AA_HDR, *af = ax + Np, *gp = af + Np, *wprev = gp + Np, *Y = wprev + Np, *Sm = Y + (size_t)mem * Np, *D = Sm + (size_t)mem * Np;
  __syncthreads();
  const int iter = (int)hdr[0];
  __syncthreads();   // everybody has read the header before thread 0 rewrites it
  if (iter < mem) {
    // Fill phase (SCS fills the memory before the first solve): only the raw pair (x, f) is recorded -- x in column
    // `iter` of S, f in column `iter` of D.  Instances that converge before the window is full (the common case at
    // 1e-4) pay two vector stores per acceleration_interval iterations and nothing else.
    double *Sx = Sm + (size_t)iter * Np, *Df = D + (size_t)iter * Np;
    for (int e = t; e < N; e += T) { Sx[e] = wprev[e]; Df[e] = w.at(e); }
    if (t == 0) { hdr[0] = iter + 1; hdr[1] = 0.0; hdr[3] = 0.0; }
    __syncthreads();
    return 0.0;
  }
  if (hdr[3] == 0.0) {
    // first solve: raw pairs 0 .. mem-1 -> difference columns 0 .. mem-2 (s_k = x_k - x_{k-1}, d_k = f_k - f_{k-1},
    // y_k = g_k - g_{k-1}, g = x - f) and the running (x, f, g) = pair mem-1: exactly what one update per pair would
    // have left behind
    for (int e = t; e < N; e += T) {
      double xp = Sm[e], fp = D[e];
      for (int k = 1; k < mem; k++) {
        const double xk = Sm[(size_t)k * Np + e], fk = D[(size_t)k * Np + e];
        Sm[(size_t)(k - 1) * Np + e] = xk - xp; D[(size_t)(k - 1) * Np + e] = fk - fp; Y[(size_t)(k - 1) * Np + e] = (xk - fk) - (xp - fp);
        xp = xk; fp = fk;
      }
      ax[e] = xp; af[e] = fp; gp[e] = xp - fp;
    }
    __syncthreads();   // (thread 0 sets hdr[3] below, after everybody has read it)
  }
  const int len = mem, idx = (iter - 1) % mem;
  double ng[1] = {0.0};
  {
    double *Yc = Y + (size_t)idx * Np, *Sc = Sm + (size_t)idx * Np, *Dc = D + (size_t)idx * Np;
    for (int e = t; e < N; e += T) {
      const double xe = wprev[e], fe = w.at(e), g = xe - fe;
      Sc[e] = xe - ax[e]; Dc[e] = fe - af[e]; Yc[e] = g - gp[e];
      gp[e] = g; ax[e] = xe; af[e] = fe;
      ng[0] = fma(g, g, ng[0]);
    }
  }
  block_reduce<1, false>(ng, red);   // (its barriers publish the new columns)
  const double norm_g = sqrt(ng[0]);
  {   // Gram entries: everything at the first solve, afterwards only what the new pair touches
    const bool full = iter == mem;
    const double *Lm = type1 ? Sm : Y;
    const int lane = t & 31, warp = t >> 5, nw = T >> 5;
    const int njobs = full ? len * len + 3 * len : 3 * len + 1;
    for (int job = warp; job < njobs; job += nw) {
      const double *pa, *pb; double *dst;
      if (full) {
        if (job < len * len) { const int i = job / len, j = job - i * len; pa = Lm + (size_t)i * Np; pb = Y + (size_t)j * Np; dst = Mm + i * BC_AA_MAXMEM + j; }
        else if (job < len * len + len) { const int c = job - len * len; pa = pb = Y + (size_t)c * Np; dst = yn + c; }
        else if (job < len * len + 2 * len) { const int c = job - len * len - len; pa = pb = Sm + (size_t)c * Np; dst = sn + c; }
        else { const int i = job - len * len - 2 * len; pa = Lm + (size_t)i * Np; pb = gp; dst = work + i; }
      } else {
        if (job < len) { pa = Lm + (size_t)job * Np; pb = Y + (size_t)idx * Np; dst = Mm + job * BC_AA_MAXMEM + idx; }
        else if (job < 2 * len - 1) { int j = job - len; if (j >= idx) j++; pa = Lm + (size_t)idx * Np; pb = Y + (size_t)j * Np; dst = Mm + idx * BC_AA_MAXMEM + j; }
        else if (job == 2 * len - 1) { pa = pb = Y + (size_t)idx * Np; dst = yn + idx; }
        else if (job == 2 * len) { pa = pb = Sm + (size_t)idx * Np; dst = sn + idx; }
        else { const int i = job - 2 * len - 1; pa = Lm + (size_t)i * Np; pb = gp; dst = work + i; }
      }
      double acc = 0.0;
      for (int e = lane; e < N; e += 32) acc = fma(pa[e], pb[e], acc);
      acc = warp_sum(acc);
      if (lane == 0) *dst = acc;
    }
  }
  __syncthreads();
  if (t < 32) {   // (M + r I) gamma = work: Gaussian elimination with partial pivoting, one row per lane, the
                  // matrix in shared memory (lu: BC_AA_MAXMEM x (BC_AA_MAXMEM + 1) doubles): a register-resident copy
                  // would make this function -- and, through the call, the kernels' iteration loops -- register-hungry
    const int lane = t, LD = BC_AA_MAXMEM + 1;
    double nys = 0.0;
    for (int c = 0; c < len; c++) nys += yn[c] + sn[c];
    const double r = (type1 ? 1e-6 : 1e-10) * nys;
    if (lane < len) {
      for (int k = 0; k < len; k++) lu[lane * LD + k] = Mm[lane * BC_AA_MAXMEM + k] + (k == lane ? r : 0.0);
      lu[lane * LD + BC_AA_MAXMEM] = work[lane];
    }
    __syncwarp();
    int myc = -1;
    bool ok = true;
    for (int c = 0; c < len; c++) {
      const double v = (lane < len && myc < 0) ? fabs(lu[lane * LD + c]) : -1.0;
      const double best = warp_max(v);
      const int p = __ffs(__ballot_sync(0xffffffffu, v == best)) - 1;
      if (!(best > 0.0)) ok = false;
      if (lane < len && myc < 0 && lane != p && ok) {
        const double f = lu[lane * LD + c] / lu[p * LD + c];
        for (int k = c; k < len; k++) lu[lane * LD + k] = fma(-f, lu[p * LD + k], lu[lane * LD + k]);
        lu[lane * LD + BC_AA_MAXMEM] = fma(-f, lu[p * LD + BC_AA_MAXMEM], lu[lane * LD + BC_AA_MAXMEM]);
      }
      if (lane == p) myc = c;
      __syncwarp();
    }
    double nrm = 0.0;
    for (int c = len - 1; c >= 0; c--) {   // the lane that pivoted on column c owns unknown c
      if (myc == c) {
        double acc = lu[lane * LD + BC_AA_MAXMEM];
        for (int k = c + 1; k < len; k++) acc = fma(-lu[lane * LD + k], sscr[k], acc);
        sscr[c] = acc / lu[lane * LD + c];
      }
      __syncwarp();
      nrm = fma(sscr[c], sscr[c], nrm);
    }
    nrm = sqrt(nrm);
    if (lane == 0) sscr[BC_AA_MAXMEM] = (ok && nrm < BC_AA_MAX_WEIGHT_NORM) ? nrm : -1.0;
  }
  __syncthreads();
  const double aa_norm = sscr[BC_AA_MAXMEM];
  if (!(aa_norm >= 0.0)) {
    if (t == 0) { hdr[0] = 0.0; hdr[1] = 0.0; hdr[3] = 0.0; }
    __syncthreads();
    return -1.0;
  }
  for (int e = t; e < N; e += T) {
    double v = w.at(e);
    for (int c = 0; c < len; c++) v = fma(-sscr[c], D[(size_t)c * Np + e], v);
    w.at(e) = v;
  }
  if (t == 0) { hdr[0] = iter + 1; hdr[1] = 1.0; hdr[2] = norm_g; hdr[3] = 1.0; }
  __syncthreads();
  return aa_norm;
}
// After one plain step from the accelerated point (w_prev = that point, w = the step's result): reject the
// acceleration if the fixed-point residual grew.  Returns true when w and w_prev were restored.  Barriers inside.
static __device__ __noinline__ bool aa_safeguard_dev(double *ws, int lookback, const AaIter w, double *red) {
  const int T = blockDim.x, t = threadIdx.x, N = w.n + w.m + 1, Np = (N + 1) & ~1;
  double *hdr = ws, *ax = ws + BC_AA_HDR, *af = ax + Np, *wprev = af + 2 * Np;
  __syncthreads();
  const bool success = hdr[1] != 0.0;
  const double norm_g = hdr[2];
  __syncthreads();
  if (!success) return false;
  double nd[1] = {0.0};
  for (int e = t; e < N; e += T) { const double q = wprev[e] - w.at(e); nd[0] = fma(q, q, nd[0]); }
  block_reduce<1, false>(nd, red);
  if (t == 0) hdr[1] = 0.0;
  const bool reject = sqrt(nd[0]) > BC_AA_SAFEGUARD_FACTOR * norm_g;
  if (reject) {
    for (int e = t; e < N; e += T) { w.at(e) = af[e]; wprev[e] = ax[e]; }
    if (t == 0) { hdr[0] = 0.0; hdr[3] = 0.0; }
  }
  __syncthreads();
  return reject;
}

// ----------------------------------------------------------------------------- matrix layouts
// Row-oriented storage: element (i, c) lives at base(i) + c for beg(i) <= c < end(i).
// step(i) = base(i+1) - base(i); column j is present in rows [row_lo(j), row_hi(j, nrows)).
struct DenseLayout {
  static constexpr bool kFullRows = true;
  int ncols;
  __device__ __forceinline__ int base(int i) const { return i * ncols; }
  __device__ __forceinline__ int step(int) const { return ncols; }
  __device__ __forceinline__ int beg(int) const { return 0; }
  __device__ __forceinline__ int end(int) const { return ncols; }
  __device__ __forceinline__ int row_lo(int) const { return 0; }
  __device__ __forceinline__ int row_hi(int, int nrows) const { return nrows; }
};
struct PackedLowerLayout {  // row i holds columns 0..i at i(i+1)/2
  static constexpr bool kFullRows = false;
  __device__ __forceinline__ int base(int i) const { return (i * (i + 1)) >> 1; }
  __device__ __forceinline__ int step(int i) const { return i + 1; }
  __device__ __forceinline__ int beg(int) const { return 0; }
  __device__ __forceinline__ int end(int i) const { return i + 1; }
  __device__ __forceinline__ int row_lo(int j) const { return j; }
  __device__ __forceinline__ int row_hi(int, int nrows) const { return nrows; }
};
struct PackedLowerStrictLayout {  // same storage, diagonal excluded (transposed half of a symmetric product)
  static constexpr bool kFullRows = false;
  __device__ __forceinline__ int base(int i) const { return (i * (i + 1)) >> 1; }
  __device__ __forceinline__ int step(int i) const { return i + 1; }
  __device__ __forceinline__ int beg(int) const { return 0; }
  __device__ __forceinline__ int end(int i) const { return i; }
  __device__ __forceinline__ int row_lo(int j) const { return j + 1; }
  __device__ __forceinline__ int row_hi(int, int nrows) const { return nrows; }
};
// Upper triangle stored row by row (row i holds columns i..n-1): the CSR order of a dense
// upper-triangular pattern.  STRICT drops the diagonal (used for the transposed half of a
// symmetric product so the diagonal is not counted twice).
template <bool STRICT>
struct PackedUpperLayout {
  static constexpr bool kFullRows = false;
  int n;
  __device__ __forceinline__ int base(int i) const { return i * n - ((i * (i + 1)) >> 1); }
  __device__ __forceinline__ int step(int i) const { return n - i - 1; }
  __device__ __forceinline__ int beg(int i) const { return STRICT ? i + 1 : i; }
  __device__ __forceinline__ int end(int) const { return n; }
  __device__ __forceinline__ int row_lo(int) const { return 0; }
  __device__ __forceinline__ int row_hi(int j, int nrows) const { return min(nrows, STRICT ? j : j + 1); }
};

// 4 row sums -> one value per 8-lane group with a halving butterfly (6 double shuffles instead
// of 20).  Returns the total of row ((lane>>4)&1)*2 + ((lane>>3)&1) in every lane of that group.
__device__ __forceinline__ double butterfly4(double a0, double a1, double a2, double a3, int lane) {
  const bool hi = lane & 16;
  double k0 = hi ? a2 : a0, k1 = hi ? a3 : a1;
  const double s0 = hi ? a0 : a2, s1 = hi ? a1 : a3;
  k0 += __shfl_xor_sync(0xffffffffu, s0, 16);
  k1 += __shfl_xor_sync(0xffffffffu, s1, 16);
  const bool hi2 = lane & 8;
  double k = hi2 ? k1 : k0;
  const double s = hi2 ? k0 : k1;
  k += __shfl_xor_sync(0xffffffffu, s, 8);
  k += __shfl_xor_sync(0xffffffffu, k, 4);
  k += __shfl_xor_sync(0xffffffffu, k, 2);
  k += __shfl_xor_sync(0xffffffffu, k, 1);
  return k;
}

// FP64 tensor-core tile product D(8x8) += A(8x4) * B(4x8), one warp (SASS: DMMA.8x8x4).  Fragment layout
// (PTX mma.m8n8k4.f64): lane holds A[lane >> 2][lane & 3], B[lane & 3][lane >> 2] and the two accumulator
// entries D[lane >> 2][2 (lane & 3) + {0, 1}].  wgmma has no f64 kind; this is the Hopper tensor path the
// dense fp64 set-up phases (K formation, Cholesky trailing update, W = L^{-1} A', S = W W') run on.
__device__ __forceinline__ void dmma884(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

__device__ __forceinline__ double c_mul_sub(double c, double x, double s, double y) { return fma(c, x, -(s * y)); }   // c x - s y
__device__ __forceinline__ double c_mul_add(double s, double x, double c, double y) { return fma(s, x, c * y); }      // s x + c y

// out_i = sum_j M[i][j] * x[j]: one warp per row, lanes across columns (conflict-free for any
// row stride), x held in registers (ncols <= 128), four rows reduced together.
// ep(i, value) is called by exactly one lane.
template <bool SQ = false, class Layout, class Epi>
__device__ __forceinline__ void matvec_rows(const double *__restrict__ M, Layout lay, int nrows, int ncols,
                                            const double *x, Epi ep) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (ncols <= 128) {
    double xr[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; xr[k] = c < ncols ? x[c] : 0.0; }
    for (int i0 = warp * 4; i0 < nrows; i0 += nw * 4) {
      int o[4], b[4], e[4];
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int i = i0 + r; const bool ok = i < nrows;
        o[r] = ok ? lay.base(i) : 0; b[r] = ok ? lay.beg(i) : 0; e[r] = ok ? lay.end(i) : 0;
      }
      double a[4] = {0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int c = lane + 32 * k;
#pragma unroll
        for (int r = 0; r < 4; r++)
          if (c >= b[r] && c < e[r]) { const double q = M[o[r] + c]; a[r] = fma(SQ ? q * q : q, xr[k], a[r]); }
      }
      const double k = butterfly4(a[0], a[1], a[2], a[3], lane);
      if ((lane & 7) == 0) {
        const int r = i0 + ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
        if (r < nrows) ep(r, k);
      }
    }
  } else {
    for (int i0 = warp * 4; i0 < nrows; i0 += nw * 4) {
      int o[4], b[4], e[4];
      int lmax = 0, bmin = 1 << 30;
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int i = i0 + r; const bool ok = i < nrows;
        o[r] = ok ? lay.base(i) : 0; b[r] = ok ? lay.beg(i) : 0; e[r] = ok ? lay.end(i) : 0;
        lmax = max(lmax, e[r]); if (ok) bmin = min(bmin, b[r]);
      }
      double a[4] = {0, 0, 0, 0};
      for (int c = (min(bmin, lmax) & ~31) + lane; c < lmax; c += 32) {
        const double xv = x[c];
#pragma unroll
        for (int r = 0; r < 4; r++)
          if (c >= b[r] && c < e[r]) { const double q = M[o[r] + c]; a[r] = fma(SQ ? q * q : q, xv, a[r]); }
      }
      const double k = butterfly4(a[0], a[1], a[2], a[3], lane);
      if ((lane & 7) == 0) {
        const int r = i0 + ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
        if (r < nrows) ep(r, k);
      }
    }
  }
}

// Work split of a transposed product over the block, computed once per kernel (integer
// divisions are expensive): thread -> (column j, row chunk [lo, hi)).
struct ColPlan {
  int j, lo, hi, CH;
  bool active, fits;
};
__device__ __forceinline__ ColPlan make_colplan(int nrows, int ncols) {
  ColPlan p;
  const int T = blockDim.x, t = threadIdx.x;
  p.fits = ncols <= T;
  p.CH = p.fits ? T / ncols : 1;
  p.j = p.fits ? t % ncols : t;
  const int c = p.fits ? t / ncols : 0;
  p.active = p.fits && c < p.CH;
  p.lo = (c * nrows) / p.CH;
  p.hi = ((c + 1) * nrows) / p.CH;
  return p;
}

// out_j = sum_i M[i][j] * y[i] (transposed product).  Thread (j, chunk): lanes across columns
// (coalesced, conflict-free), row range split in chunks, partials combined through `part`
// (needs blockDim.x doubles).  Contains two __syncthreads(); ep(j, value) called once per column.
template <bool SQ = false, class Layout, class Epi>
__device__ __forceinline__ void matvec_cols(const double *__restrict__ M, Layout lay, int nrows, int ncols,
                                            const double *y, double *part, Epi ep, const ColPlan &pl) {
  const int T = blockDim.x, t = threadIdx.x;
  if (pl.fits) {
    if (pl.active) {
      const int j = pl.j;
      int i = max(pl.lo, lay.row_lo(j));
      const int hi = min(pl.hi, lay.row_hi(j, nrows));
      double a0 = 0, a1 = 0;
      if (i < hi) {
        const double *p = M + lay.base(i) + j;
        if (Layout::kFullRows) {
          const int st = lay.step(0);
          for (; i + 3 < hi; i += 4) {
            const double q0 = p[0], q1 = p[st], q2 = p[2 * st], q3 = p[3 * st];
            a0 = fma(SQ ? q0 * q0 : q0, y[i], a0); a1 = fma(SQ ? q1 * q1 : q1, y[i + 1], a1);
            a0 = fma(SQ ? q2 * q2 : q2, y[i + 2], a0); a1 = fma(SQ ? q3 * q3 : q3, y[i + 3], a1);
            p += 4 * st;
          }
          for (; i < hi; i++) { const double q = p[0]; a0 = fma(SQ ? q * q : q, y[i], a0); p += st; }
        } else {
          for (; i + 1 < hi; i += 2) {
            const int s0 = lay.step(i);
            const double q0 = p[0], q1 = p[s0];
            a0 = fma(SQ ? q0 * q0 : q0, y[i], a0); a1 = fma(SQ ? q1 * q1 : q1, y[i + 1], a1);
            p += s0 + lay.step(i + 1);
          }
          if (i < hi) { const double q = p[0]; a0 = fma(SQ ? q * q : q, y[i], a0); }
        }
      }
      part[t] = a0 + a1;
    }
    __syncthreads();
    if (t < ncols) {
      double a = 0;
      for (int cc = 0; cc < pl.CH; cc++) a += part[cc * ncols + t];
      ep(t, a);
    }
    __syncthreads();
  } else {
    for (int j = t; j < ncols; j += T) {
      double a = 0;
      const int hi = lay.row_hi(j, nrows);
      for (int i = lay.row_lo(j); i < hi; i++) { const double q = M[lay.base(i) + j]; a = fma(SQ ? q * q : q, y[i], a); }
      ep(j, a);
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------- wide dense products
// Dense row-major A (n even, n <= 128) read with 128-bit shared-memory loads: lanes own column
// pairs.  rows: out_i = sum_j A_ij x_j (4 rows per butterfly); cols: out_j = sum_i A_ij y_i with the
// rows split in 8 chunks whose partials are combined through `part` (needs 8 n doubles).
template <bool SQ = false, class Epi>
__device__ __forceinline__ void dense_rows2(const double *__restrict__ A, int m, int n, const double *x, Epi ep) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const bool ok0 = 2 * lane < n, ok1 = 2 * lane + 64 < n;
  const double2 x0 = ok0 ? make_double2(x[2 * lane], x[2 * lane + 1]) : make_double2(0.0, 0.0);
  const double2 x1 = ok1 ? make_double2(x[2 * lane + 64], x[2 * lane + 65]) : make_double2(0.0, 0.0);
  for (int i0 = warp * 4; i0 < m; i0 += nw * 4) {
    double a[4] = {0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int i = i0 + r;
      if (i < m) {
        const double2 *p2 = reinterpret_cast<const double2 *>(A + i * n) + lane;
        if (ok0) { double2 q = p2[0]; if (SQ) { q.x *= q.x; q.y *= q.y; } a[r] = fma(q.x, x0.x, a[r]); a[r] = fma(q.y, x0.y, a[r]); }
        if (ok1) { double2 q = p2[32]; if (SQ) { q.x *= q.x; q.y *= q.y; } a[r] = fma(q.x, x1.x, a[r]); a[r] = fma(q.y, x1.y, a[r]); }
      }
    }
    const double tot = butterfly4(a[0], a[1], a[2], a[3], lane);
    if ((lane & 7) == 0) {
      const int i = i0 + ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
      if (i < m) ep(i, tot);
    }
  }
}
template <bool SQ = false, class Epi>
__device__ __forceinline__ void dense_cols2(const double *__restrict__ A, int m, int n, const double *y, double *part, Epi ep) {
  const int T = blockDim.x, t = threadIdx.x, npair = n >> 1;
  const int CH = min(8, T / npair), pr = t % npair, c = t / npair;
  if (c < CH) {
    const int lo = (c * m) / CH, hi = ((c + 1) * m) / CH;
    const double2 *p2 = reinterpret_cast<const double2 *>(A + lo * n) + pr;
    double2 a0 = make_double2(0.0, 0.0), a1 = make_double2(0.0, 0.0);
    int i = lo;
    for (; i + 1 < hi; i += 2) {
      double2 q0 = p2[0], q1 = p2[npair];
      if (SQ) { q0.x *= q0.x; q0.y *= q0.y; q1.x *= q1.x; q1.y *= q1.y; }
      const double y0 = y[i], y1 = y[i + 1];
      a0.x = fma(q0.x, y0, a0.x); a0.y = fma(q0.y, y0, a0.y);
      a1.x = fma(q1.x, y1, a1.x); a1.y = fma(q1.y, y1, a1.y);
      p2 += 2 * npair;
    }
    if (i < hi) { double2 q0 = p2[0]; if (SQ) { q0.x *= q0.x; q0.y *= q0.y; } const double y0 = y[i]; a0.x = fma(q0.x, y0, a0.x); a0.y = fma(q0.y, y0, a0.y); }
    *reinterpret_cast<double2 *>(part + c * n + 2 * pr) = make_double2(a0.x + a1.x, a0.y + a1.y);
  }
  __syncthreads();
  if (t < n) {
    double a = 0;
    for (int cc = 0; cc < CH; cc++) a += part[cc * n + t];
    ep(t, a);
  }
  __syncthreads();
}

// CSR products for arbitrary patterns (index arrays stay in global memory: they are shared by
// every CTA of the grid and sit in L1/L2).  Sub-warp groups of G lanes per row.
template <bool SQ = false, class Epi>
__device__ __forceinline__ void csr_rows(const double *__restrict__ vals, const int *__restrict__ indptr,
                                         const int *__restrict__ indices, int nrows,
                                         const double *x, Epi ep) {
  constexpr int G = 4;
  const int g = threadIdx.x % G, grp = threadIdx.x / G, ngrp = blockDim.x / G;
  for (int base = 0; base < nrows; base += ngrp) {  // block-uniform trip count (full-mask shuffles below)
    const int i = base + grp;
    double a = 0;
    if (i < nrows) {
      const int e = __ldg(indptr + i + 1);
      for (int k = __ldg(indptr + i) + g; k < e; k += G) { const double q = vals[k]; a = fma(SQ ? q * q : q, x[__ldg(indices + k)], a); }
    }
    a += __shfl_xor_sync(0xffffffffu, a, 1);
    a += __shfl_xor_sync(0xffffffffu, a, 2);
    if (g == 0 && i < nrows) ep(i, a);
  }
}
template <bool SQ = false, class Epi>
__device__ __forceinline__ void csr_cols(const double *__restrict__ vals, const int *__restrict__ colptr,
                                         const int *__restrict__ rowidx, const int *__restrict__ perm, int ncols,
                                         const double *y, Epi ep) {
  constexpr int G = 4;
  const int g = threadIdx.x % G, grp = threadIdx.x / G, ngrp = blockDim.x / G;
  for (int base = 0; base < ncols; base += ngrp) {
    const int j = base + grp;
    double a = 0;
    if (j < ncols) {
      const int e = __ldg(colptr + j + 1);
      for (int k = __ldg(colptr + j) + g; k < e; k += G) { const double q = vals[__ldg(perm + k)]; a = fma(SQ ? q * q : q, y[__ldg(rowidx + k)], a); }
    }
    a += __shfl_xor_sync(0xffffffffu, a, 1);
    a += __shfl_xor_sync(0xffffffffu, a, 2);
    if (g == 0 && j < ncols) ep(j, a);
  }
}

// A x  and  A' y  for the instance's (scaled) values in shared memory.
// `wide`: caller guarantees n even, n <= 128, Av 16-byte aligned and (for AT_mul) part >= 8 n doubles.
template <bool DENSE, bool SQ = false, class Epi>
__device__ __forceinline__ void A_mul(const DevStruct &S, const double *Av, const double *x, Epi ep, bool wide = false) {
  if (DENSE && wide) dense_rows2<SQ>(Av, S.m, S.n, x, ep);
  else if (DENSE) matvec_rows<SQ>(Av, DenseLayout{S.n}, S.m, S.n, x, ep);
  else csr_rows<SQ>(Av, S.A_indptr, S.A_indices, S.m, x, ep);
}
// NOTE: ends with a __syncthreads() in the dense case; callers sync themselves in the CSR case.
template <bool DENSE, bool SQ = false, class Epi>
__device__ __forceinline__ void AT_mul(const DevStruct &S, const double *Av, const double *y, double *part, Epi ep, const ColPlan &plA,
                                       bool wide = false) {
  if (DENSE && wide) dense_cols2<SQ>(Av, S.m, S.n, y, part, ep);
  else if (DENSE) matvec_cols<SQ>(Av, DenseLayout{S.n}, S.m, S.n, y, part, ep, plA);
  else { csr_cols<SQ>(Av, S.At_colptr, S.At_rowidx, S.At_perm, S.n, y, ep); __syncthreads(); }
}

// out[i] += (P x)[i] for symmetric P given by its upper triangle (values Pv in shared or global
// memory): row pass over the upper triangle, then the transposed pass over the strict upper part.
// No atomics: every out[i] has a single writer per pass.  Ends with __syncthreads().
template <bool SQ = false, class Epi>
__device__ __forceinline__ void P_mul(const DevStruct &S, const double *Pv, const double *x, double *part, Epi ep, const ColPlan &plN) {
  const int n = S.n;
  if (S.p_dense) {
    matvec_rows<SQ>(Pv, PackedUpperLayout<false>{n}, n, n, x, ep);
    __syncthreads();
    matvec_cols<SQ>(Pv, PackedUpperLayout<true>{n}, n, n, x, part, ep, plN);
  } else {
    csr_rows<SQ>(Pv, S.P_indptr, S.P_indices, n, x, ep);
    __syncthreads();
    // CSC view of the upper triangle; the diagonal entry (row == col) is skipped here
    constexpr int G = 4;
    const int g = threadIdx.x % G, grp = threadIdx.x / G, ngrp = blockDim.x / G;
    for (int base = 0; base < n; base += ngrp) {
      const int j = base + grp;
      double a = 0;
      if (j < n) {
        const int e = __ldg(S.Pt_colptr + j + 1);
        for (int k = __ldg(S.Pt_colptr + j) + g; k < e; k += G) {
          const int i = __ldg(S.Pt_rowidx + k);
          if (i != j) { const double q = Pv[__ldg(S.Pt_perm + k)]; a = fma(SQ ? q * q : q, x[i], a); }
        }
      }
      a += __shfl_xor_sync(0xffffffffu, a, 1);
      a += __shfl_xor_sync(0xffffffffu, a, 2);
      if (g == 0 && j < n) ep(j, a);
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------- packed Cholesky + inverse
// In-place Cholesky K = L L' of a packed-lower SPD matrix (row i at i(i+1)/2) and in-place inverse X = L^{-1}:
// the factor is applied afterwards as triangular / dense products, which keeps every solve free of sequential
// substitution.  Everything advances EIGHT columns / rows per step and is latency / barrier bound with 16 warps
// (tools/microbench.cu), so the design minimises steps and warp-instructions and overlaps the serial chain:
//   * ONE sweep does both jobs.  Block row s of L is final (left of its diagonal) once panel s-1 is done, so its
//     inverse step X_s = -M_s L_s X_{<s} runs inside factor step s: two barriers per step for both.
//   * The diagonal block s is overwritten by M_s = L_ss^{-1} as soon as it is factored (nothing reads L_ss itself).
//   * Phase A (thread-parallel): store X_{s-1} from the staging rows | panel s (one row per thread) |
//     Z_s = -M_s L_s in place (one column per thread).
//   * Phase B (warp-parallel, tensor cores): warp 0 updates the trailing tile that holds the next diagonal block
//     and factors + inverts that 8 x 8 block right away (two 4 x 4 blocks with a 4 x 4 update between them: 8 dependent
//     rsqrt, the serial chain of the algorithm, one step ahead of everybody else); the other warps share the rank-8
//     trailing update (two DMMA k-steps on one accumulator per 8 x 8 tile) and the inverse step (Z_s X_{<s}: one 8 x 8
//     output tile per warp).  The trailing work shrinks with s while the inverse work grows.
//   * X_s cannot overwrite Z_s while other warps still read it, so its tiles wait for the next phase A: the first tile of
//     each warp in that warp's registers, the rest (n > 8 x the phase-B warps) in staging rows.
// tmp: scratch of chol_scratch_doubles(n, blockDim.x) doubles (staging rows + the pd flag).  Block-uniform result (false:
// not positive definite).
__host__ __device__ __forceinline__ int chol_held_cols(int threads) { return 8 * (threads > 32 ? (threads >> 5) - 1 : 1); }
__host__ __device__ __forceinline__ int chol_scratch_doubles(int n, int threads) {
  const int ld = 8 * ((n + 7) >> 3) - chol_held_cols(threads);
  return 8 * (ld > 0 ? ld : 0) + 2;
}
// 1 / sqrt(x) for the Cholesky pivots: hardware approximation (2^-23) + two Newton steps (full double precision up to
// a couple of ulp); roughly half the dependent latency of the library rsqrt, and eight of them are chained per block.
__device__ __forceinline__ double rsqrt_nr(double x) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  double e = fma(-x * y, y, 1.0);
  y = fma(0.5 * y, e, y);
  e = fma(-x * y, y, 1.0);
  return fma(0.5 * y, e, y);
}
struct Tri4 { double l00, l10, l11, l20, l21, l22, l30, l31, l32, l33, m00, m10, m11, m20, m21, m22, m30, m31, m32, m33; bool pd; };
// Cholesky factor (l) and its inverse (m) of the jb x jb (jb <= 4) diagonal block at (r0, r0).
// Missing rows / columns are padded with the identity.
__device__ __forceinline__ Tri4 tri4_block(const double *K, int r0, int jb) {
  Tri4 q;
  const double *R0 = K + ((r0 * (r0 + 1)) >> 1) + r0;
  const double *R1 = K + (((r0 + 1) * (r0 + 2)) >> 1) + r0, *R2 = K + (((r0 + 2) * (r0 + 3)) >> 1) + r0, *R3 = K + (((r0 + 3) * (r0 + 4)) >> 1) + r0;
  const double d00 = R0[0];
  const double d10 = jb > 1 ? R1[0] : 0.0, d11 = jb > 1 ? R1[1] : 1.0;
  const double d20 = jb > 2 ? R2[0] : 0.0, d21 = jb > 2 ? R2[1] : 0.0, d22 = jb > 2 ? R2[2] : 1.0;
  const double d30 = jb > 3 ? R3[0] : 0.0, d31 = jb > 3 ? R3[1] : 0.0, d32 = jb > 3 ? R3[2] : 0.0, d33 = jb > 3 ? R3[3] : 1.0;
  const double p0 = d00, r0_ = rsqrt_nr(p0);
  q.l00 = p0 * r0_; q.l10 = d10 * r0_; q.l20 = d20 * r0_; q.l30 = d30 * r0_;
  const double p1 = fma(-q.l10, q.l10, d11), r1_ = rsqrt_nr(p1);
  q.l11 = p1 * r1_; q.l21 = fma(-q.l20, q.l10, d21) * r1_; q.l31 = fma(-q.l30, q.l10, d31) * r1_;
  const double p2 = fma(-q.l21, q.l21, fma(-q.l20, q.l20, d22)), r2_ = rsqrt_nr(p2);
  q.l22 = p2 * r2_; q.l32 = fma(-q.l31, q.l21, fma(-q.l30, q.l20, d32)) * r2_;
  const double p3 = fma(-q.l32, q.l32, fma(-q.l31, q.l31, fma(-q.l30, q.l30, d33))), r3_ = rsqrt_nr(p3);
  q.l33 = p3 * r3_;
  q.pd = (p0 > 0) && (p1 > 0) && (p2 > 0) && (p3 > 0);
  q.m00 = r0_; q.m11 = r1_; q.m22 = r2_; q.m33 = r3_;
  q.m10 = -q.l10 * q.m00 * r1_;
  q.m20 = -fma(q.l21, q.m10, q.l20 * q.m00) * r2_; q.m21 = -q.l21 * q.m11 * r2_;
  q.m30 = -fma(q.l32, q.m20, fma(q.l31, q.m10, q.l30 * q.m00)) * r3_;
  q.m31 = -fma(q.l32, q.m21, q.l31 * q.m11) * r3_; q.m32 = -q.l32 * q.m22 * r3_;
  return q;
}
#ifdef BC_CHOLPROF   // sub-phase cycle counters for tools/microbench.cu (thread 0, slots 17..20 of prof)
#define CP_STAMP(k) if (prof && t == 0) { const long long now_ = clock64(); atomicAdd(prof + (k), (unsigned long long)(now_ - tt)); tt = now_; }
#else
#define CP_STAMP(k)
#endif
static __device__ __noinline__ bool chol_inv_packed(double *K, int n, double *tmp, unsigned long long *prof = nullptr) {
  const int T = blockDim.x, t = threadIdx.x, lane = t & 31, warp = t >> 5, nw = T >> 5;
  // inverse-step output columns [0, held) stay in registers (h0, h1: tile w0 of the warp, row fr, columns 8 w0 + 2 fc, + 1),
  // the others wait in the staging rows
  const int W = nw > 1 ? nw - 1 : 1, w0 = nw > 1 ? warp - 1 : 0, held = chol_held_cols(T);
  const int lds = max(0, 8 * ((n + 7) >> 3) - held);
  // scratch: staging rows of the inverse step | pd flag
  double *Tst = tmp, *flag = tmp + 8 * lds;
  double h0 = 0.0, h1 = 0.0;
  long long t0 = 0;
  if (prof && t == 0) t0 = clock64();
#ifdef BC_CHOLPROF
  long long tt = t0;
#endif
  const int fr = lane >> 2, fc = lane & 3;
  auto rowp = [&](int i) { return K + ((i * (i + 1)) >> 1); };
  // M (lane 0) over the jb x jb (jb <= 4) diagonal block at r0
  auto put_m = [&](int r0, int jb, const Tri4 &q) {
    double *D0 = rowp(r0) + r0;
    D0[0] = q.m00;
    if (jb > 1) { double *D1 = rowp(r0 + 1) + r0; D1[0] = q.m10; D1[1] = q.m11; }
    if (jb > 2) { double *D2 = rowp(r0 + 2) + r0; D2[0] = q.m20; D2[1] = q.m21; D2[2] = q.m22; }
    if (jb > 3) { double *D3 = rowp(r0 + 3) + r0; D3[0] = q.m30; D3[1] = q.m31; D3[2] = q.m32; D3[3] = q.m33; }
  };
  // Diagonal block at J0 (warp 0), replaced in place by its inverse M = L_D^{-1}:  L_D = [L11 0; L21 L22] with
  // L11 L11' = D11, L21 = D21 M11', L22 L22' = D22 - L21 L21', and M21 = -M22 L21 M11.  The 4 x 4 blocks are factored by
  // every lane (tri4_block); the 4 x 4 products take one entry (r, c) per lane of the first half-warp and meet in place.
  auto diag_block = [&](int J0) {
    const int jb = min(8, n - J0), jb2 = jb - 4;
    const Tri4 a = tri4_block(K, J0, min(4, jb));
    bool pd = a.pd;
    __syncwarp();   // every lane has read D11
    if (lane == 0) put_m(J0, min(4, jb), a);
    if (jb2 > 0) {
      const int r = fr, c = fc;
      const bool own = lane < 16 && r < jb2;
      double *Rr = rowp(J0 + 4 + r) + J0;   // row 4 + r of the block
      __syncwarp();   // M11 is in place
      double v = 0.0;
      if (own) {      // L21 = D21 M11'
#pragma unroll
        for (int k = 0; k < 4; k++)
          if (k <= c) v = fma(Rr[k], rowp(J0 + c)[J0 + k], v);
      }
      __syncwarp();   // every lane has read D21
      if (own) Rr[c] = v;
      __syncwarp();
      if (own && c <= r) {   // D22 - L21 L21'
        const double *Rc = rowp(J0 + 4 + c) + J0;
        double g = Rr[4 + c];
#pragma unroll
        for (int k = 0; k < 4; k++) g = fma(-Rr[k], Rc[k], g);
        Rr[4 + c] = g;
      }
      __syncwarp();
      const Tri4 b = tri4_block(K, J0 + 4, jb2);
      pd = pd && b.pd;
      double u = 0.0;   // U = L21 M11
      if (own) {
#pragma unroll
        for (int k = 0; k < 4; k++)
          if (k >= c) u = fma(Rr[k], rowp(J0 + k)[J0 + c], u);
      }
      __syncwarp();   // every lane has read D22 - L21 L21' and L21
      if (lane == 0) put_m(J0 + 4, jb2, b);
      __syncwarp();
      double s = 0.0;   // M21 = -M22 U; U[k][c] is held by lane 4 k + c
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const double uk = __shfl_sync(0xffffffffu, u, 4 * k + c);
        if (own && k <= r) s = fma(Rr[4 + k], uk, s);
      }
      if (own) Rr[c] = -s;
    }
    if (lane == 0 && !pd) *flag = 0.0;
  };
  // One 8 x 8 tile (ta, tb), tb <= ta, of the trailing update K[i][j] -= sum_c L[i][J0+c] L[j][J0+c], i, j >= R0.
  auto trail_tile = [&](int ta, int tb, int J0, int jb, int R0) {
    const int ra = R0 + 8 * ta + fr, rb = R0 + 8 * tb + fr;
    const double *La = rowp(ra) + J0, *Lb = rowp(rb) + J0;
    const double fa0 = (ra < n && fc < jb) ? -La[fc] : 0.0, fa1 = (ra < n && fc + 4 < jb) ? -La[fc + 4] : 0.0;
    const double fb0 = (rb < n && fc < jb) ? Lb[fc] : 0.0, fb1 = (rb < n && fc + 4 < jb) ? Lb[fc + 4] : 0.0;
    const int cc = R0 + 8 * tb + 2 * fc;
    double *pc = rowp(ra) + cc;   // C entries (ra, cc), (ra, cc + 1)
    const bool ok0 = ra < n && cc <= ra, ok1 = ra < n && cc + 1 <= ra;
    double c0 = ok0 ? pc[0] : 0.0, c1 = ok1 ? pc[1] : 0.0;
    dmma884(c0, c1, fa0, fb0);
    dmma884(c0, c1, fa1, fb1);
    if (ok0) pc[0] = c0;
    if (ok1) pc[1] = c1;
  };
  // Inverse step of block row I0 (ib rows, I0 a multiple of 8), output columns [8 jt, 8 jt + 8): (Z X_{<I0})[:, cols]
  // into registers (jt < W: the warp's first tile) or the staging rows.
  auto inv_tile = [&](int jt, int I0, int ib) {
    double c0 = 0.0, c1 = 0.0, d0 = 0.0, d1 = 0.0;
    const bool zr = fr < ib;
    const double *zrow = rowp(I0 + (zr ? fr : 0));
    const int jcol = 8 * jt + fr;
    int k0 = 8 * jt + fc;
    {  // rows [8 jt, 8 jt + 8) of X meet the diagonal: triangular guard
      const double a0 = zr ? zrow[k0] : 0.0, a1 = zr ? zrow[k0 + 4] : 0.0;
      const double b0 = jcol <= k0 ? rowp(k0)[jcol] : 0.0, b1 = jcol <= k0 + 4 ? rowp(k0 + 4)[jcol] : 0.0;
      dmma884(c0, c1, a0, b0);
      dmma884(d0, d1, a1, b1);
      k0 += 8;
    }
    // full rows below: no guards, packed row offsets advanced incrementally, two accumulators in flight
    int o0 = ((k0 * (k0 + 1)) >> 1) + jcol;
    for (; k0 < I0; k0 += 8) {                         // (k0 - fc is a multiple of 8 and so is I0)
      const int o1 = o0 + 4 * k0 + 10;                 // row k0 + 4
      const double a0 = zr ? zrow[k0] : 0.0, a1 = zr ? zrow[k0 + 4] : 0.0;
      const double b0 = K[o0], b1 = K[o1];
      dmma884(c0, c1, a0, b0);
      dmma884(d0, d1, a1, b1);
      o0 += 8 * k0 + 36;                               // row k0 + 8
    }
    if (jt < W) { h0 = c0 + d0; h1 = c1 + d1; }
    else {
      const int col = 8 * jt + 2 * fc - held;
      Tst[fr * lds + col] = c0 + d0; Tst[fr * lds + col + 1] = c1 + d1;   // col + 1 <= 8 jt + 7 - held < lds
    }
  };
  // X rows of block row I0 (left of the diagonal block, which already holds M) from the registers and the staging rows
  auto store_X = [&](int I0) {
    const int ib = min(8, n - I0);
    if ((warp > 0 || nw == 1) && 8 * w0 < I0 && fr < ib) { double *p = rowp(I0 + fr) + 8 * w0 + 2 * fc; p[0] = h0; p[1] = h1; }
    for (int j = held + (t + (T >> 1)) % T; j < I0; j += T) {   // (phase A runs three jobs: each starts on its own warps)
#pragma unroll
      for (int r = 0; r < 8; r++)
        if (r < ib) rowp(I0 + r)[j] = Tst[r * lds + j - held];
    }
  };
  if (warp == 0) {
    if (lane == 0) *flag = 1.0;
    __syncwarp();
    diag_block(0);
  }
  __syncthreads();
  for (int J0 = 0; J0 < n; J0 += 8) {
    const int jb = min(8, n - J0), R0 = J0 + jb;
    if (*flag == 0.0) return false;   // block-uniform: written before the last barrier
    // ---- phase A: X of the previous block row | panel | Z of this block row ----
    if (J0 > 0) store_X(J0 - 8);
    const int tz = (t + T - (T >> 2)) % T;   // Z starts at thread T / 4, the panel at thread 0, the X store at T / 2
    if (R0 + t < n || tz < J0) {
      const double *Md = rowp(J0) + J0;   // M = L_D^{-1}: entry (r, c) at Md[r (r + 1) / 2 + r J0 + c]
      for (int i = R0 + t; i < n; i += T) {   // panel: l_i = a_i L_D^{-T}
        double *row = rowp(i) + J0;
        double a[8];
#pragma unroll
        for (int c = 0; c < 8; c++) a[c] = c < jb ? row[c] : 0.0;
#pragma unroll
        for (int c = 0; c < 8; c++) {
          if (c < jb) {
            const double *Mc = Md + ((c * (c + 1)) >> 1) + c * J0;
            double s = 0.0;
#pragma unroll
            for (int k = 0; k <= c; k++) s = fma(a[k], Mc[k], s);
            row[c] = s;
          }
        }
      }
      for (int i = tz; i < J0; i += T) {      // Z = -M L on block row J0
        double a[8];
#pragma unroll
        for (int r = 0; r < 8; r++) a[r] = r < jb ? rowp(J0 + r)[i] : 0.0;
#pragma unroll
        for (int r = 0; r < 8; r++) {
          if (r < jb) {
            const double *Mr = Md + ((r * (r + 1)) >> 1) + r * J0;
            double s = 0.0;
#pragma unroll
            for (int k = 0; k <= r; k++) s = fma(Mr[k], a[k], s);
            rowp(J0 + r)[i] = -s;
          }
        }
      }
    }
    CP_STAMP(17);
    __syncthreads();
    CP_STAMP(18);
    // ---- phase B: trailing update + next diagonal block | inverse step of this block row ----
    {
      const int ntl = R0 < n ? (n - R0 + 7) >> 3 : 0, ntile = (ntl * (ntl + 1)) >> 1;
      const int ntj = J0 >> 3;                         // inverse tiles (output columns < J0)
      if (warp == 0 && ntile > 0) {
        trail_tile(0, 0, J0, jb, R0);
        __syncwarp();
        diag_block(R0);
      }
      if (warp > 0 || nw == 1) {
        const int nwork = ntj + (ntile > 0 ? ntile - 1 : 0);   // inverse tiles first (longest first), then trailing tiles 1..
        int ta = 0, tb = 0, e_cur = 0;
        for (int u = w0; u < nwork; u += W) {
          if (u < ntj) inv_tile(u, J0, jb);
          else {
            const int e = u - ntj + 1;
            tb += e - e_cur; e_cur = e;
            while (tb > ta) { tb -= ta + 1; ta++; }
            trail_tile(ta, tb, J0, jb, R0);
          }
        }
      }
    }
    CP_STAMP(19);
    __syncthreads();
    CP_STAMP(20);
  }
  if (*flag == 0.0) return false;
  store_X(((n - 1) >> 3) << 3);
  __syncthreads();
  if (prof && t == 0) { const long long t1 = clock64(); atomicAdd(prof + 5, (unsigned long long)(t1 - t0)); }
  return true;
}

// ----------------------------------------------------------------------------- cone projections
// Projection of the non-polyhedral blocks of v (length m, y-space) onto K*; zero rows untouched,
// nonneg rows are handled elementwise by the caller.  One warp per cone block.
// scratch: per-warp workspace of 2*max_psd^2 + max_psd doubles (only touched for PSD blocks).
__device__ void jacobi_eig_warp(int k, double *X, double *V);

__device__ __forceinline__ void project_soc_warp(double *v, int sz) {
  const int lane = threadIdx.x & 31;
  if (sz == 1) { if (lane == 0 && v[0] < 0) v[0] = 0; return; }
  double ss = 0;
  for (int i = 1 + lane; i < sz; i += 32) ss += v[i] * v[i];
  ss = warp_sum(ss);
  const double nx = sqrt(ss), t = v[0];
  __syncwarp();   // every lane holds t before lane 0 may overwrite v[0] in either branch below (with independent thread scheduling a
                  // lane that ran ahead made its neighbours read the NEW v[0] and take a different branch: a rare wrong projection)
  if (nx <= t) return;
  if (nx <= -t) { for (int i = lane; i < sz; i += 32) v[i] = 0; return; }
  const double a = 0.5 * (1.0 + t / nx);
  for (int i = 1 + lane; i < sz; i += 32) v[i] *= a;
  if (lane == 0) v[0] = a * nx;
}

// svec index helpers (lower triangle, column-major, off-diagonals scaled by sqrt2;
// reference layout: src/cvxpylayers/torch/cvxpylayer.py:201-222)
__device__ __forceinline__ void svec_to_mat_warp(int k, const double *v, double *X) {
  const int lane = threadIdx.x & 31;
  const double is2 = 0.70710678118654752440;
  for (int e = lane; e < k * k; e += 32) {
    int i = e / k, j = e % k;
    int r = max(i, j), c = min(i, j);
    int idx = c * k - (c * (c - 1)) / 2 + (r - c);
    X[e] = (i == j) ? v[idx] : v[idx] * is2;
  }
}
__device__ __forceinline__ void mat_to_svec_warp(int k, const double *X, double *v) {
  const int lane = threadIdx.x & 31;
  const double s2 = 1.41421356237309504880;
  for (int e = lane; e < k * k; e += 32) {
    int i = e / k, j = e % k;
    if (i < j) continue;
    int idx = j * k - (j * (j - 1)) / 2 + (i - j);
    v[idx] = (i == j) ? X[i * k + i] : 0.5 * (X[i * k + j] + X[j * k + i]) * s2;
  }
}

// Cyclic Jacobi on a k x k symmetric matrix by one warp (row-major X, eigenvectors in V's columns).
__device__ inline void jacobi_eig_warp(int k, double *X, double *V) {
  const int lane = threadIdx.x & 31;
  for (int e = lane; e < k * k; e += 32) V[e] = (e / k == e % k) ? 1.0 : 0.0;
  __syncwarp();
  for (int sweep = 0; sweep < 30; sweep++) {
    int rotations = 0;   // warp-uniform: every lane reads the same shared-memory words
    for (int p = 0; p < k - 1; p++) for (int q = p + 1; q < k; q++) {
      const double apq = X[p * k + q];
      // skip negligible off-diagonals; the sweep loop ends when a whole sweep rotates nothing
      if (fabs(apq) <= 1e-17 * (fabs(X[p * k + p]) + fabs(X[q * k + q])) || apq == 0.0) continue;
      rotations++;
      const double app = X[p * k + p], aqq = X[q * k + q];
      const double theta = (aqq - app) / (2.0 * apq);
      const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      __syncwarp();
      for (int r = lane; r < k; r += 32) {
        double xp = X[r * k + p], xq = X[r * k + q];
        X[r * k + p] = c * xp - s * xq; X[r * k + q] = s * xp + c * xq;
        double vp = V[r * k + p], vq = V[r * k + q];
        V[r * k + p] = c * vp - s * vq; V[r * k + q] = s * vp + c * vq;
      }
      __syncwarp();
      for (int r = lane; r < k; r += 32) {
        double xp = X[p * k + r], xq = X[q * k + r];
        X[p * k + r] = c * xp - s * xq; X[q * k + r] = s * xp + c * xq;
      }
      __syncwarp();
    }
    if (rotations == 0) break;
  }
  __syncwarp();
}

// C(i, j) = sum_q fa(i, q) fb(q, j), i, j, q < k <= 16, by one warp on the FP64 tensor cores (DMMA.8x8x4): the
// k x k matrices are padded to 8 x 8 output tiles and k-steps of 4 through the accessors (which must return 0
// outside the matrix); st(i, j, value) receives every entry of the padded result once (guard inside).
template <class FA, class FB, class ST>
__device__ __forceinline__ void warp_mm16(int k, FA fa, FB fb, ST st) {
  const int lane = threadIdx.x & 31, fr = lane >> 2, fc = lane & 3;
  const int nt = (k + 7) >> 3, nk = (k + 3) >> 2;
  for (int ti = 0; ti < nt; ti++) {
    double d[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    for (int ks = 0; ks < nk; ks++) {
      const double a = fa(8 * ti + fr, 4 * ks + fc);
#pragma unroll
      for (int tj = 0; tj < 2; tj++) if (tj < nt) dmma884(d[tj][0], d[tj][1], a, fb(4 * ks + fc, 8 * tj + fr));
    }
#pragma unroll
    for (int tj = 0; tj < 2; tj++) if (tj < nt) { st(8 * ti + fr, 8 * tj + 2 * fc, d[tj][0]); st(8 * ti + fr, 8 * tj + 2 * fc + 1, d[tj][1]); }
  }
}

// Parallel-ordered (round-robin) Jacobi on a symmetric k x k matrix T (row-major, shared memory) by one warp:
// every round rotates k/2 DISJOINT pairs at once -- the angles on one lane per pair, then all column updates of T and
// of the accumulated eigenvector matrix V (V <- V J), then all row updates -- three warp barriers per round instead
// of three per rotation.  V is updated, not reset: the caller passes the identity (cold) or the eigenvectors of a
// nearby matrix after transforming T <- V' T V (warm start: one or two sweeps instead of six to eight).
// A sweep that met no |a_pq| above 1e-7 (|a_pp| + |a_qq|) is the last one: quadratic convergence leaves the off-diagonal
// part below 1e-13 of the diagonal after it.  k <= 16.
// 1 / x by the hardware approximation + two Newton steps (a couple of ulp; a third of the latency of the IEEE division).
__device__ __forceinline__ double rcp_nr(double x) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  double e = fma(-x, y, 1.0);
  y = fma(y, e, y);
  e = fma(-x, y, 1.0);
  return fma(y, e, y);
}
__device__ inline void jacobi_par_warp(int k, double *T, double *V) {
  const int lane = threadIdx.x & 31;
  const int kk = (k + 1) & ~1, np = kk >> 1, nr = kk - 1;   // players (a dummy when k is odd), pairs per round, rounds
  // work items of the update phases: (line, pair) for e = lane + 32 trip < k np -- fixed for the whole call
  // (k <= 16: at most four trips); the line is a row of T and V in the column phase, a column of T in the row phase
  constexpr int MAXT = 4;
  int ln[MAXT], pj_[MAXT];
  const int ntrip = (k * np + 31) >> 5;
#pragma unroll
  for (int tr = 0; tr < MAXT; tr++) { const int e = lane + 32 * tr; ln[tr] = e < k * np ? e / np : -1; pj_[tr] = e < k * np ? e - (e / np) * np : 0; }
  auto pair_of = [&](int r, int j, int &p, int &q) {   // circle method: the last player stays, the others rotate
    int a = r + j; if (a >= nr) a -= nr;
    int b = r - j; if (b < 0) b += nr;
    if (j == 0) { a = kk - 1; b = r; }
    p = min(a, b); q = max(a, b);
  };
  for (int sweep = 0; sweep < 30; sweep++) {
    bool big = false;
    for (int r = 0; r < nr; r++) {
      double c = 1.0, s = 0.0;
      if (lane < np) {
        int p, q;
        pair_of(r, lane, p, q);
        if (q < k) {
          const double apq = T[p * k + q], app = T[p * k + p], aqq = T[q * k + q];
          const double lim = fabs(app) + fabs(aqq);
          if (!(fabs(apq) <= 1e-17 * lim) && apq != 0.0) {
            big = big || fabs(apq) > 1e-7 * lim;
            const double theta = (aqq - app) * rcp_nr(2.0 * apq), th2 = fma(theta, theta, 1.0);
            const double t = (theta >= 0 ? 1.0 : -1.0) * rcp_nr(fabs(theta) + th2 * rsqrt_nr(th2));
            c = rsqrt_nr(fma(t, t, 1.0)); s = t * c;
          }
        }
      }
      __syncwarp();   // every angle has been taken from the un-rotated matrix
#pragma unroll
      for (int tr = 0; tr < MAXT; tr++) {   // columns p, q of T and V (warp-uniform trip count: shuffles inside)
        if (tr < ntrip) {
          const double cj = __shfl_sync(0xffffffffu, c, pj_[tr]), sj = __shfl_sync(0xffffffffu, s, pj_[tr]);
          int p, q;
          pair_of(r, pj_[tr], p, q);
          if (ln[tr] >= 0 && q < k && sj != 0.0) {
            const int row = ln[tr];
            const double xp = T[row * k + p], xq = T[row * k + q];
            T[row * k + p] = c_mul_sub(cj, xp, sj, xq); T[row * k + q] = c_mul_add(sj, xp, cj, xq);
            const double vp = V[row * k + p], vq = V[row * k + q];
            V[row * k + p] = c_mul_sub(cj, vp, sj, vq); V[row * k + q] = c_mul_add(sj, vp, cj, vq);
          }
        }
      }
      __syncwarp();
#pragma unroll
      for (int tr = 0; tr < MAXT; tr++) {   // rows p, q of T
        if (tr < ntrip) {
          const double cj = __shfl_sync(0xffffffffu, c, pj_[tr]), sj = __shfl_sync(0xffffffffu, s, pj_[tr]);
          int p, q;
          pair_of(r, pj_[tr], p, q);
          if (ln[tr] >= 0 && q < k && sj != 0.0) {
            const int col = ln[tr];
            const double xp = T[p * k + col], xq = T[q * k + col];
            T[p * k + col] = c_mul_sub(cj, xp, sj, xq); T[q * k + col] = c_mul_add(sj, xp, cj, xq);
          }
        }
      }
      __syncwarp();
    }
    if (!__any_sync(0xffffffffu, big)) break;
  }
}

// v (svec) <- Pi_PSD(v).  scr: 2 k^2 + k doubles of per-warp scratch.  Vp: k^2 doubles that persist across the
// calls of one instance (eigenvectors of the previous iterate) or nullptr; warm = Vp holds them.
// k <= 16: warm start T = Vp' X Vp and the reconstruction V diag(lam+) V' run on the tensor cores (warp_mm16).
__device__ inline void project_psd_warp(double *v, int k, double *scr, double *Vp = nullptr, bool warm = false) {
  const int lane = threadIdx.x & 31;
  double *X = scr, *W = scr + k * k, *lam = W + k * k;
  svec_to_mat_warp(k, v, X);
  __syncwarp();
  if (k > 16 || !Vp) {   // large blocks: the serial cyclic Jacobi (cold every time)
    jacobi_eig_warp(k, X, W);
    for (int i = lane; i < k; i += 32) lam[i] = fmax(X[i * k + i], 0.0);
    __syncwarp();
    for (int e = lane; e < k * k; e += 32) {
      int i = e / k, j = e % k;
      double a = 0;
      for (int q = 0; q < k; q++) a = fma(W[i * k + q] * lam[q], W[j * k + q], a);
      X[e] = a;
    }
    __syncwarp();
    mat_to_svec_warp(k, X, v);
    __syncwarp();
    return;
  }
  auto inb = [&](int i, int j) { return i < k && j < k; };
  if (warm) {   // T = Vp' (X Vp)
    warp_mm16(k, [&](int i, int q) { return inb(i, q) ? X[i * k + q] : 0.0; }, [&](int q, int j) { return inb(q, j) ? Vp[q * k + j] : 0.0; },
              [&](int i, int j, double val) { if (inb(i, j)) W[i * k + j] = val; });
    __syncwarp();
    warp_mm16(k, [&](int i, int q) { return inb(i, q) ? Vp[q * k + i] : 0.0; }, [&](int q, int j) { return inb(q, j) ? W[q * k + j] : 0.0; },
              [&](int i, int j, double val) { if (inb(i, j)) X[i * k + j] = val; });
    __syncwarp();
    // (the product is symmetric up to rounding; the rotations read the upper triangle for the angles)
  } else {
    for (int e = lane; e < k * k; e += 32) Vp[e] = (e / k == e % k) ? 1.0 : 0.0;
    __syncwarp();
  }
  jacobi_par_warp(k, X, Vp);
  for (int i = lane; i < k; i += 32) lam[i] = fmax(X[i * k + i], 0.0);
  __syncwarp();
  warp_mm16(k, [&](int i, int q) { return inb(i, q) ? Vp[i * k + q] * lam[q] : 0.0; }, [&](int q, int j) { return inb(q, j) ? Vp[j * k + q] : 0.0; },
            [&](int i, int j, double val) { if (inb(i, j)) W[i * k + j] = val; });
  __syncwarp();
  mat_to_svec_warp(k, W, v);
  __syncwarp();
}

// ----------------------------------------------------------------------------- exponential cone
// K_exp = cl{(x,y,z): y > 0, y e^{x/y} <= z}.  Thread-level projection (one cone per thread):
// closed-form cases, else bisection on the dual variable with an inner 1-D Newton (Parikh & Boyd,
// Proximal Algorithms 6.3.4) and a Newton polish of the univariate optimality condition in
// rho = x/y; Jacobian by implicit differentiation of the projection's KKT system (4x4 solve).
__device__ inline double exp_newton_one_d(double rho, double yh, double zh) {
  double t = fmax(-zh, 1e-6);
  for (int i = 0; i < 100; i++) {
    const double f = t * (t + zh) / rho / rho - yh / rho + log(t / rho) + 1.0;
    const double fp = (2.0 * t + zh) / rho / rho + 1.0 / t;
    t -= f / fp;
    if (t <= -zh) return 0.0;
    if (t <= 0.0) return zh;
    if (fabs(f) < 1e-13) break;
  }
  return t + zh;
}
__device__ inline double exp_calc_grad(const double *v, double *x, double rho) {
  x[2] = exp_newton_one_d(rho, v[1], v[2]);
  x[1] = (x[2] - v[2]) * x[2] / rho;
  x[0] = v[0] - rho;
  if (x[1] <= 1e-12) return x[0];
  return x[0] + x[1] * log(x[1] / x[2]);
}
__device__ inline double exp_h(double r, double s, double t, double rho, double *y, double *mu) {
  const double E = exp(rho), id = 1.0 / (rho + E * E);
  *y = (r + t * E) * id;
  *mu = (r * E - t * rho) * id;   // = y e^rho - t without its cancellation once y e^rho ~ t
  return *y + *mu * E * (1.0 - rho) - s;
}
// Newton on h(rho) = 0 (rho = x / y of the projection p = (rho y, y, y e^rho); h is the stationarity residual of the
// y-coordinate, exp_h above) with the analytic derivative, started from *rho0 (the previous iterate's root; the
// cone moves little between operator-splitting iterations) or from a crude guess.  Accepts only a root with y > 0,
// mu >= 0 and |h| at rounding level; anything else (no decrease, leaving the domain) returns false and the caller falls
// back to the bisection.  Typically 2-4 iterations warm, 5-8 cold.
__device__ inline bool exp_newton_rho(double r, double s, double t, double *rho0, double *x) {
  double rho = (rho0 && *rho0 == *rho0) ? *rho0 : (s > 0 ? fmin(fmax(r / s, -20.0), 20.0) : (t > 0 && r > 0 ? fmin(log(fmax(t, 1e-300) / fmax(r, 1e-300)) , 20.0) : 0.0));
  const double scale = fmax(1.0, fmax(fabs(r), fmax(fabs(s), fabs(t))));
  double y, mu, hv = exp_h(r, s, t, rho, &y, &mu);
  for (int it = 0; it < 30; it++) {
    if (!(hv == hv)) return false;
    if (fabs(hv) <= 1e-15 * scale) break;
    const double E = exp(rho), den = rho + E * E;
    const double yp = (t * E * den - (r + t * E) * (1.0 + 2.0 * E * E)) / (den * den);
    const double mup = (yp + y) * E;
    const double hp = yp + mup * E * (1.0 - rho) - mu * E * rho;
    if (hp == 0.0 || !(hp == hp)) return false;
    double step = -hv / hp, rn, yn, mn, hn;
    int bt = 0;
    bool stalled = false;
    for (;; bt++) {   // damping: accept the first step that reduces |h| inside the domain
      rn = rho + step;
      hn = exp_h(r, s, t, rn, &yn, &mn);
      if (hn == hn && fabs(hn) < fabs(hv)) break;   // (rho + e^{2 rho} may have either sign: roots exist on both sides of its zero)
      if (bt == 12) { stalled = true; break; }
      step *= 0.5;
    }
    if (stalled) {   // no decrease left: at rounding level that is convergence, anywhere else a failure
      if (fabs(hv) <= 1e-11 * scale) break;
      return false;
    }
    const bool tiny = fabs(step) <= 1e-15 * fmax(1.0, fabs(rn));
    rho = rn; hv = hn; y = yn; mu = mn;
    if (tiny) break;
  }
  if (!(fabs(hv) <= 1e-11 * scale) || !(y > 0)) return false;
  // Certificate (the projection is the unique point with p in K, v - p in the polar cone, p'(v - p) = 0): h = 0 alone can
  // be met by a spurious root where mu = y e^rho - t is pure cancellation, so the dual part is checked on d = v - p itself.
  const double E = exp(rho);
  const double px = y * rho, py = y, pz = y * E;
  const double dx = r - px, dy = s - py, dz = t - pz;           // must be mu (E, (1 - rho) E, -1), mu >= 0
  // the normal divided by max(1, e^rho): mu2 = -dz would carry the rounding of t - y e^rho, times e^rho, into dx
  const double na = E >= 1.0 ? 1.0 : E, n0 = na, n1 = na * (1.0 - rho), n2 = E >= 1.0 ? -1.0 / E : -1.0;
  const double nn = sqrt(n0 * n0 + n1 * n1 + n2 * n2), mu2 = (dx * n0 + dy * n1 + dz * n2) / nn;
  if (!(mu2 >= -1e-13 * scale)) return false;
  if (fabs(dx - mu2 * n0 / nn) > 1e-9 * scale || fabs(dy - mu2 * n1 / nn) > 1e-9 * scale || fabs(dz - mu2 * n2 / nn) > 1e-9 * scale) return false;
  if (fabs(px * dx + py * dy + pz * dz) > 1e-9 * scale * scale) return false;
  x[0] = px; x[1] = py; x[2] = pz;
  if (rho0) *rho0 = rho;
  return true;
}
// The same from a handful of fixed starting points when the first attempt (warm start or crude guess) fails: the
// bisection it saves costs ~10^6 cycles of one thread (measured: cold failures drop from 21 % to 2 % of the iterative cases).
__device__ inline bool exp_newton_multi(double r, double s, double t, double *rho0, double *x) {
  if (exp_newton_rho(r, s, t, rho0, x)) return true;
  const double starts[6] = {0.0, -1.0, 1.0, -3.0, 3.0, 8.0};
#pragma unroll 1
  for (int k = 0; k < 6; k++) {
    double g = starts[k];
    if (exp_newton_rho(r, s, t, &g, x)) { if (rho0) *rho0 = g; return true; }
  }
  return false;
}
// v <- Pi_{K_exp}(v); returns the case (0 inside, 1 polar, 2 analytic face, 3 iterative).  rho0: optional warm start
// slot of this cone (NaN = none), updated when the Newton path was taken.
__device__ inline int proj_exp_unit(double *v, double *rho0) {
  const double r = v[0], s = v[1], t = v[2];
  if ((s > 0 && s * exp(fmin(r / s, 700.0)) - t <= 1e-13) || (r <= 0 && s == 0 && t >= 0)) return 0;
  if ((r > 0 && r * exp(fmin(s / r, 700.0)) + 2.718281828459045 * t <= 1e-13) || (r == 0 && s <= 0 && t <= 0)) { v[0] = v[1] = v[2] = 0; return 1; }
  if (r < 0 && s < 0) { v[1] = 0.0; v[2] = fmax(t, 0.0); return 2; }
  double x[3];
  if (exp_newton_multi(r, s, t, rho0, x)) { v[0] = x[0]; v[1] = x[1]; v[2] = x[2]; return 3; }
  if (rho0) *rho0 = nan("");
  double lb = 0.0, ub = 0.125;
  while (exp_calc_grad(v, x, ub) > 0 && ub < 1e300) { lb = ub; ub *= 2.0; }
  for (int i = 0; i < 200; i++) {
    const double rho = 0.5 * (ub + lb), g = exp_calc_grad(v, x, rho);
    if (g > 0) lb = rho; else ub = rho;
    if (ub - lb < 1e-10 * fmax(1.0, rho)) break;
  }
  if (x[1] > 1e-12) {
    double rr = x[0] / x[1], y, mu, hv = exp_h(r, s, t, rr, &y, &mu);
    for (int it = 0; it < 8; it++) {
      const double d = 1e-7 * fmax(1.0, fabs(rr));
      double y2, m2;
      const double dh = (exp_h(r, s, t, rr + d, &y2, &m2) - exp_h(r, s, t, rr - d, &y2, &m2)) / (2.0 * d);
      if (dh == 0.0) break;
      double yn, mn;
      const double rn = rr - hv / dh, hn = exp_h(r, s, t, rn, &yn, &mn);
      if (!(fabs(hn) < fabs(hv) && yn > 0 && mn >= 0)) break;
      rr = rn; hv = hn; y = yn; mu = mn;
    }
    if (y > 0 && mu >= 0) { x[0] = y * rr; x[1] = y; x[2] = y * exp(rr); if (rho0) *rho0 = rr; }   // next call starts Newton from this root
  }
  v[0] = x[0]; v[1] = x[1]; v[2] = x[2];
  return 3;
}
// The projection is positively homogeneous and its Jacobian homogeneous of degree 0: both work on v / 2^k with max|v_i| in
// [1, 2), so that the absolute thresholds of proj_exp_unit (the 1e-13 case tests, the 1e-12 face test, the Newton and
// bisection tolerances) are relative to |v|; a power of two keeps the scaling exact.
// 2^-k and 2^k are built from the exponent field (k clamped so both stay normal); returns 2^k.
__device__ inline double exp_unit_scale(const double *v, double *u) {
  const double m = fmax(fabs(v[0]), fmax(fabs(v[1]), fabs(v[2])));
  const int k = m > 0.0 ? min(max((int)((__double_as_longlong(m) >> 52) & 0x7ff) - 1023, -1000), 1000) : 0;
  const double down = __longlong_as_double((long long)(1023 - k) << 52);
#pragma unroll
  for (int i = 0; i < 3; i++) u[i] = v[i] * down;
  return __longlong_as_double((long long)(1023 + k) << 52);
}
__device__ inline int proj_exp(double *v, double *rho0 = nullptr) {
  double u[3];
  const double up = exp_unit_scale(v, u);
  const int cs = proj_exp_unit(u, rho0);
#pragma unroll
  for (int i = 0; i < 3; i++) v[i] = u[i] * up;
  return cs;
}
// J (3x3 row-major) = D Pi_{K_exp}(v)
__device__ inline void dproj_exp_mat(const double *v0, double *J) {
  double v[3];
  exp_unit_scale(v0, v);
  double p[3] = {v[0], v[1], v[2]};
  const int cs = proj_exp_unit(p, nullptr);
  for (int i = 0; i < 9; i++) J[i] = 0;
  if (cs == 0) { J[0] = J[4] = J[8] = 1.0; return; }
  if (cs == 1) return;
  if (cs == 2) { J[0] = 1.0; J[8] = v[2] > 0 ? 1.0 : 0.0; return; }
  if (!(p[1] > 1e-12)) { J[0] = v[0] < 0 ? 1.0 : 0.0; J[8] = p[2] > 0 ? 1.0 : 0.0; return; }
  const double rho = p[0] / p[1], E = exp(rho), mu = p[2] - v[2], a = mu * E / p[1];
  double K[4][7] = {{1.0 + a, -a * rho, 0.0, E, 1, 0, 0},
                    {-a * rho, 1.0 + a * rho * rho, 0.0, E * (1.0 - rho), 0, 1, 0},
                    {0.0, 0.0, 1.0, -1.0, 0, 0, 1},
                    {E, E * (1.0 - rho), -1.0, 0.0, 0, 0, 0}};
#pragma unroll
  for (int c = 0; c < 4; c++) {
    int pv = c;
#pragma unroll
    for (int r2 = c + 1; r2 < 4; r2++) if (fabs(K[r2][c]) > fabs(K[pv][c])) pv = r2;
#pragma unroll
    for (int r2 = 0; r2 < 4; r2++) if (r2 == pv && pv != c) {
#pragma unroll
      for (int k = 0; k < 7; k++) { const double tmp = K[c][k]; K[c][k] = K[r2][k]; K[r2][k] = tmp; }
    }
    const double ip = 1.0 / K[c][c];
#pragma unroll
    for (int k = 0; k < 7; k++) K[c][k] *= ip;
#pragma unroll
    for (int r2 = 0; r2 < 4; r2++) if (r2 != c) {
      const double f = K[r2][c];
#pragma unroll
      for (int k = 0; k < 7; k++) K[r2][k] -= f * K[c][k];
    }
  }
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) J[i * 3 + j] = K[i][4 + j];
}
// y-block versions: rows whose primal cone is K_exp project onto K* (Moreau), rows whose primal
// cone is the dual exponential cone project onto K_exp itself.
__device__ inline void proj_exp_dualblock(double *v, bool primal_is_exp, double *rho0 = nullptr) {
  if (primal_is_exp) { double w[3] = {-v[0], -v[1], -v[2]}; proj_exp(w, rho0); v[0] += w[0]; v[1] += w[1]; v[2] += w[2]; }
  else proj_exp(v, rho0);
}
__device__ inline void dproj_exp_dualblock_mat(const double *v, bool primal_is_exp, double *J) {
  if (primal_is_exp) {
    double w[3] = {-v[0], -v[1], -v[2]};
    dproj_exp_mat(w, J);
#pragma unroll
    for (int i = 0; i < 9; i++) J[i] = ((i % 4 == 0) ? 1.0 : 0.0) - J[i];
  } else dproj_exp_mat(v, J);
}

// v (y-space, length m) <- Pi_{K*}(v) for the SOC/PSD blocks; warps stride over cone blocks.
// psd_scr: [per-warp scratch (2 max_psd^2 + max_psd) x warps | persistent eigenvectors, max_psd^2 per PSD block |
// one warm-start slot per exponential cone].  warm: the persistent part was written by a previous call of this instance.
__host__ __device__ inline size_t cone_scratch_doubles(int threads, int max_psd, int ns, int nexp) {
  return (size_t)(max_psd > 0 ? (threads / 32) * (2 * (size_t)max_psd * max_psd + max_psd) + (size_t)ns * max_psd * max_psd : 0) + (size_t)nexp;
}
__device__ __forceinline__ void project_cones(const DevStruct &S, double *v, double *psd_scr, bool warm) {
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int scr_stride = 2 * S.max_psd * S.max_psd + S.max_psd;
  double *persist = psd_scr + (S.max_psd > 0 ? nw * scr_stride : 0);
  for (int cb = warp; cb < S.ncones; cb += nw) {
    const int ty = __ldg(S.cone_type + cb), st = __ldg(S.cone_start + cb);
    if (ty == BC_CSOC) project_soc_warp(v + st, __ldg(S.cone_size + cb));
    else project_psd_warp(v + st, __ldg(S.cone_order + cb), psd_scr + warp * scr_stride, persist + (cb - S.nq) * S.max_psd * S.max_psd, warm);
  }
  double *rho = persist + (S.max_psd > 0 ? S.ns * S.max_psd * S.max_psd : 0);
  for (int e = threadIdx.x; e < S.ep + S.ed; e += blockDim.x) {
    if (!warm) rho[e] = nan("");
    proj_exp_dualblock(v + S.exp_start + 3 * e, e < S.ep, rho + e);
  }
}

// ----------------------------------------------------------------------------- LSMR
// The adjoint / forward-mode least-squares solve with diffcp's mode = "lsmr": LSMR (Fong & Saunders 2011) with the recurrences,
// norm / condition estimates and stopping rules of scipy.sparse.linalg.lsmr at damp = 0 (SciPy's rotation Qhat is then
// (sign(alphabar), 0, |alphabar|)).  Shared by the three backward kernels, which differ only in the operator.

// SciPy's _sym_ortho: the stable Givens rotation [c s; -s c] [a; b] = [r; 0]
__device__ __forceinline__ void sym_ortho(double a, double b, double &c, double &s, double &r) {
  if (b == 0) { c = a > 0 ? 1.0 : (a < 0 ? -1.0 : 0.0); s = 0.0; r = fabs(a); }
  else if (a == 0) { c = 0.0; s = b > 0 ? 1.0 : -1.0; r = fabs(b); }
  else if (fabs(b) > fabs(a)) { const double tau = a / b; s = copysign(1.0, b) / sqrt(1.0 + tau * tau); c = s * tau; r = b / s; }
  else { const double tau = b / a; c = copysign(1.0, a) / sqrt(1.0 + tau * tau); s = c * tau; r = a / c; }
}

// Block-cooperative LSMR on an N x N operator B: every thread of the block calls it with the same arguments.  U holds the
// right-hand side on entry; V, H, Hb are work vectors; X returns the solution (B'B X = B' rhs in the least-squares sense).
// opB(in, out, coef): out <- B in + coef out, opBT the same with B'; both return ||out||^2 (the same bits in every thread)
// and end with a barrier.  Returns the iteration count (0: b = 0 or B'b = 0, X = 0).
template <class OpB, class OpBT>
__device__ __forceinline__ int lsmr_block(int N, double *U, double *V, double *H, double *Hb, double *X, double *red, const bc_settings &st,
                                       int iter_lim, OpB opB, OpBT opBT) {
  const int t = threadIdx.x, T = blockDim.x;
  const double atol = st.lsqr_atol, btol = st.lsqr_btol, ctol = st.lsqr_conlim > 0 ? 1.0 / st.lsqr_conlim : 0.0;
  double r1[1] = {0};
  for (int k = t; k < N; k += T) { r1[0] = fma(U[k], U[k], r1[0]); X[k] = 0.0; V[k] = 0.0; }
  block_reduce<1, false>(r1, red);
  const double normb = sqrt(r1[0]);
  double beta = normb, alpha = 0;
  if (beta > 0) {
    const double ib = 1.0 / beta;
    for (int k = t; k < N; k += T) U[k] *= ib;
    __syncthreads();
    alpha = sqrt(opBT(U, V, 0.0));   // v = B' u
  }
  {
    const double ia = alpha > 0 ? 1.0 / alpha : 1.0;
    for (int k = t; k < N; k += T) { const double v = V[k] * ia; V[k] = v; H[k] = v; Hb[k] = 0.0; }
    __syncthreads();
  }
  if (alpha * beta == 0.0) return 0;   // SciPy: normar = alpha beta = 0 or normb = 0 -> x = 0
  double zetabar = alpha * beta, alphabar = alpha, rho = 1, rhobar = 1, cbar = 1, sbar = 0;
  double betadd = beta, betad = 0, rhodold = 1, tautildeold = 0, thetatilde = 0, zeta = 0, d = 0;
  double normA2 = alpha * alpha, maxrbar = 0, minrbar = 1e100;
  int itn = 0;
  while (itn < iter_lim) {
    itn++;
    beta = sqrt(opB(V, U, -alpha));   // u = B v - alpha u
    double vs = 1.0;                    // v's normalisation, applied in the update pass below
    if (beta > 0) {
      const double ib = 1.0 / beta;
      for (int k = t; k < N; k += T) U[k] *= ib;
      __syncthreads();
      alpha = sqrt(opBT(U, V, -beta));   // v = B' u - beta v
      if (alpha > 0) vs = 1.0 / alpha;
    }
    double chat, shat, alphahat;
    sym_ortho(alphabar, 0.0, chat, shat, alphahat);
    const double rhoold = rho;
    double c, s;
    sym_ortho(alphahat, beta, c, s, rho);
    const double thetanew = s * alpha;
    alphabar = c * alpha;
    const double rhobarold = rhobar, zetaold = zeta, thetabar = sbar * rho, rhotemp = cbar * rho;
    sym_ortho(cbar * rho, thetanew, cbar, sbar, rhobar);
    zeta = cbar * zetabar;
    zetabar = -sbar * zetabar;
    // hbar = h - thetabar rho / (rhoold rhobarold) hbar;  x += zeta / (rho rhobar) hbar;  h = v - thetanew / rho h;  ||x||^2
    const double chb = -(thetabar * rho / (rhoold * rhobarold)), cx = zeta / (rho * rhobar), ch = -(thetanew / rho);
    r1[0] = 0;
    for (int k = t; k < N; k += T) {
      const double v = V[k] * vs, h = H[k];
      const double hb = fma(Hb[k], chb, h), x = fma(cx, hb, X[k]);
      V[k] = v; Hb[k] = hb; X[k] = x; H[k] = fma(h, ch, v);
      r1[0] = fma(x, x, r1[0]);
    }
    block_reduce<1, false>(r1, red);
    const double normx = sqrt(r1[0]);
    // ||r|| estimate
    const double betaacute = chat * betadd, betacheck = -shat * betadd, betahat = c * betaacute;
    betadd = -s * betaacute;
    const double thetatildeold = thetatilde;
    double ctildeold, stildeold, rhotildeold;
    sym_ortho(rhodold, thetabar, ctildeold, stildeold, rhotildeold);
    thetatilde = stildeold * rhobar;
    rhodold = ctildeold * rhobar;
    betad = -stildeold * betad + ctildeold * betahat;
    tautildeold = (zetaold - thetatildeold * tautildeold) / rhotildeold;
    const double taud = (zeta - thetatilde * tautildeold) / rhodold;
    d += betacheck * betacheck;
    const double normr = sqrt(d + (betad - taud) * (betad - taud) + betadd * betadd);
    // ||B|| and cond(B) estimates
    normA2 += beta * beta;
    const double normA = sqrt(normA2);
    normA2 += alpha * alpha;
    maxrbar = fmax(maxrbar, rhobarold);
    if (itn > 1) minrbar = fmin(minrbar, rhobarold);
    const double condA = fmax(maxrbar, rhotemp) / fmin(minrbar, rhotemp);
    // stopping rules
    const double normar = fabs(zetabar);
    const double test1 = normr / normb, test2 = normA * normr != 0.0 ? normar / (normA * normr) : INFINITY, test3 = 1.0 / condA;
    const double t1 = test1 / (1.0 + normA * normx / normb), rtol = btol + atol * normA * normx / normb;
    int istop = 0;
    if (itn >= iter_lim) istop = 7;
    if (1.0 + test3 <= 1.0) istop = 6;
    if (1.0 + test2 <= 1.0) istop = 5;
    if (1.0 + t1 <= 1.0) istop = 4;
    if (test3 <= ctol) istop = 3;
    if (test2 <= atol) istop = 2;
    if (test1 <= rtol) istop = 1;
    if (istop) break;
  }
  return itn;
}

// ----------------------------------------------------------------------------- host entry points
// Everything api.cu calls in the kernel files, declared once so that the compiler checks each definition against its uses.
// Per kernel family: the size functions, and one lookup from the variant to the kernel's address (nullptr: no such
// instantiation).  api.cu configures and launches through that address, so a new kernel variant is registered by adding its
// row to the family's lookup.
extern "C" {
// fwd.cu
size_t bc_fwd_smem_bytes(int n, int m, int nnzA, int threads, int max_psd, int indirect, int ns, int nexp, int vals_global);
size_t bc_fwd_ws_doubles(int n, int m, int vectors, int with_factor, int nnzA_global);
const void *bc_fwd_kernel(int dense, int indirect, int small_cta, int vals_global);
// fwd_fast.cu
size_t bc_fwdf_smem_bytes(int n, int m);
int bc_fwdf_threads(void);
size_t bc_fwdf_cache_doubles(int n, int m);
int bc_fwdf_eligible(int n, int m);
const void *bc_fwdf_kernel(int n, int m);
// bwd.cu (adjoint and forward mode; lsmr: the LSMR variant, one more N-vector)
size_t bc_bwd_smem_bytes(int n, int m, int npoly, int nnzA, int nnzP_smem, int threads, int max_psd, int psd_total, int nexp, int vec_global,
                         int vals_global, int lsmr);
size_t bc_bwd_ws_doubles(int n, int m, int npoly, int lsmr);
const void *bc_lsqr_kernel(int dense, int small_cta, int jvp, int vals_global, int lsmr);
// bwd_fast.cu, bwd_block.cu
size_t bc_bwdf_smem_bytes(int n, int m, int nnzA, int nnzP, int threads, int lsmr);
const void *bc_bwdf_kernel(int n, int lsmr);
size_t bc_bwdb_smem_bytes(int n, int m, int threads);   // (the same for both variants)
const void *bc_bwdb_kernel(int lsmr);
// bwd_lsmr.cu, bwd_fast_lsmr.cu, bwd_block_lsmr.cu: the LSMR kernels (reached through the three lookups above)
const void *bc_lsmr_kernel(int dense, int small_cta, int jvp, int vals_global);
const void *bc_bwdf_lsmr_kernel(int n);
const void *bc_bwdb_lsmr_kernel(void);
// refine.cu (bwd.cu compiled with BC_REFINE)
size_t bc_refine_smem_bytes(int n, int m, int npoly, int nnzA, int nnzP_smem, int threads, int max_psd, int psd_total, int nexp, int vec_global,
                            int vals_global);
size_t bc_refine_ws_doubles(int n, int m, int npoly);
const void *bc_refine_kernel(int dense, int small_cta, int vals_global);
// polish.cu
size_t bc_polish_smem_bytes(int n, int m, int threads, long long stage_cap);
const void *bc_polish_kernel(int dense);
// polish_large.cu (the slab tier of polishing)
long long bc_polish_large_slab_doubles(int n, int m, int threads, int p_diag);
size_t bc_polish_large_smem_bytes(int threads);
int bc_polish_large_threads(void);
const void *bc_polish_large_kernel(int dense);
// pack.cu
cudaError_t bc_b2e(const double *in, double *out, int K, int B, int ldo, int roff, const int *smap, const int *dmap, double sign, long long ldb,
                   cudaStream_t st);
cudaError_t bc_e2b(const double *in, double *out, int K, int B, int ldi, int roff, const int *smap, const int *dmap, double sign, long long ldb,
                   cudaStream_t st);
cudaError_t bc_p2e(const double *p, const int *rptr, const int *cols, const double *vals, double *out, int K, int B, int ldo, int roff,
                   const int *smap, const int *dmap, double sign, long long ldp, cudaStream_t st);
cudaError_t bc_e2p(const double *in, const int *rptr, const int *cols, const double *vals, double *dp, int K, int B, int ldi, int roff,
                   const int *smap, const int *dmap, double sign, int skip, long long ldp, cudaStream_t st);
cudaError_t bc_rows_from_param(const double *param, long long stride, const int *map, int K, int B, int op, double *rows, cudaStream_t st);
cudaError_t bc_param_from_rows(const double *grows, const double *param, long long stride, const int *map, int K, int B, int op, double *gparam,
                               cudaStream_t st);
cudaError_t bc_gather_cols(const double *in, long long ld, const int *map, const double *scale, int K, int B, int op, double *out, cudaStream_t st);
cudaError_t bc_scatter_cols(const double *gout, const double *out, long long ld, const int *map, const double *scale, int K, int B, int op, double *gin,
                            cudaStream_t st);
// shared.cu
size_t bc_shared_part_doubles(const DevStruct *S, int B);
cudaError_t bc_shared_grad(const DevStruct *S, const double *rec, const double *x, int B, double *dA, double *dP, double *part, cudaStream_t st);
}
