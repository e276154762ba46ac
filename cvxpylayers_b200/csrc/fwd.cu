// fwd.cu -- forward solve kernel: operator splitting on the homogeneous self-dual embedding
// (the work diffcp/SCS do for the reference at src/cvxpylayers/interfaces/diffcp_if.py:365,369;
// rows F3-F6 of SURVEY.md section 8a).  One persistent CTA per instance; the instance's CSR
// values (TMA bulk copy), the packed inverse Cholesky factor of the reduced normalised KKT
// matrix and every iterate vector stay in shared memory for the whole solve (larger instances: see the modes below and the
// values-off-chip build, fwd_kernel<.., VG = true>).
//
// Per iteration (all on-chip):
//   t_n  = rho_x w_x - A' w_y                         (transposed product, lanes across columns)
//   p_x  = Linv' (Linv t_n)                            (two packed-triangular products)
//   p_y  = w_y + (A p_x) / r_y                         (row product, warp per row, butterfly reduce)
//   tau~ = positive root of the embedding's quadratic  (four fused R-weighted dot products)
//   u    = Pi_{R^n x K* x R+}(2 u~ - w),  w += alpha (u - u~)
// Every check_interval iterations: SCS termination quantities on the un-normalised data,
// infeasibility certificates, adaptive scale (re-factorisation on chip).
#include "common.cuh"

// Sub-phase cycle counters (tools/phase_profile.py, slots 16..28) cost registers and issue slots in the iteration
// loop: compiled in only with -DBC_SUBPROF.  The five coarse phases (slots 0..4) are always available.
#ifdef BC_SUBPROF
#define SUB_DECL(name) PhaseTimer name; name.start(a.prof)
#define SUB_SKIP(name) name.skip()
#define SUB_STAMP(name, k) name.stamp(k)
#else
#define SUB_DECL(name)
#define SUB_SKIP(name)
#define SUB_STAMP(name, k)
#endif

struct FwdSmem {
  double *Av, *Li, *w, *u, *ut, *g, *bh, *ch, *Dm, *En, *tn, *tn2, *tn3, *tm, *part, *red, *psd, *cr, *cp, *cq, *kd, *cx;
  uint64_t *bar;
  int *ibuf;
};

// Vector block shared by both modes (doubles): iterate + work vectors (+ CG vectors when INDIRECT).
__host__ __device__ inline size_t fwd_vec_doubles(int n, int m, int indirect) {
  size_t N = (size_t)n + m + 1;
  return 3 * N + (n + m) + m + n + m + n + n + n + n + m + (indirect ? 5 * (size_t)n : 0);
}
// DIRECT: everything on chip.  INDIRECT (instances whose n x n Cholesky does not fit): the CSR values,
// the reduction scratch and the PSD scratch stay in shared memory, the vectors move to a global slab.
__host__ __device__ inline size_t fwd_part_doubles(int n, int threads) {   // (also the LU scratch of the Anderson step: BC_AA_LU = 272)
  const size_t d = (size_t)(8 * n > threads ? 8 * n : threads);
  return d > 272 ? d : 272;
}
// vals_global: the CSR values live in the per-CTA slab instead (instances whose values do not fit next to the rest).
__host__ __device__ inline size_t fwd_smem_doubles(int n, int m, int nnzA, int threads, int max_psd, int indirect, int ns, int nexp, int vals_global) {
  size_t nA = vals_global ? 0 : ((size_t)nnzA + 1) & ~(size_t)1;
  size_t d = 4 + nA + fwd_part_doubles(n, threads) + 8 * 32;
  if (!indirect) d += (size_t)n * (n + 1) / 2 + fwd_vec_doubles(n, m, 0);
  return d + cone_scratch_doubles(threads, max_psd, ns, nexp);
}

// gws != nullptr: the vectors live in the per-CTA global slab; li_global: the packed Cholesky factor follows them there
// (mode 2: instances whose values fit on chip but whose factor does not -- the factor is then read from L2 / HBM twice per
// iteration, which is still far cheaper than the conjugate-gradient solve of the indirect mode).
// VG: the values are at `vals` (the front of the slab) and take no shared memory.
template <bool VG = false>
__device__ __forceinline__ void carve(FwdSmem &M, double *base, double *gws, int n, int m, int nnzA, int threads, int max_psd, bool li_global = false,
                                      double *vals = nullptr) {
  const int N = n + m + 1;
  double *q = base;
  M.bar = (uint64_t *)q; q += 2;
  M.ibuf = (int *)q; q += 2;
  if (VG) M.Av = vals;
  else { M.Av = q; q += (nnzA + 1) & ~1; }
  M.part = q; q += fwd_part_doubles(n, threads); M.red = q; q += 8 * 32;
  if (!gws) { M.Li = q; q += n * (n + 1) / 2; } else M.Li = nullptr;
  double *v = gws ? gws : q;
  M.w = v; v += N; M.u = v; v += N; M.ut = v; v += N;
  M.g = v; v += n + m; M.bh = v; v += m; M.ch = v; v += n; M.Dm = v; v += m; M.En = v; v += n;
  M.tn = v; v += n; M.tn2 = v; v += n; M.tn3 = v; v += n; M.tm = v; v += m;
  if (gws) { M.cr = v; v += n; M.cp = v; v += n; M.cq = v; v += n; M.kd = v; v += n; M.cx = v; v += n; if (li_global) { v += ((size_t)(v - gws) & 1); M.Li = v; } }
  else { M.cr = M.cp = M.cq = M.kd = M.cx = nullptr; q = v; }
  M.psd = q;
}

__device__ __forceinline__ double inv_ry(const DevStruct &S, int i, double scale) {
  return i < S.z ? BC_ZERO_CONE_FACTOR * scale : scale;
}

// ----------------------------------------------------------------------------- INDIRECT linear system
// out = K v,  K = rho_x I + P^ + A^' R_y^{-1} A^   (two sparse products; SCS "indirect" mode)
template <bool DENSE>
__device__ void K_mul(const FwdArgs &a, FwdSmem &M, const double *Pv, double scale, double rho_x, const double *v, double *out,
                      const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const bool wide = DENSE && (S.n % 2 == 0) && S.n <= 128;
  const int n = S.n, T = blockDim.x, t = threadIdx.x;
  A_mul<DENSE>(S, M.Av, v, [&](int i, double q) { M.tm[i] = q * inv_ry(S, i, scale); }, wide);
  __syncthreads();
  AT_mul<DENSE>(S, M.Av, M.tm, M.part, [&](int j, double q) { out[j] = q + rho_x * v[j]; }, plA, wide);
  if (Pv) {
    for (int j = t; j < n; j += T) M.tn3[j] = M.En[j] * v[j];
    __syncthreads();
    P_mul(S, Pv, M.tn3, M.part, [&](int j, double q) { out[j] += M.En[j] * q; }, plN);
  }
}
// Jacobi-preconditioned CG on K x = rhs, warm-started from x; stops at ||r|| <= tol.  Returns iterations.
template <bool DENSE>
__device__ int cg_solve(const FwdArgs &a, FwdSmem &M, const double *Pv, double scale, double rho_x, const double *rhs, double *x,
                        double tol, int maxit, const ColPlan &plA, const ColPlan &plN) {
  const int n = a.S.n, T = blockDim.x, t = threadIdx.x;
  K_mul<DENSE>(a, M, Pv, scale, rho_x, x, M.cq, plA, plN);
  double r2[2] = {0, 0};
  for (int j = t; j < n; j += T) {
    const double r = rhs[j] - M.cq[j], z = r / M.kd[j];
    M.cr[j] = r; M.cp[j] = z; r2[0] = fma(r, z, r2[0]); r2[1] = fma(r, r, r2[1]);
  }
  block_reduce<2, false>(r2, M.red);
  double rz = r2[0];
  int it = 0;
  while (it < maxit && sqrt(r2[1]) > tol) {
    it++;
    __syncthreads();
    K_mul<DENSE>(a, M, Pv, scale, rho_x, M.cp, M.cq, plA, plN);
    double pq[1] = {0};
    for (int j = t; j < n; j += T) pq[0] = fma(M.cp[j], M.cq[j], pq[0]);
    block_reduce<1, false>(pq, M.red);
    const double alpha = rz / pq[0];
    r2[0] = 0; r2[1] = 0;
    for (int j = t; j < n; j += T) {
      x[j] = fma(alpha, M.cp[j], x[j]);
      const double r = fma(-alpha, M.cq[j], M.cr[j]), z = r / M.kd[j];
      M.cr[j] = r; M.cq[j] = z; r2[0] = fma(r, z, r2[0]); r2[1] = fma(r, r, r2[1]);
    }
    block_reduce<2, false>(r2, M.red);
    const double beta = r2[0] / rz;
    rz = r2[0];
    for (int j = t; j < n; j += T) M.cp[j] = fma(beta, M.cp[j], M.cq[j]);
  }
  __syncthreads();
  return it;
}

// K = rho_x I + P^ + A^' R_y^{-1} A^ (packed lower) -> Cholesky -> in-place inverse Linv;
// then g = (R_z + M)^{-1} h and g'Rg.  Returns false if the factorisation broke down.
template <bool DENSE, bool INDIRECT>
__device__ bool factor_and_g(const FwdArgs &a, FwdSmem &M, const double *Pv, double scale, double rho_x, double &gRg,
                             const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  const int npk = n * (n + 1) / 2;
  const bool wide = DENSE && (n % 2 == 0) && n <= 128;
  double *K = M.Li;
  SUB_DECL(pf);
  if (INDIRECT) {
    // Jacobi preconditioner diag(K), then g = (R_z + M)^{-1} h by CG at tight tolerance
    for (int i = t; i < m; i += T) M.tm[i] = inv_ry(S, i, scale);
    for (int j = t; j < n; j += T) M.tn3[j] = 0.0;
    __syncthreads();
    AT_mul<DENSE, true>(S, M.Av, M.tm, M.part, [&](int j, double v) { M.kd[j] = rho_x + v; }, plA, wide);
    if (Pv) {
      for (int k = t; k < S.nnzP; k += T) { const int i = __ldg(S.P_rowof + k); if (__ldg(S.P_indices + k) == i) M.kd[i] += Pv[k] * M.En[i] * M.En[i]; }
      __syncthreads();
    }
    for (int i = t; i < m; i += T) M.tm[i] = M.bh[i] * inv_ry(S, i, scale);
    __syncthreads();
    AT_mul<DENSE>(S, M.Av, M.tm, M.part, [&](int j, double v) { M.tn[j] = M.ch[j] - v; M.g[j] = 0.0; }, plA, wide);
    double nr[1] = {0};
    for (int j = t; j < n; j += T) nr[0] = fma(M.tn[j], M.tn[j], nr[0]);
    block_reduce<1, false>(nr, M.red);
    cg_solve<DENSE>(a, M, Pv, scale, rho_x, M.tn, M.g, 1e-13 * fmax(1.0, sqrt(nr[0])), 10 * n, plA, plN);
    A_mul<DENSE>(S, M.Av, M.g, [&](int i, double v) { M.g[n + i] = (M.bh[i] + v) * inv_ry(S, i, scale); }, wide);
    __syncthreads();
    double acc[1] = {0};
    for (int k = t; k < n + m; k += T) {
      const double r = k < n ? rho_x : 1.0 / inv_ry(S, k - n, scale);
      acc[0] = fma(r * M.g[k], M.g[k], acc[0]);
    }
    block_reduce<1, false>(acc, M.red);
    gRg = acc[0];
    return true;
  }
  if (DENSE && wide) {
    // K_jk = scale * sum_i w_i A_ij A_ik (w = 1000 on zero-cone rows): 2x2 register tiles, 128-bit loads
    const int nb = n >> 1, ntile = (nb * (nb + 1)) >> 1;
    for (int e = t; e < ntile; e += T) {
      int J = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
      while (((J + 1) * (J + 2)) >> 1 <= e) J++;
      while ((J * (J + 1)) >> 1 > e) J--;
      const int Kb = e - ((J * (J + 1)) >> 1);
      const double2 *pj = reinterpret_cast<const double2 *>(M.Av) + J, *pk = reinterpret_cast<const double2 *>(M.Av) + Kb;
      double z00 = 0, z01 = 0, z10 = 0, z11 = 0, s00 = 0, s01 = 0, s10 = 0, s11 = 0;
      int i = 0;
      for (; i < S.z; i++) { const double2 u = pj[i * nb], v = pk[i * nb]; z00 = fma(u.x, v.x, z00); z01 = fma(u.x, v.y, z01); z10 = fma(u.y, v.x, z10); z11 = fma(u.y, v.y, z11); }
      for (; i < m; i++) { const double2 u = pj[i * nb], v = pk[i * nb]; s00 = fma(u.x, v.x, s00); s01 = fma(u.x, v.y, s01); s10 = fma(u.y, v.x, s10); s11 = fma(u.y, v.y, s11); }
      const int j0 = 2 * J, k0 = 2 * Kb;
      K[((j0 * (j0 + 1)) >> 1) + k0] = (z00 * BC_ZERO_CONE_FACTOR + s00) * scale + (j0 == k0 ? rho_x : 0.0);
      if (k0 + 1 <= j0) K[((j0 * (j0 + 1)) >> 1) + k0 + 1] = (z01 * BC_ZERO_CONE_FACTOR + s01) * scale;
      K[(((j0 + 1) * (j0 + 2)) >> 1) + k0] = (z10 * BC_ZERO_CONE_FACTOR + s10) * scale;
      K[(((j0 + 1) * (j0 + 2)) >> 1) + k0 + 1] = (z11 * BC_ZERO_CONE_FACTOR + s11) * scale + (j0 == k0 ? rho_x : 0.0);
    }
    __syncthreads();
  } else if (DENSE) {
    for (int e = t; e < npk; e += T) {
      int j = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
      while ((j + 1) * (j + 2) / 2 <= e) j++;
      while (j * (j + 1) / 2 > e) j--;
      const int k = e - j * (j + 1) / 2;
      double acc0 = 0, acc1 = 0;
      const double *cj = M.Av + j, *ck = M.Av + k;
      int i = 0;
      for (; i < S.z; i++) acc0 = fma(cj[i * n], ck[i * n], acc0);
      for (; i < m; i++) acc1 = fma(cj[i * n], ck[i * n], acc1);
      K[e] = (acc0 * BC_ZERO_CONE_FACTOR + acc1) * scale + (j == k ? rho_x : 0.0);
    }
    __syncthreads();
  } else {
    for (int e = t; e < npk; e += T) K[e] = 0.0;
    __syncthreads();
    for (int e = t; e < n; e += T) K[e * (e + 1) / 2 + e] = rho_x;
    // The diagonal must be in place before ANY thread accumulates into it: without this barrier a fast thread's atomicAdd on a
    // diagonal entry could land before the plain store above and be overwritten by it -- K then lacks a_jj^2 terms, may lose
    // positive definiteness, and the instance is reported FAILED.  (Round 1's code had the race; it surfaced as an
    // intermittent failure of one in ~2000 SOCP instances once two launches shared the SMs; compute-sanitizer racecheck named
    // this line and no other.)
    __syncthreads();
    for (int k = t; k < S.nnzA; k += T) {
      const int i = __ldg(S.A_rowof + k), ja = __ldg(S.A_indices + k);
      const double va = M.Av[k] * inv_ry(S, i, scale);
      const int e = __ldg(S.A_indptr + i + 1);
      for (int k2 = __ldg(S.A_indptr + i); k2 < e; k2++) {
        const int jb = __ldg(S.A_indices + k2);
        if (jb <= ja) atomicAdd(&K[ja * (ja + 1) / 2 + jb], va * M.Av[k2]);
      }
    }
    __syncthreads();
  }
  SUB_STAMP(pf, 19);
  if (Pv) {
    for (int k = t; k < S.nnzP; k += T) {
      const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);  // j >= i
      atomicAdd(&K[j * (j + 1) / 2 + i], Pv[k] * M.En[i] * M.En[j]);
    }
    __syncthreads();
  }
  SUB_STAMP(pf, 20);
  if (!chol_inv_packed(K, n, M.part)) return false;   // scratch: part (8 n) + red (256) are contiguous
  SUB_STAMP(pf, 21);
  // ---- g = (R_z + M)^{-1} h, h = (c^, b^) ----
  for (int i = t; i < m; i += T) M.tm[i] = M.bh[i] * inv_ry(S, i, scale);
  __syncthreads();
  AT_mul<DENSE>(S, M.Av, M.tm, M.part, [&](int j, double v) { M.tn[j] = M.ch[j] - v; }, plA, wide);
  if (DENSE) { /* AT_mul ended with a sync */ }
  matvec_rows(M.Li, PackedLowerLayout{}, n, n, M.tn, [&](int i, double v) { M.tn2[i] = v; });
  __syncthreads();
  matvec_cols(M.Li, PackedLowerLayout{}, n, n, M.tn2, M.part, [&](int j, double v) { M.g[j] = v; }, plN);
  A_mul<DENSE>(S, M.Av, M.g, [&](int i, double v) { M.g[n + i] = (M.bh[i] + v) * inv_ry(S, i, scale); }, wide);
  __syncthreads();
  double acc[1] = {0};
  for (int k = t; k < n + m; k += T) {
    const double r = k < n ? rho_x : 1.0 / inv_ry(S, k - n, scale);
    acc[0] = fma(r * M.g[k], M.g[k], acc[0]);
  }
  block_reduce<1, false>(acc, M.red);
  gRg = acc[0];
  SUB_STAMP(pf, 22);
  return true;
}

// SMALL: instances that run with <= 256 threads per CTA and a few tens of KB of shared memory are bound by the latency of one
// CTA's dependent chain (barriers, reductions, a single projecting warp); compiled for four resident CTAs per SM (64 registers)
// they overlap each other's stalls.  The large variant keeps 128 registers and one CTA of up to 512 threads per SM.
// VG (values off chip): instances whose CSR values do not fit in shared memory.  Each CTA copies the instance's values to the
// front of its slab (Ruiz rescales them in place, the caller's A_vals stay untouched) and every product reads them from L2 / HBM;
// the vectors and the factor stay on chip when they fit (a.slab_vectors = 0), else they follow the values in the slab.
template <bool DENSE, bool INDIRECT, bool SMALL = false, bool VG = false>
__global__ void __launch_bounds__(SMALL ? 256 : 512, SMALL ? 4 : 1) fwd_kernel(const __grid_constant__ FwdArgs a) {
  extern __shared__ __align__(16) double smem[];
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, N = n + m + 1, T = blockDim.x, t = threadIdx.x;
  const bc_settings &st = a.st;
  FwdSmem M;
  if constexpr (VG) {
    double *const slab = a.ws + (size_t)blockIdx.x * a.ws_stride;   // [values (even count: 16-byte aligned) | vectors | factor]
    const bool vecs = INDIRECT || a.slab_vectors;
    carve<true>(M, smem, vecs ? slab + ((S.nnzA + 1) & ~1) : nullptr, n, m, S.nnzA, T, S.max_psd, !INDIRECT && vecs, slab);
  } else {
    carve(M, smem, a.ws ? a.ws + (size_t)blockIdx.x * a.ws_stride : nullptr, n, m, S.nnzA, T, S.max_psd, !INDIRECT && a.ws != nullptr);
  }
  if (t == 0) { mbar_init(M.bar, 1); fence_mbar_init(); }
  __syncthreads();
  uint32_t tma_phase = 0;
  const ColPlan plA = make_colplan(m, n), plN = make_colplan(n, n);
  const bool wide = DENSE && (n % 2 == 0) && n <= 128;
  const double rho_x = st.rho_x, alpha = st.alpha, dtau = BC_TAU_FACTOR;

  for (;;) {
    if (t == 0) M.ibuf[0] = atomicAdd(a.counter, 1);
    __syncthreads();
    const int inst = M.ibuf[0];
    if (inst >= a.B) break;
    const double *Ag = a.A_vals + (size_t)inst * a.sA;
    const double *Pg = (a.P_vals && S.nnzP > 0) ? a.P_vals + (size_t)inst * a.sP : nullptr;
    const double *bg = a.b + (size_t)inst * m, *cg = a.c + (size_t)inst * n;
    PhaseTimer pt; pt.start(a.prof);
    SUB_DECL(pi);

    // ---- stage the instance: one TMA bulk copy for the CSR values, plain loads for b, c ----
    if constexpr (VG) {   // values into the slab: 128-bit copies when the instance's row is 16-byte aligned
      if ((((uintptr_t)Ag) & 15) == 0) {
        const double2 *src = reinterpret_cast<const double2 *>(Ag);
        double2 *dst = reinterpret_cast<double2 *>(M.Av);
        for (int k = t; k < (S.nnzA >> 1); k += T) dst[k] = __ldg(src + k);
        if ((S.nnzA & 1) && t == 0) M.Av[S.nnzA - 1] = __ldg(Ag + S.nnzA - 1);
      } else {
        for (int k = t; k < S.nnzA; k += T) M.Av[k] = __ldg(Ag + k);
      }
    } else if (a.use_tma) {
      if (t == 0) {
        fence_proxy_async();
        mbar_expect_tx(M.bar, (uint32_t)(S.nnzA * sizeof(double)));
        tma_bulk_g2s(M.Av, Ag, (uint32_t)(S.nnzA * sizeof(double)), M.bar);
      }
    } else {
      for (int k = t; k < S.nnzA; k += T) M.Av[k] = Ag[k];
    }
    double nb0 = 0, nc0 = 0;
    for (int i = t; i < m; i += T) { const double v = bg[i]; M.bh[i] = v; M.Dm[i] = 1.0; nb0 = fmax(nb0, fabs(v)); }
    for (int j = t; j < n; j += T) { const double v = cg[j]; M.ch[j] = v; M.En[j] = 1.0; nc0 = fmax(nc0, fabs(v)); }
    if (!VG && a.use_tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }
    __syncthreads();

    pt.stamp(0);   // load
    // ---- Ruiz equilibration: A^ = D A E, P^ = E P E (SURVEY.md 8a F4) ----
    if (st.normalize) {
      for (int pass = 0; pass < st.ruiz_passes; pass++) {
        SUB_SKIP(pi);
        // row and column inf-norms of the current A^ (and P^)
        if (DENSE && n <= 128) {
          // lazily scaled pass: A stays unscaled in shared memory, norms are taken through the running
          // D, E; one sweep yields row maxima (warp reduce) and column maxima (per-lane, 8 slots)
          const int lane = t & 31, warp = t >> 5, nw = T >> 5;
          double er[4], cacc[4] = {0, 0, 0, 0};
#pragma unroll
          for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; er[k] = c < n ? M.En[c] : 0.0; }
          for (int i = warp; i < m; i += nw) {
            const double d = M.Dm[i];
            const double *row = M.Av + i * n;
            double r = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
              const int c = lane + 32 * k;
              if (c < n) { const double v = fabs(row[c]) * er[k]; r = fmax(r, v); cacc[k] = fmax(cacc[k], v * d); }
            }
            r = warp_max(r) * d;
            if (lane == 0) M.tm[i] = r;
          }
          const int slot = warp & 7;
          if (warp < 8) {
#pragma unroll
            for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; if (c < n) M.part[slot * n + c] = cacc[k]; }
          }
          __syncthreads();
          if (warp >= 8) {
#pragma unroll
            for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; if (c < n) M.part[slot * n + c] = fmax(M.part[slot * n + c], cacc[k]); }
          }
          __syncthreads();
          if (t < n) { double r = 0; const int ns = nw < 8 ? nw : 8; for (int q = 0; q < ns; q++) r = fmax(r, M.part[q * n + t]); M.tn[t] = r; }
          __syncthreads();
        } else if (DENSE) {
          const int lane = t & 31, warp = t >> 5, nw = T >> 5;
          for (int i = warp; i < m; i += nw) {
            double r = 0;
            for (int c = lane; c < n; c += 32) r = fmax(r, fabs(M.Av[i * n + c]));
            r = warp_max(r);
            if (lane == 0) M.tm[i] = r;
          }
          for (int jj = t; jj < n; jj += T) { double r = 0; for (int i = 0; i < m; i++) r = fmax(r, fabs(M.Av[i * n + jj])); M.tn[jj] = r; }
          __syncthreads();
        } else {
          for (int i = t; i < m; i += T) {
            double r = 0;
            for (int k = __ldg(S.A_indptr + i); k < __ldg(S.A_indptr + i + 1); k++) r = fmax(r, fabs(M.Av[k]));
            M.tm[i] = r;
          }
          for (int j = t; j < n; j += T) {
            double r = 0;
            for (int k = __ldg(S.At_colptr + j); k < __ldg(S.At_colptr + j + 1); k++) r = fmax(r, fabs(M.Av[__ldg(S.At_perm + k)]));
            M.tn[j] = r;
          }
          __syncthreads();
        }
        SUB_STAMP(pi, 16);
        if (Pg) {
          for (int k = t; k < S.nnzP; k += T) {
            const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);
            const double v = fabs(Pg[k] * M.En[i] * M.En[j]);
            atomicMax((unsigned long long *)&M.tn[i], (unsigned long long)__double_as_longlong(v));
            atomicMax((unsigned long long *)&M.tn[j], (unsigned long long)__double_as_longlong(v));
          }
          __syncthreads();
        }
        SUB_STAMP(pi, 17);
        for (int i = t; i < m; i += T) { const double r = M.tm[i]; M.tm[i] = fmin(fmax(r < 1e-8 ? 1.0 : rsqrt(r), BC_EQ_MIN), BC_EQ_MAX); }
        for (int j = t; j < n; j += T) { const double r = M.tn[j]; M.tn[j] = fmin(fmax(r < 1e-8 ? 1.0 : rsqrt(r), BC_EQ_MIN), BC_EQ_MAX); }
        __syncthreads();
        if (S.ep + S.ed > 0) {
          for (int e = t; e < S.ep + S.ed; e += T) {
            double *q = M.tm + S.exp_start + 3 * e;
            const double mean = (q[0] + q[1] + q[2]) / 3.0;
            q[0] = mean; q[1] = mean; q[2] = mean;
          }
          __syncthreads();
        }
        if (S.ncones > 0) {  // one scale per non-separable cone: the block mean
          const int lane = t & 31, warp = t >> 5, nw = T >> 5;
          for (int cb = warp; cb < S.ncones; cb += nw) {
            const int s0 = __ldg(S.cone_start + cb), sz = __ldg(S.cone_size + cb);
            double sum = 0;
            for (int i = lane; i < sz; i += 32) sum += M.tm[s0 + i];
            sum = warp_sum(sum) / sz;
            for (int i = lane; i < sz; i += 32) M.tm[s0 + i] = sum;
          }
          __syncthreads();
        }
        if (DENSE && n <= 128) {
          /* scaling is applied once, after the last pass */
        } else if (DENSE) {
          for (int k = t; k < S.nnzA; k += T) M.Av[k] *= M.tm[k / n] * M.tn[k % n];
        } else {
          for (int k = t; k < S.nnzA; k += T) M.Av[k] *= M.tm[__ldg(S.A_rowof + k)] * M.tn[__ldg(S.A_indices + k)];
        }
        for (int i = t; i < m; i += T) M.Dm[i] *= M.tm[i];
        for (int j = t; j < n; j += T) M.En[j] *= M.tn[j];
        __syncthreads();
        SUB_STAMP(pi, 18);
      }
      if (DENSE && n <= 128 && st.ruiz_passes > 0) {   // A^ = D A E in one sweep
        const int lane = t & 31, warp = t >> 5, nw = T >> 5;
        double er[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; er[k] = c < n ? M.En[c] : 0.0; }
        for (int i = warp; i < m; i += nw) {
          const double d = M.Dm[i];
          double *row = M.Av + i * n;
#pragma unroll
          for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; if (c < n) row[c] *= d * er[k]; }
        }
        __syncthreads();
      }
    }
    double sigma;
    {
      double v[4] = {nb0, nc0, 0, 0};
      for (int i = t; i < m; i += T) { const double q = M.Dm[i] * M.bh[i]; M.bh[i] = q; v[2] = fmax(v[2], fabs(q)); }
      for (int j = t; j < n; j += T) { const double q = M.En[j] * M.ch[j]; M.ch[j] = q; v[3] = fmax(v[3], fabs(q)); }
      block_reduce<4, true>(v, M.red);
      nb0 = v[0]; nc0 = v[1];
      sigma = fmax(v[2], v[3]);
      sigma = (!st.normalize || sigma < 1e-6) ? 1.0 : 1.0 / sigma;
      for (int i = t; i < m; i += T) M.bh[i] *= sigma;
      for (int j = t; j < n; j += T) M.ch[j] *= sigma;
      __syncthreads();
    }

    pt.stamp(1);   // equilibration + sigma
    double scale = st.scale, gRg = 0;
    int status = BCONE_INACCURATE, it = 0;
    bool okf = factor_and_g<DENSE, INDIRECT>(a, M, Pg, scale, rho_x, gRg, plA, plN);
    for (int k = t; k < N; k += T) { M.w[k] = (k == N - 1) ? 1.0 : 0.0; M.u[k] = 0; M.ut[k] = 0; }
    if (a.x0) {
      // Warm start (SURVEY.md 8f.2; the reference exposes it for one backend only, torch/cvxpylayer.py:464-487): start the
      // splitting at the fixed point a previous solution (x0, y0, s0) would be for this instance -- w = u + R^{-1} v with
      // u = (x0 sigma / E, y0 sigma / D, 1), v_y = s0 D sigma (the inverse of the write-back below at tau = 1).
      // A row with a non-finite value (the NaN rows of a non-solved instance) starts cold: from it tau never turns positive.
      const double *x0 = a.x0 + (size_t)inst * n, *y0 = a.y0 + (size_t)inst * m, *s0 = a.s0 + (size_t)inst * m;
      bool bad = false;
      for (int j = t; j < n; j += T) bad |= !isfinite(x0[j]);
      for (int i = t; i < m; i += T) bad |= !isfinite(y0[i]) || !isfinite(s0[i]);
      if (!__syncthreads_or(bad)) {
        for (int j = t; j < n; j += T) M.w[j] = x0[j] * sigma / M.En[j];
        for (int i = t; i < m; i += T) M.w[n + i] = y0[i] * sigma / M.Dm[i] + s0[i] * M.Dm[i] * sigma * inv_ry(S, i, scale);
      }
    }
    if (INDIRECT) for (int j = t; j < n; j += T) M.cx[j] = 0.0;
    __syncthreads();
    pt.stamp(2);   // K formation + Cholesky + inverse + g
    double sum_log = 0, rp = nan(""), rd = nan(""), gap = nan("");
    int n_log = 0, last_up = 0;
    // adaptive check schedule (oracle: cone_oracle.c): log-linear extrapolation of the distance to the tolerance
    int next_check = st.check_interval < 10 ? st.check_interval : 10, prev_it = 0;
    double prev_lr = 0;
    if (!okf) status = BCONE_FAILED;
    // Anderson acceleration of w (common.cuh; oracle: aa_apply / aa_safeguard in cone_oracle.c)
    const int aa_lb = a.aa_ws ? st.acceleration_lookback : 0, aa_iv = st.acceleration_interval > 0 ? st.acceleration_interval : 1;
    double *const aaw = aa_lb ? a.aa_ws + (size_t)blockIdx.x * a.aa_stride : nullptr;
    const AaIter aait{M.w, n, M.w + n, m, M.w + N - 1};
    if (aa_lb) aa_reset_dev(aaw);

    for (it = 1; okf && it <= st.max_iters; it++) {
      const bool aa_now = aa_lb && it > 1 && (it - 1) % aa_iv == 0;
      if (aa_now) aa_apply_dev(aaw, aa_lb, aait, M.red + 128, M.red, M.part);
      if (aa_lb && (aa_now || it % aa_iv == 0)) { aa_store_prev(aaw, aa_lb, aait, M.w[N - 1]); __syncthreads(); }
      // ---- affine step ----
      const double w_tau = M.w[N - 1];   // read before anything of this iteration can overwrite it
      double d4[4] = {0, 0, 0, 0};       // mu'g, p'Rg, p'Rp, p'mu  (R-weighted; accumulated in the product epilogues)
      auto dots = [&](double r, double pk, double wk, double gk) {
        d4[0] = fma(r * wk, gk, d4[0]); d4[1] = fma(r * pk, gk, d4[1]);
        d4[2] = fma(r * pk, pk, d4[2]); d4[3] = fma(r * pk, wk, d4[3]);
      };
      SUB_SKIP(pi);
      AT_mul<DENSE>(S, M.Av, M.w + n, M.part, [&](int j, double v) { M.tn[j] = rho_x * M.w[j] - v; }, plA, wide);
      SUB_STAMP(pi, 23);
      if (INDIRECT) {
        // warm start from the previous p_x = ut_x + tau~ g_x; tolerance tightens with the iteration count
        double nr[1] = {0};
        for (int j = t; j < n; j += T) { nr[0] = fma(M.tn[j], M.tn[j], nr[0]); M.ut[j] = M.cx[j]; }
        block_reduce<1, false>(nr, M.red);
        const double tol = fmax(1e-13, fmin(1e-6, 0.1 / pow((double)it, 1.5))) * fmax(1.0, sqrt(nr[0]));
        cg_solve<DENSE>(a, M, Pg, scale, rho_x, M.tn, M.ut, tol, 4 * n, plA, plN);
        for (int j = t; j < n; j += T) { const double pk = M.ut[j]; M.cx[j] = pk; dots(rho_x, pk, M.w[j], M.g[j]); }   // keep p_x for the next warm start
        __syncthreads();
      } else {
        matvec_rows(M.Li, PackedLowerLayout{}, n, n, M.tn, [&](int i, double v) { M.tn2[i] = v; });
        __syncthreads();
        SUB_STAMP(pi, 24);
        matvec_cols(M.Li, PackedLowerLayout{}, n, n, M.tn2, M.part, [&](int j, double v) { M.ut[j] = v; dots(rho_x, v, M.w[j], M.g[j]); }, plN);
        SUB_STAMP(pi, 25);
      }
      A_mul<DENSE>(S, M.Av, M.ut, [&](int i, double v) {
        const double iry = inv_ry(S, i, scale), wk = M.w[n + i], pk = wk + v * iry;
        M.ut[n + i] = pk; dots(1.0 / iry, pk, wk, M.g[n + i]); }, wide);
      SUB_STAMP(pi, 26);
      block_reduce<4, false>(d4, M.red);   // (its barriers also publish ut)
      SUB_STAMP(pi, 27);
      const double qa = dtau + gRg, qb = d4[0] - 2.0 * d4[1] - dtau * w_tau, qc = d4[2] - d4[3];
      double disc = qb * qb - 4.0 * qa * qc;
      if (disc < 0) disc = 0;
      const double tau_t = (-qb + sqrt(disc)) / (2.0 * qa);
      const bool check = st.adaptive_check ? (it >= next_check || it == st.max_iters) : ((it % st.check_interval == 0) || it == st.max_iters);
      // ---- cone step + relaxation (fused when the cone is polyhedral and no check is due) ----
      const bool nonpoly = S.ncones + S.ep + S.ed > 0;
      const bool fused = !nonpoly && !check;
      for (int k = t; k < N; k += T) {
        const double utk = (k == N - 1) ? tau_t : M.ut[k] - tau_t * M.g[k];
        const double wk = M.w[k];
        double uk = 2.0 * utk - wk;
        if (k >= n + S.z && k < n + S.z + S.l) uk = fmax(uk, 0.0);
        if (k == N - 1) uk = fmax(uk, 0.0);
        M.ut[k] = utk; M.u[k] = uk;
        if (fused) M.w[k] = wk + alpha * (uk - utk);
      }
      __syncthreads();
      if (nonpoly) { project_cones(S, M.u + n, M.psd, it > 1); __syncthreads(); }

      SUB_STAMP(pi, 28);
      pt.stamp(3);   // iteration body
      if (check) {
        // ---- termination quantities on the un-normalised data (SURVEY.md 8a F6) ----
        const double tau = M.u[N - 1];
        A_mul<DENSE>(S, M.Av, M.u, [&](int i, double v) { M.tm[i] = v; }, wide);
        AT_mul<DENSE>(S, M.Av, M.u + n, M.part, [&](int j, double v) { M.tn[j] = v; }, plA, wide);
        for (int j = t; j < n; j += T) { M.tn2[j] = 0.0; M.tn3[j] = M.En[j] * M.u[j]; }
        __syncthreads();
        if (Pg) {  // P^ u_x = E (P (E u_x)); no atomics
          P_mul(S, Pg, M.tn3, M.part, [&](int j, double v) { M.tn2[j] += v; }, plN);
          for (int j = t; j < n; j += T) M.tn2[j] *= M.En[j];
          __syncthreads();
        }
        double sm[3] = {0, 0, 0};   // xPx_u, ctx_u, bty_u
        double mx[7] = {0, 0, 0, 0, 0, 0, 0};  // rp, nAx, nS, nAxs, rd, nPx, nATy
        for (int i = t; i < m; i += T) {
          const int k = n + i;
          const double rsk = (M.u[k] - (2.0 * M.ut[k] - M.w[k])) / inv_ry(S, i, scale);
          const double sc = 1.0 / (M.Dm[i] * sigma), ax = M.tm[i];
          mx[0] = fmax(mx[0], fabs(ax + rsk - M.bh[i] * tau) * sc);
          mx[1] = fmax(mx[1], fabs(ax) * sc); mx[2] = fmax(mx[2], fabs(rsk) * sc);
          mx[3] = fmax(mx[3], fabs(ax + rsk) * sc);
          sm[2] = fma(M.bh[i], M.u[k], sm[2]);
        }
        for (int j = t; j < n; j += T) {
          const double sc = 1.0 / (M.En[j] * sigma), px = M.tn2[j], aty = M.tn[j];
          mx[4] = fmax(mx[4], fabs(px + aty + M.ch[j] * tau) * sc);
          mx[5] = fmax(mx[5], fabs(px) * sc); mx[6] = fmax(mx[6], fabs(aty) * sc);
          sm[0] = fma(M.u[j], px, sm[0]); sm[1] = fma(M.ch[j], M.u[j], sm[1]);
        }
        block_reduce<3, false>(sm, M.red);
        block_reduce<7, true>(mx, M.red);
        const double s2 = sigma * sigma;
        bool done = false;
        if (tau > 1e-12) {
          const double itau = 1.0 / tau;
          const double xPx = sm[0] * itau * itau / s2, ctx = sm[1] * itau / s2, bty = sm[2] * itau / s2;
          rp = mx[0] * itau; rd = mx[4] * itau; gap = fabs(xPx + ctx + bty);
          const double np_ = fmax(fmax(mx[1] * itau, mx[2] * itau), nb0);
          const double nd_ = fmax(fmax(mx[5] * itau, mx[6] * itau), nc0);
          const double tp = st.eps_abs + st.eps_rel * np_, td = st.eps_abs + st.eps_rel * nd_;
          const double tg = st.eps_abs + st.eps_rel * fmax(fmax(fabs(xPx), fabs(ctx)), fabs(bty));
          if (rp <= tp && rd <= td && gap <= tg) { status = BCONE_SOLVED; done = true; }
          else if (st.adaptive_check) {
            const double lr = log(fmax(fmax(rp / tp, rd / td), gap / tg));
            int step = st.check_interval;
            if (prev_it > 0 && lr < prev_lr) { const double need = lr * (it - prev_it) / (prev_lr - lr); step = (int)ceil(0.9 * need) + 1; }
            step = max(3, min(step, st.check_interval));
            prev_it = it; prev_lr = lr; next_check = it + step;
          }
          if (!done && st.adaptive_scale) {
            const double relp = rp / fmax(np_, 1e-18), reld = rd / fmax(nd_, 1e-18);
            if (relp > 0 && reld > 0) { sum_log += log(relp) - log(reld); n_log++; }
          }
        }
        if (st.adaptive_check && next_check <= it) next_check = it + st.check_interval;
        if (!done) {
          const double bty_c = sm[2] / s2, ctx_c = sm[1] / s2;
          if (bty_c < 0 && mx[6] / (-bty_c) <= st.eps_infeas) { status = BCONE_INFEASIBLE; done = true; }
          else if (ctx_c < 0 && fmax(mx[5], mx[3]) / (-ctx_c) <= st.eps_infeas) { status = BCONE_UNBOUNDED; done = true; }
        }
        if (done) break;
        if (st.adaptive_scale && n_log > 0 && it - last_up >= BC_RESCALE_MIN_ITERS) {
          const double fac = sqrt(exp(sum_log / n_log));
          if (fac > 3.1622776601683795 || fac < 0.31622776601683794) {
            const double ns = fmin(fmax(scale * fac, BC_MIN_SCALE), BC_MAX_SCALE);
            if (ns != scale) {
              // keep R (w + u - 2 u~) invariant across the metric change (y block only)
              const double ratio = ns / scale;  // r_old / r_new
              for (int i = t; i < m; i += T) {
                const int k = n + i;
                M.w[k] = ratio * (M.w[k] + M.u[k] - 2.0 * M.ut[k]) + 2.0 * M.ut[k] - M.u[k];
              }
              scale = ns;
              __syncthreads();
              okf = factor_and_g<DENSE, INDIRECT>(a, M, Pg, scale, rho_x, gRg, plA, plN);
              if (!okf) { status = BCONE_FAILED; break; }
              sum_log = 0; n_log = 0; last_up = it;
              if (aa_lb) aa_reset_dev(aaw);   // the fixed-point map changed
            }
          }
        }
      }
      if (check) pt.stamp(4);   // termination check (+ rescale)
      if (!fused && it < st.max_iters) {  // (the last iterate keeps w so that s = R(u - t) is recoverable)
        for (int k = t; k < N; k += T) M.w[k] += alpha * (M.u[k] - M.ut[k]);
        __syncthreads();
      }
      // safeguard after the convergence check: it acts on w, convergence is judged on u
      if (aa_now && it < st.max_iters) aa_safeguard_dev(aaw, aa_lb, aait, M.red);
    }
    if (it > st.max_iters) it = st.max_iters;
    pt.stamp(4);
    // ---- write back ----
    {
      double *xo = a.x + (size_t)inst * n, *yo = a.y + (size_t)inst * m, *so = a.s + (size_t)inst * m;
      // the iteration limit was hit without tau ever turning positive: x / tau would be garbage scaled by 1e12 (the problem
      // is probably infeasible or unbounded but not certified yet).  SCS / diffcp raise here; so does the interface on FAILED.
      if (status == BCONE_INACCURATE && !(M.u[N - 1] > 1e-12) && okf) status = BCONE_FAILED;
      if (status == BCONE_SOLVED || status == BCONE_INACCURATE) {
        double tau = M.u[N - 1];
        if (!(tau > 1e-12)) tau = 1e-12;
        const double k0 = 1.0 / (sigma * tau);
        for (int j = t; j < n; j += T) xo[j] = M.En[j] * M.u[j] * k0;
        for (int i = t; i < m; i += T) {
          const int k = n + i;
          const double rsk = (M.u[k] - (2.0 * M.ut[k] - M.w[k])) / inv_ry(S, i, scale);
          yo[i] = M.Dm[i] * M.u[k] * k0;
          so[i] = rsk * k0 / M.Dm[i];
        }
      } else {
        const double qn = nan("");
        for (int j = t; j < n; j += T) xo[j] = qn;
        for (int i = t; i < m; i += T) { yo[i] = qn; so[i] = qn; }
      }
      if (t == 0) {
        a.status[inst] = status; a.iters[inst] = it;
        if (a.resid) { a.resid[inst * 3 + 0] = rp; a.resid[inst * 3 + 1] = rd; a.resid[inst * 3 + 2] = gap; }
      }
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------- host entry points
extern "C" size_t bc_fwd_smem_bytes(int n, int m, int nnzA, int threads, int max_psd, int indirect, int ns, int nexp, int vals_global) {
  return fwd_smem_doubles(n, m, nnzA, threads, max_psd, indirect, ns, nexp, vals_global) * sizeof(double);
}
// per-CTA slab: the values when they are off chip (nnzA_global > 0), then the vectors, then the packed factor
extern "C" size_t bc_fwd_ws_doubles(int n, int m, int vectors, int with_factor, int nnzA_global) {
  return (((size_t)nnzA_global + 1) & ~(size_t)1) + (vectors ? ((fwd_vec_doubles(n, m, 1) + 1) & ~(size_t)1) : 0) +
         (with_factor ? (((size_t)n * (n + 1) / 2 + 1) & ~(size_t)1) : 0);
}

// The instantiations that exist.  small_cta: the 4-CTA/SM build, direct solve with the values on chip only; vals_global: the
// values-off-chip builds (512-thread only: the tier serves large instances).
extern "C" const void *bc_fwd_kernel(int dense, int indirect, int small_cta, int vals_global) {
  if (small_cta && (indirect || vals_global)) return nullptr;
  if (vals_global) {
    if (dense) return indirect ? (const void *)fwd_kernel<true, true, false, true> : (const void *)fwd_kernel<true, false, false, true>;
    return indirect ? (const void *)fwd_kernel<false, true, false, true> : (const void *)fwd_kernel<false, false, false, true>;
  }
  if (small_cta) return dense ? (const void *)fwd_kernel<true, false, true> : (const void *)fwd_kernel<false, false, true>;
  if (dense) return indirect ? (const void *)fwd_kernel<true, true> : (const void *)fwd_kernel<true, false>;
  return indirect ? (const void *)fwd_kernel<false, true> : (const void *)fwd_kernel<false, false>;
}
