// bwd.cu -- backward kernel: adjoint of the cone-program solution map (what the reference gets
// from diffcp's adjoint closure at src/cvxpylayers/interfaces/diffcp_if.py:86; rows B1-B4 of
// SURVEY.md section 8a).  One persistent CTA per instance:
//   v = y - s, pi_y = Pi_{K*}(v), D = DPi_{K*}(v)           (cone Jacobian, block diagonal)
//   dz = [dx ; D dy ; -(x'dx + y'dy)]                        (ds = 0, diffcp_if.py:84)
//   r  = LSQR(M', dz),  M = (DQ - I) blkdiag(I, D, 1) + I    (Paige-Saunders, SciPy stopping rules)
//   dA_ij = x_j r_{n+i} - pi_y,i r_j  on EVERY structural entry;  db = pi_y r_tau - r_y;
//   dc = x r_tau - r_x;  dP_ij = (r_tau x_i - r_x,i) x_j (+ transpose term off the diagonal)
// The instance's CSR values are staged once by TMA and stay in shared memory for all LSQR
// iterations (each applies A and A' twice); P values are read from L2.  Values that do not fit on chip are read in place from
// A_vals instead (bwd_kernel<.., VG = true>).
// The same kernel with JVP = true is the forward-mode derivative (bcone_jvp), the transpose of the above.
#include "common.cuh"

struct BwdSmem {
  double *Av, *Pv, *x, *piy, *v, *b, *c, *px2c, *U, *V, *W, *X, *t1, *t2, *Lsc, *Rsc, *tin, *part, *red, *psdVL, *psdscr, *expJ;
  uint64_t *bar;
  int *ibuf;
};

// v is only kept for the non-polyhedral rows (nonneg rows use pi_y > 0 <=> v > 0 as their mask).  LSMR keeps one more N-vector,
// solution refinement (refine.cu) the iterate x, v, its pi_y and the y rows of its residual.
__host__ __device__ inline size_t bwd_vec_doubles(int n, int m, int npoly, int lsmr = 0, int refine = 0) {
  size_t N = (size_t)n + m + 1;
  return 3 * (size_t)n + 2 * (size_t)m + (m - npoly) + (lsmr ? 8 : 7) * N + 2 * (size_t)m + (refine ? (size_t)n + 3 * (size_t)m : 0);
}
// vec_global: large instances keep the LSQR vectors in a per-CTA slab of global memory.
// vals_global: the CSR values are read in place from the caller's A_vals (instances whose values do not fit on chip).
__host__ __device__ inline size_t bwd_smem_doubles(int n, int m, int npoly, int nnzA, int nnzP_smem, int threads, int max_psd, int psd_total, int nexp, int vec_global,
                                                   int vals_global, int lsmr = 0, int refine = 0) {
  size_t d = 4 + (vals_global ? 0 : ((size_t)nnzA + 1) & ~(size_t)1) + (((size_t)nnzP_smem + 1) & ~(size_t)1) + threads + 2 * 32;
  if (!vec_global) d += bwd_vec_doubles(n, m, npoly, lsmr, refine);
  if (max_psd > 0) d += psd_total + (size_t)(threads / 32) * (3 * (size_t)max_psd * max_psd + max_psd);
  return d + 9 * (size_t)nexp;
}

// VG: no shared memory for the values (M.Av is set per instance); LSMR: one more N-vector behind t2 (LSMR's h-bar; not a
// member of BwdSmem, whose layout the LSQR kernels' code depends on); REFINE: n + 3m doubles behind t2 (refine.cu)
template <bool VG = false, bool LSMR = false, bool REFINE = false>
__device__ __forceinline__ void carve_b(BwdSmem &M, double *base, double *gws, int n, int m, int npoly, int nnzA, int nnzP_smem, int threads, int max_psd, int psd_total, int nexp) {
  const int N = n + m + 1;
  double *q = base;
  M.bar = (uint64_t *)q; q += 2;
  M.ibuf = (int *)q; q += 2;
  if (VG) M.Av = nullptr;
  else { M.Av = q; q += (nnzA + 1) & ~1; }
  M.Pv = q; q += (nnzP_smem + 1) & ~1;
  M.part = q; q += threads; M.red = q; q += 2 * 32;
  double *v = gws ? gws : q;
  M.x = v; v += n; M.c = v; v += n; M.px2c = v; v += n;
  M.piy = v; v += m; M.b = v; v += m;
  M.v = v - npoly; v += m - npoly;  // indexed by the original row i >= npoly
  M.U = v; v += N; M.V = v; v += N; M.W = v; v += N; M.X = v; v += N;
  M.Lsc = v; v += N; M.Rsc = v; v += N; M.tin = v; v += N;
  M.t1 = v; v += m; M.t2 = v; v += m;
  if (LSMR) v += N;
  if (REFINE) v += n + 3 * m;
  if (!gws) q = v;
  M.expJ = q; q += 9 * nexp;
  M.psdVL = q; q += psd_total;
  M.psdscr = q;
}

// out_y = D in_y  (D = DPi_{K*}(v)); zero rows identity, nonneg rows mask, SOC closed form,
// PSD  V (B o (V' dX V)) V'  with V, lambda precomputed in psdVL.  Ends with __syncthreads().
__device__ __forceinline__ void apply_D(const DevStruct &S, const BwdSmem &M, const double *in, double *out) {
  const int T = blockDim.x, t = threadIdx.x, pl = S.z + S.l;
  for (int i = t; i < pl; i += T) out[i] = (i < S.z || M.piy[i] > 0) ? in[i] : 0.0;
  if (S.ncones > 0) {
    const int lane = t & 31, warp = t >> 5, nw = T >> 5;
    int psd_off = 0;
    for (int cb = 0; cb < S.ncones; cb++) {
      const int ty = __ldg(S.cone_type + cb), s0 = __ldg(S.cone_start + cb), sz = __ldg(S.cone_size + cb);
      const int k = __ldg(S.cone_order + cb);
      const int my_off = psd_off;
      if (ty == BC_CPSD) psd_off += k * k + k;
      if (cb % nw != warp) continue;
      const double *vb = M.v + s0, *ib = in + s0;
      double *ob = out + s0;
      if (ty == BC_CSOC) {
        if (sz == 1) { if (lane == 0) ob[0] = vb[0] > 0 ? ib[0] : 0.0; continue; }
        double ss = 0, xd = 0;
        for (int i = 1 + lane; i < sz; i += 32) { ss = fma(vb[i], vb[i], ss); xd = fma(vb[i], ib[i], xd); }
        ss = warp_sum(ss); xd = warp_sum(xd);
        const double nx = sqrt(ss), tt = vb[0], d0 = ib[0];
        if (nx <= tt) { for (int i = lane; i < sz; i += 32) ob[i] = ib[i]; }
        else if (nx <= -tt) { for (int i = lane; i < sz; i += 32) ob[i] = 0.0; }
        else {
          const double h = 0.5 / nx;
          for (int i = 1 + lane; i < sz; i += 32) ob[i] = (vb[i] * d0 + (tt + nx) * ib[i] - tt * vb[i] * xd / (nx * nx)) * h;
          if (lane == 0) ob[0] = 0.5 * (d0 + xd / nx);
        }
      } else {
        const double *Vm = M.psdVL + my_off, *lam = Vm + k * k;
        double *Xd = M.psdscr + warp * (3 * S.max_psd * S.max_psd + S.max_psd), *T1 = Xd + k * k, *T2 = T1 + k * k;
        svec_to_mat_warp(k, ib, Xd);
        __syncwarp();
        if (k <= 16) {   // the two congruences V' . V and V . V' on the FP64 tensor cores (DMMA.8x8x4, common.cuh warp_mm16)
          auto inb = [&](int i, int j) { return i < k && j < k; };
          warp_mm16(k, [&](int i, int q) { return inb(i, q) ? Xd[i * k + q] : 0.0; }, [&](int q, int j) { return inb(q, j) ? Vm[q * k + j] : 0.0; },
                    [&](int i, int j, double val) { if (inb(i, j)) T1[i * k + j] = val; });                       // T1 = Xd V
          __syncwarp();
          warp_mm16(k, [&](int i, int q) { return inb(i, q) ? Vm[q * k + i] : 0.0; }, [&](int q, int j) { return inb(q, j) ? T1[q * k + j] : 0.0; },
                    [&](int i, int j, double val) {                                                                // T2 = B o (V' T1)
                      if (!inb(i, j)) return;
                      const double li = lam[i], lj = lam[j];
                      double bij;
                      if (li > 0 && lj > 0) bij = 1.0; else if (li <= 0 && lj <= 0) bij = 0.0;
                      else { const double lp = li > 0 ? li : lj, ln = li > 0 ? lj : li; bij = lp / (lp - ln); }
                      T2[i * k + j] = val * bij; });
          __syncwarp();
          warp_mm16(k, [&](int i, int q) { return inb(i, q) ? Vm[i * k + q] : 0.0; }, [&](int q, int j) { return inb(q, j) ? T2[q * k + j] : 0.0; },
                    [&](int i, int j, double val) { if (inb(i, j)) T1[i * k + j] = val; });                       // T1 = V T2
          __syncwarp();
          warp_mm16(k, [&](int i, int q) { return inb(i, q) ? T1[i * k + q] : 0.0; }, [&](int q, int j) { return inb(q, j) ? Vm[j * k + q] : 0.0; },
                    [&](int i, int j, double val) { if (inb(i, j)) Xd[i * k + j] = val; });                       // Xd = T1 V'
          __syncwarp();
          mat_to_svec_warp(k, Xd, ob);
          continue;
        }
        for (int e = lane; e < k * k; e += 32) {  // T1 = Xd V
          const int i = e / k, j = e % k; double acc = 0;
          for (int q = 0; q < k; q++) acc = fma(Xd[i * k + q], Vm[q * k + j], acc);
          T1[e] = acc;
        }
        __syncwarp();
        for (int e = lane; e < k * k; e += 32) {  // T2 = B o (V' T1)
          const int i = e / k, j = e % k; double acc = 0;
          for (int q = 0; q < k; q++) acc = fma(Vm[q * k + i], T1[q * k + j], acc);
          const double li = lam[i], lj = lam[j];
          double bij;
          if (li > 0 && lj > 0) bij = 1.0; else if (li <= 0 && lj <= 0) bij = 0.0;
          else { const double lp = li > 0 ? li : lj, ln = li > 0 ? lj : li; bij = lp / (lp - ln); }
          T2[e] = acc * bij;
        }
        __syncwarp();
        for (int e = lane; e < k * k; e += 32) {  // T1 = V T2
          const int i = e / k, j = e % k; double acc = 0;
          for (int q = 0; q < k; q++) acc = fma(Vm[i * k + q], T2[q * k + j], acc);
          T1[e] = acc;
        }
        __syncwarp();
        for (int e = lane; e < k * k; e += 32) {  // Xd = T1 V'
          const int i = e / k, j = e % k; double acc = 0;
          for (int q = 0; q < k; q++) acc = fma(T1[i * k + q], Vm[j * k + q], acc);
          Xd[e] = acc;
        }
        __syncwarp();
        mat_to_svec_warp(k, Xd, ob);
      }
    }
  }
  for (int e = t; e < S.ep + S.ed; e += T) {
    const double *J = M.expJ + 9 * e, *ib = in + S.exp_start + 3 * e;
    double *ob = out + S.exp_start + 3 * e;
    const double i0 = ib[0], i1 = ib[1], i2 = ib[2];
    ob[0] = J[0] * i0 + J[1] * i1 + J[2] * i2; ob[1] = J[3] * i0 + J[4] * i1 + J[5] * i2; ob[2] = J[6] * i0 + J[7] * i1 + J[8] * i2;
  }
  __syncthreads();
}

// out += sc o (M' in)   (B = M' is the LSQR system matrix; sc = left scaling or nullptr).  in/out length N.
template <bool DENSE>
__device__ __forceinline__ void op_MT(const BwdArgs &a, const BwdSmem &M, const double *Pg, double xPx,
                                      const double *in, double *out, const double *sc, const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  const double it = in[n + m];
  // x rows: -A' in_y + P in_x - (2Px + c) in_tau
  AT_mul<DENSE>(S, M.Av, in + n, M.part, [&](int j, double v) { out[j] += (sc ? sc[j] : 1.0) * (-v - M.px2c[j] * it); }, plA);
  if (Pg) P_mul(S, Pg, in, M.part, [&](int j, double v) { out[j] += (sc ? sc[j] : 1.0) * v; }, plN);
  // t1_y = A in_x - b in_tau - in_y ; y rows: D t1_y + in_y
  A_mul<DENSE>(S, M.Av, in, [&](int i, double v) { M.t1[i] = v - M.b[i] * it - in[n + i]; });
  double d2[2] = {0, 0};
  for (int j = t; j < n; j += T) d2[0] = fma(M.c[j], in[j], d2[0]);
  for (int i = t; i < m; i += T) d2[1] = fma(M.b[i], in[n + i], d2[1]);
  block_reduce<2, false>(d2, M.red);  // (syncs: t1 complete)
  apply_D(S, M, M.t1, M.t2);
  for (int i = t; i < m; i += T) out[n + i] += (sc ? sc[n + i] : 1.0) * (M.t2[i] + in[n + i]);
  if (t == 0) out[n + m] += (sc ? sc[n + m] : 1.0) * (d2[0] + d2[1] + xPx * it);
  __syncthreads();
}

// out += sc o (M in)
template <bool DENSE>
__device__ __forceinline__ void op_M(const BwdArgs &a, const BwdSmem &M, const double *Pg, double xPx,
                                     const double *in, double *out, const double *sc, const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  const double it = in[n + m];
  apply_D(S, M, in + n, M.t2);  // t2 = D in_y
  // x rows: A' t2 + P in_x + c in_tau
  AT_mul<DENSE>(S, M.Av, M.t2, M.part, [&](int j, double v) { out[j] += (sc ? sc[j] : 1.0) * (v + M.c[j] * it); }, plA);
  if (Pg) P_mul(S, Pg, in, M.part, [&](int j, double v) { out[j] += (sc ? sc[j] : 1.0) * v; }, plN);
  // y rows: -A in_x + b in_tau - t2 + in_y
  A_mul<DENSE>(S, M.Av, in, [&](int i, double v) { out[n + i] += (sc ? sc[n + i] : 1.0) * (-v + M.b[i] * it - M.t2[i] + in[n + i]); });
  double d2[2] = {0, 0};
  for (int j = t; j < n; j += T) d2[0] = fma(M.px2c[j], in[j], d2[0]);
  for (int i = t; i < m; i += T) d2[1] = fma(M.b[i], M.t2[i], d2[1]);
  block_reduce<2, false>(d2, M.red);
  if (t == 0) out[n + m] += (sc ? sc[n + m] : 1.0) * (-d2[0] - d2[1] + xPx * it);
  __syncthreads();
}

// 2-norm Ruiz scaling of a 0/1-skeleton surrogate of M' (see oracle/cone_oracle.c lsqr_equilibrate):
// Lsc / Rsc <- left / right diagonal scalings; inactive nonneg rows get 0 (their unknown is dz_i = 0).
// Row / column sums of squares need four products with the elementwise-squared A per pass.
template <bool DENSE>
__device__ void equilibrate(const BwdArgs &a, const BwdSmem &M, const double *Pg, double xPx, int passes,
                            const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, N = n + m + 1, T = blockDim.x, t = threadIdx.x;
  const int lo = S.z, hi = S.z + S.l;
  double *L = M.Lsc, *R = M.Rsc, *rs = M.V, *cs = M.W, *sq = M.X;  // V, W, X are free before LSQR starts
  for (int k = t; k < N; k += T) {
    double v = 1.0;
    if (k >= n && k < n + m) { const int i = k - n; if (i >= lo && i < hi && !(M.piy[i] > 0)) v = 0.0; }
    L[k] = v; R[k] = v;
  }
  __syncthreads();
  for (int pass = 0; pass < passes; pass++) {
    const double Lt = L[N - 1], Rt = R[N - 1];
    // ---- vector terms + tau row / column (reductions) ----
    double s4[2] = {0, 0};  // rs[tau], cs[tau]
    for (int j = t; j < n; j += T) {
      const double e1 = M.px2c[j] * M.px2c[j] * L[j] * L[j] * Rt * Rt;
      const double e2 = M.c[j] * M.c[j] * Lt * Lt * R[j] * R[j];
      rs[j] = e1; cs[j] = e2; s4[1] += e1; s4[0] += e2;
    }
    for (int i = t; i < m; i += T) {
      const int k = n + i;
      const double b2 = M.b[i] * M.b[i];
      const double e1 = b2 * L[k] * L[k] * Rt * Rt, e2 = b2 * Lt * Lt * R[k] * R[k];
      const double e3 = (i >= hi ? 1.0 : 0.0) * L[k] * L[k] * R[k] * R[k];
      rs[k] = e1 + e3; cs[k] = e2 + e3; s4[1] += e1; s4[0] += e2;
    }
    block_reduce<2, false>(s4, M.red);
    const double ett = xPx * xPx * Lt * Lt * Rt * Rt;
    // ---- A block: four products with A.^2 ----
    for (int k = t; k < N; k += T) sq[k] = R[k] * R[k];
    __syncthreads();
    AT_mul<DENSE, true>(S, M.Av, sq + n, M.part, [&](int j, double v) { rs[j] += v * L[j] * L[j]; }, plA);       // (x-row j, y-col i)
    A_mul<DENSE, true>(S, M.Av, sq, [&](int i, double v) { rs[n + i] += v * L[n + i] * L[n + i]; });          // (y-row i, x-col j)
    __syncthreads();
    for (int k = t; k < N; k += T) sq[k] = L[k] * L[k];
    __syncthreads();
    A_mul<DENSE, true>(S, M.Av, sq, [&](int i, double v) { cs[n + i] += v * R[n + i] * R[n + i]; });          // (x-row j, y-col i)
    AT_mul<DENSE, true>(S, M.Av, sq + n, M.part, [&](int j, double v) { cs[j] += v * R[j] * R[j]; }, plA);         // (y-row i, x-col j)
    if (Pg) {  // P.^2 block (x rows, x cols): rs_i += L_i^2 (P.^2 R_x^2)_i ; cs_j += R_j^2 (P.^2 L_x^2)_j
      P_mul<true>(S, Pg, sq, M.part, [&](int j, double v) { cs[j] += v * R[j] * R[j]; }, plN);
      for (int k = t; k < n; k += T) sq[k] = R[k] * R[k];
      __syncthreads();
      P_mul<true>(S, Pg, sq, M.part, [&](int j, double v) { rs[j] += v * L[j] * L[j]; }, plN);
    }
    __syncthreads();
    for (int k = t; k < N; k += T) {
      const double r = (k == N - 1) ? s4[0] + ett : rs[k], c = (k == N - 1) ? s4[1] + ett : cs[k];
      if (L[k] > 0 && r > 1e-300) L[k] /= sqrt(sqrt(r));
      if (R[k] > 0 && c > 1e-300) R[k] /= sqrt(sqrt(c));
    }
    __syncthreads();
  }
}

// U <- g = [-dA' pi_y - dc - dP x ; dA x - db ; pi_y'db + x'dc + x'dP x] for the data tangents of instance `inst`
// (read from global memory; W holds dP x on the way).  Returns max|g| (block-uniform).  Starts with a barrier.
// Not inlined: it runs once per instance, and inlined its products raise the spill of the LSQR loop.
template <bool DENSE>
__device__ __noinline__ double jvp_rhs(const BwdArgs &a, const BwdSmem &M, int inst, const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  const double *tAg = a.tA + (size_t)inst * a.sA, *tbg = a.tb + (size_t)inst * m, *tcg = a.tc + (size_t)inst * n;
  const double *tPg = (a.tP && S.nnzP > 0) ? a.tP + (size_t)inst * a.sP : nullptr;
  for (int j = t; j < n; j += T) { M.U[j] = -tcg[j]; M.W[j] = 0.0; }
  __syncthreads();
  AT_mul<DENSE>(S, tAg, M.piy, M.part, [&](int j, double v) { M.U[j] -= v; }, plA);
  if (tPg) P_mul(S, tPg, M.x, M.part, [&](int j, double v) { M.W[j] += v; }, plN);
  A_mul<DENSE>(S, tAg, M.x, [&](int i, double v) { M.U[n + i] = v - tbg[i]; });
  __syncthreads();
  double d2[2] = {0, 0};
  for (int j = t; j < n; j += T) {
    const double w = M.W[j];
    M.U[j] -= w; d2[0] = fma(M.x[j], w + tcg[j], d2[0]); d2[1] = fmax(d2[1], fabs(M.U[j]));
  }
  for (int i = t; i < m; i += T) { d2[0] = fma(M.piy[i], tbg[i], d2[0]); d2[1] = fmax(d2[1], fabs(M.U[n + i])); }
  double s1[1] = {d2[0]}; block_reduce<1, false>(s1, M.red);
  double m1[1] = {d2[1]}; block_reduce<1, true>(m1, M.red);
  if (t == 0) M.U[n + m] = s1[0];
  return fmax(m1[0], fabs(s1[0]));
}

// The equilibrated solve drops the unknown z_{n+i} of an inactive nonneg row together with its equation (row n+i of M is
// [-A_i, e_i', b_i] and z_{n+i} appears nowhere else); dx and dy do not need it, ds does: recover it from that equation,
// z_{n+i} = (dA x - db)_i + (A z_x)_i - b_i z_tau.  Ends with a barrier.
template <bool DENSE>
__device__ __noinline__ void jvp_inactive_rows(const BwdArgs &a, const BwdSmem &M, int inst) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, lo = S.z, hi = S.z + S.l;
  const double *tAg = a.tA + (size_t)inst * a.sA, *tbg = a.tb + (size_t)inst * m;
  const double zt = M.X[n + m];
  auto inactive = [&](int i) { return i >= lo && i < hi && !(M.piy[i] > 0); };
  A_mul<DENSE>(S, M.Av, M.X, [&](int i, double v) { if (inactive(i)) M.t1[i] = v - M.b[i] * zt; });
  __syncthreads();
  A_mul<DENSE>(S, tAg, M.x, [&](int i, double v) { if (inactive(i)) M.X[n + i] = M.t1[i] + v - tbg[i]; });
  __syncthreads();
}

#ifdef BC_REFINE
// Solution refinement (refine.cu): U <- -R at the point in x, pi_y (v = vw + alpha z_y on the polyhedral rows, M.v elsewhere),
//   R = [P x + A' pi_y + c ;  b - A x - (pi_y - v) ;  -(x'P x + c'x + b'pi_y)],
// the residual map of the homogeneous embedding at tau = 1.  Returns ||R||_2^2 (block-uniform).  W holds P x on the way.
template <bool DENSE>
__device__ __noinline__ double refine_rhs(const BwdArgs &a, const BwdSmem &M, const double *Pg, const double *vw, double alpha,
                                          const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x, npoly = S.z + S.l;
  for (int j = t; j < n; j += T) M.W[j] = 0.0;
  __syncthreads();
  AT_mul<DENSE>(S, M.Av, M.piy, M.part, [&](int j, double v) { M.U[j] = -(v + M.c[j]); }, plA);
  if (Pg) P_mul(S, Pg, M.x, M.part, [&](int j, double v) { M.W[j] += v; }, plN);
  A_mul<DENSE>(S, M.Av, M.x, [&](int i, double v) {
    const double vi = i >= npoly ? M.v[i] : fma(alpha, M.X[n + i], vw[i]);
    M.U[n + i] = v + M.piy[i] - vi - M.b[i]; });
  __syncthreads();
  double d2[2] = {0, 0};   // tau component, ||R_x||^2 + ||R_y||^2
  for (int j = t; j < n; j += T) {
    const double w = M.W[j], u = M.U[j] - w;
    M.U[j] = u; d2[0] = fma(M.x[j], w + M.c[j], d2[0]); d2[1] = fma(u, u, d2[1]);
  }
  for (int i = t; i < m; i += T) { const double u = M.U[n + i]; d2[0] = fma(M.b[i], M.piy[i], d2[0]); d2[1] = fma(u, u, d2[1]); }
  block_reduce<2, false>(d2, M.red);
  if (t == 0) M.U[n + m] = d2[0];
  return fma(d2[0], d2[0], d2[1]);
}

// The equilibrated solve drops an inactive nonneg row's unknown with its equation (as for the forward mode, jvp_inactive_rows):
// recover it from that equation, z_{n+i} = (A z_x)_i - R_{y,i}  (ryw = -R_y; the tau column is masked).  Ends with a barrier.
template <bool DENSE>
__device__ __noinline__ void refine_inactive_rows(const BwdArgs &a, const BwdSmem &M, const double *ryw) {
  const DevStruct &S = a.S;
  const int n = S.n, lo = S.z, hi = S.z + S.l;
  A_mul<DENSE>(S, M.Av, M.X, [&](int i, double v) { if (i >= lo && i < hi && !(M.piy[i] > 0)) M.X[n + i] = v + ryw[i]; });
  __syncthreads();
}

// Polishing's acceptance metrics of the point (x, y, s) (shared or global memory): rp = |A x + s - b|_inf,
// rd = |P x + A'y + c|_inf, gap = |x'P x + c'x + b'y|; NaN counts as inf.  Block-uniform.  Uses V, W, t1.
struct RefMet { double r[3]; };
template <bool DENSE>
__device__ __noinline__ RefMet refine_metrics(const BwdArgs &a, const BwdSmem &M, const double *Pg, const double *x, const double *y,
                                              const double *s, const ColPlan &plA, const ColPlan &plN) {
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  __syncthreads();
  for (int j = t; j < n; j += T) M.W[j] = 0.0;
  A_mul<DENSE>(S, M.Av, x, [&](int i, double v) { M.t1[i] = v; });
  AT_mul<DENSE>(S, M.Av, y, M.part, [&](int j, double v) { M.V[j] = v; }, plA);   // (ends synchronised)
  if (Pg) P_mul(S, Pg, x, M.part, [&](int j, double v) { M.W[j] += v; }, plN);
  __syncthreads();
  auto amax = [](double acc, double v) { const double e = fabs(v); return e == e ? fmax(acc, e) : INFINITY; };
  double mx[2] = {0, 0}, sm[1] = {0};
  for (int i = t; i < m; i += T) { mx[0] = amax(mx[0], M.t1[i] + s[i] - M.b[i]); sm[0] = fma(M.b[i], y[i], sm[0]); }
  for (int j = t; j < n; j += T) { mx[1] = amax(mx[1], M.W[j] + M.V[j] + M.c[j]); sm[0] = fma(x[j], M.W[j] + M.c[j], sm[0]); }
  block_reduce<2, true>(mx, M.red);
  block_reduce<1, false>(sm, M.red);
  return RefMet{{mx[0], mx[1], fabs(sm[0])}};
}
#endif

// JVP: the forward-mode derivative (bcone_jvp) instead of the adjoint -- the exact transpose of the map above:
//   g  = [-dA' pi_y - dc - dP x ; dA x - db ; pi_y'db + x'dc + x'dP x]   (tangents dA, dP, db, dc read from global memory)
//   z  = LSQR(M, g);  dx = z_x - x z_tau,  dy = D z_y - y z_tau,  ds = D z_y - z_y - s z_tau
// The adjoint's gradient assembly is G' and its dz is E'w, so it computes G' M^-T E'w; this computes E M^-1 G.
// VG (values off chip): the instance's values are read in place from A_vals -- this kernel never writes them -- so nothing is
// staged and shared memory holds only the vectors (when they fit) and the cone scratch.
// LSMR: diffcp's mode = "lsmr" (settings.lsmr = 1) -- LSMR (common.cuh lsmr_block) in place of LSQR on the same operator,
// scalings and right-hand side.  bwd_lsmr.cu compiles this file again with BC_LSMR defined: the same kernels with LSMR, named
// bwd_lsmr_kernel, in a translation unit of their own (so that the LSQR kernels compile to the code they had without them).
// REFINE: solution refinement (bcone_refine) -- refine.cu compiles this file with BC_REFINE defined: the forward-mode kernel
// (JVP = true) named refine_kernel, with the residual as its right-hand side, the tau column masked, a Newton loop with a
// line search around set-up and LSQR, and its own write-back.
#if defined(BC_REFINE)
#define BWD_KERNEL refine_kernel
constexpr bool LSMR = false, REFINE = true;
#elif defined(BC_LSMR)
#define BWD_KERNEL bwd_lsmr_kernel
constexpr bool LSMR = true, REFINE = false;
#else
#define BWD_KERNEL bwd_kernel
constexpr bool LSMR = false, REFINE = false;
#endif
template <bool DENSE, bool SMALL = false, bool JVP = false, bool VG = false>   // SMALL: <= 256 threads, four resident CTAs per SM (see fwd.cu)
#ifdef BC_REFINE
__global__ void __launch_bounds__(SMALL ? 256 : 512, SMALL ? 4 : 1) BWD_KERNEL(const __grid_constant__ RefineArgs ra) {
  const BwdArgs &a = ra.a;
#else
__global__ void __launch_bounds__(SMALL ? 256 : 512, SMALL ? 4 : 1) BWD_KERNEL(const __grid_constant__ BwdArgs a) {
#endif
  extern __shared__ __align__(16) double smem[];
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, N = n + m + 1, T = blockDim.x, t = threadIdx.x;
  const bc_settings &st = a.st;
  BwdSmem M;
  carve_b<VG, LSMR, REFINE>(M, smem, a.ws ? a.ws + (size_t)blockIdx.x * a.ws_stride : nullptr, n, m, S.z + S.l, S.nnzA, a.p_in_smem ? S.nnzP : 0, T, S.max_psd,
              a.psd_total, S.ep + S.ed);
  if (t == 0) { mbar_init(M.bar, 1); fence_mbar_init(); }
  __syncthreads();
  uint32_t tma_phase = 0;
  const ColPlan plA = make_colplan(m, n), plN = make_colplan(n, n);
#ifdef BC_REFINE
  // the iterate w = (x, v): x, v, pi_y(v), and -R_y at w (the y rows of the last accepted right-hand side; later s)
  double *const xw = M.t2 + m, *const vw = xw + n, *const yw = vw + m, *const ryw = yw + m;
#endif

  for (;;) {
    if constexpr (LSMR) {   // (also the second pass of the block-preconditioned LSMR adjoint: the instances on its device-side list)
      if (t == 0) {
        const int k = atomicAdd(a.counter, 1), nwork = a.B_dev ? *a.B_dev : a.B;
        M.ibuf[0] = k < nwork ? (a.inst_list ? a.inst_list[k] : k) : a.B;
      }
    } else {
      if (t == 0) M.ibuf[0] = atomicAdd(a.counter, 1);
    }
    __syncthreads();
    const int inst = M.ibuf[0];
    if (inst >= a.B) break;
    const double *Ag = a.A_vals + (size_t)inst * a.sA;
    const double *Pglob = (a.P_vals && S.nnzP > 0) ? a.P_vals + (size_t)inst * a.sP : nullptr;
    const double *Pg = (Pglob && a.p_in_smem) ? M.Pv : Pglob;
    const bool tmaP = a.use_tma && Pglob && a.p_in_smem && (S.nnzP % 2 == 0) && (((uintptr_t)Pglob & 15) == 0);
    if constexpr (VG) {
      M.Av = const_cast<double *>(Ag);   // (read only: the one store to M.Av is the staging below)
      if (tmaP && t == 0) {
        fence_proxy_async();
        mbar_expect_tx(M.bar, (uint32_t)(S.nnzP * sizeof(double)));
        tma_bulk_g2s(M.Pv, Pglob, (uint32_t)(S.nnzP * sizeof(double)), M.bar);
      }
    } else if (a.use_tma) {
      if (t == 0) {
        fence_proxy_async();
        mbar_expect_tx(M.bar, (uint32_t)((S.nnzA + (tmaP ? S.nnzP : 0)) * sizeof(double)));
        tma_bulk_g2s(M.Av, Ag, (uint32_t)(S.nnzA * sizeof(double)), M.bar);
        if (tmaP) tma_bulk_g2s(M.Pv, Pglob, (uint32_t)(S.nnzP * sizeof(double)), M.bar);
      }
    } else {
      for (int k = t; k < S.nnzA; k += T) M.Av[k] = Ag[k];
    }
    if (Pglob && a.p_in_smem && !tmaP) for (int k = t; k < S.nnzP; k += T) M.Pv[k] = Pglob[k];
    const double *dxg = a.dx + (size_t)inst * n, *dyg = a.dy + (size_t)inst * m;
#ifdef BC_REFINE
    // ---- the input: status and finiteness, w = (x, y - s), its acceptance metrics ----
    (void)dyg;
    const double *xg = a.x + (size_t)inst * n, *yg = a.y + (size_t)inst * m, *sg = a.s + (size_t)inst * m;
    bool finite = true;
    for (int j = t; j < n; j += T) { const double v = xg[j]; xw[j] = v; M.c[j] = a.c[(size_t)inst * n + j]; finite &= isfinite(v); }
    for (int i = t; i < m; i += T) {
      const double yi = yg[i], si = sg[i];
      vw[i] = yi - si; M.b[i] = a.b[(size_t)inst * m + i]; finite &= isfinite(yi) && isfinite(si);
    }
    for (int k = t; k < N; k += T) M.X[k] = 0.0;
    if (VG ? tmaP : (bool)a.use_tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }
    finite = __syncthreads_and(finite);
    const int stat = ra.status[inst];
    if ((stat != 1 && stat != 2) || !finite) {
      if (t == 0) ra.flags[inst] = -1;
      continue;
    }
    const RefMet r0 = refine_metrics<DENSE>(a, M, Pg, xg, yg, sg, plA, plN);
    // ---- Newton loop: each pass sets up the trial point w + alpha z (z = M.X; alpha = 0: the input) and takes its residual.
    //      Accepted (the first point, or ||R|| below the iterate's): w <- trial, then LSQR for the next z.  Rejected: alpha halves
    //      down to 1/32, then stop. ----
    double alpha = 0.0, rn_w = 0.0;
    int steps = 0;
    bool have_w = false;
    for (;;) {
    for (int j = t; j < n; j += T) { M.x[j] = fma(alpha, M.X[j], xw[j]); M.px2c[j] = 0.0; }
    for (int i = t; i < m; i += T) {
      const double vi = fma(alpha, M.X[n + i], vw[i]);
      if (i >= S.z + S.l) M.v[i] = vi;
      M.piy[i] = (i >= S.z && i < S.z + S.l) ? fmax(vi, 0.0) : vi;
    }
    __syncthreads();
#else
    for (int j = t; j < n; j += T) {
      M.x[j] = a.x[(size_t)inst * n + j]; M.c[j] = a.c[(size_t)inst * n + j]; M.px2c[j] = 0.0;
    }
    for (int i = t; i < m; i += T) {
      const double yi = a.y[(size_t)inst * m + i], si = a.s[(size_t)inst * m + i];
      const double vi = yi - si;
      if (i >= S.z + S.l) M.v[i] = vi;
      M.b[i] = a.b[(size_t)inst * m + i];
      M.piy[i] = (i >= S.z && i < S.z + S.l) ? fmax(vi, 0.0) : vi;
      if constexpr (!JVP) M.t1[i] = dyg[i];
    }
    if (VG ? tmaP : (bool)a.use_tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }
    __syncthreads();
#endif
    // ---- cone Jacobian set-up: pi_y on SOC/PSD blocks, eigen-decompositions for PSD blocks ----
    if (S.ncones > 0) {
      const int lane = t & 31, warp = t >> 5, nw = T >> 5;
      int psd_off = 0;
      for (int cb = 0; cb < S.ncones; cb++) {
        const int ty = __ldg(S.cone_type + cb), s0 = __ldg(S.cone_start + cb), k = __ldg(S.cone_order + cb);
        const int my_off = psd_off;
        if (ty == BC_CPSD) psd_off += k * k + k;
        if (cb % nw != warp) continue;
        if (ty == BC_CSOC) project_soc_warp(M.piy + s0, __ldg(S.cone_size + cb));
        else {
          double *Vm = M.psdVL + my_off, *lam = Vm + k * k;
          double *Xd = M.psdscr + warp * (3 * S.max_psd * S.max_psd + S.max_psd);
          svec_to_mat_warp(k, M.v + s0, Xd);
          __syncwarp();
          if (k <= 16) {   // parallel-ordered Jacobi (common.cuh), cold start
            for (int e = lane; e < k * k; e += 32) Vm[e] = (e / k == e % k) ? 1.0 : 0.0;
            __syncwarp();
            jacobi_par_warp(k, Xd, Vm);
          } else jacobi_eig_warp(k, Xd, Vm);
          for (int i = lane; i < k; i += 32) lam[i] = Xd[i * k + i];
          __syncwarp();
          for (int e = lane; e < k * k; e += 32) {  // pi = V max(lam,0) V'
            const int i = e / k, j = e % k; double acc = 0;
            for (int q = 0; q < k; q++) acc = fma(Vm[i * k + q] * fmax(lam[q], 0.0), Vm[j * k + q], acc);
            Xd[k * k + e] = acc;
          }
          __syncwarp();
          mat_to_svec_warp(k, Xd + k * k, M.piy + s0);
        }
      }
      __syncthreads();
    }
    if (S.ep + S.ed > 0) {   // exponential cones: pi_y and the 3x3 Jacobians, one cone per thread
      for (int e = t; e < S.ep + S.ed; e += T) {
        const int s0 = S.exp_start + 3 * e;
        dproj_exp_dualblock_mat(M.v + s0, e < S.ep, M.expJ + 9 * e);
        proj_exp_dualblock(M.piy + s0, e < S.ep);
      }
      __syncthreads();
    }
    // ---- 2Px + c, x'Px ----
    double xPx = 0;
    if (Pg) {
      P_mul(S, Pg, M.x, M.part, [&](int j, double v) { M.px2c[j] += v; }, plN);
      double d1[1] = {0};
      for (int j = t; j < n; j += T) d1[0] = fma(M.x[j], M.px2c[j], d1[0]);
      block_reduce<1, false>(d1, M.red);
      xPx = d1[0];
    }
    for (int j = t; j < n; j += T) M.px2c[j] = 2.0 * M.px2c[j] + M.c[j];
    double d3[3] = {0, 0, 0};
    if constexpr (JVP) {
#ifdef BC_REFINE
      const double rn = refine_rhs<DENSE>(a, M, Pg, vw, alpha, plA, plN);   // -R -> U (syncs px2c)
      if (!have_w || rn < rn_w) {   // (NaN: rejected)
        for (int j = t; j < n; j += T) xw[j] = M.x[j];
        for (int i = t; i < m; i += T) { vw[i] = fma(alpha, M.X[n + i], vw[i]); yw[i] = M.piy[i]; ryw[i] = M.U[n + i]; }
        rn_w = rn; have_w = true;
        if (steps == ra.steps || !(rn > 0)) break;
        steps++;
        d3[1] = 1.0;
      } else if ((alpha *= 0.5) < 1.0 / 32) {
        break;
      } else {
        continue;
      }
#else
      d3[1] = jvp_rhs<DENSE>(a, M, inst, plA, plN);   // g -> U (syncs px2c)
#endif
    } else {
      // ---- dz -> U ----
      apply_D(S, M, M.t1, M.t2);  // t2 = D dy   (also syncs px2c)
      for (int j = t; j < n; j += T) { const double d = dxg[j]; M.U[j] = d; d3[0] = fma(M.x[j], d, d3[0]); d3[1] = fmax(d3[1], fabs(d)); }
      for (int i = t; i < m; i += T) {
        const double yi = a.y[(size_t)inst * m + i];
        M.U[n + i] = M.t2[i]; d3[0] = fma(yi, M.t1[i], d3[0]); d3[1] = fmax(d3[1], fabs(M.t2[i]));
      }
      {
        double s1[1] = {d3[0]}; block_reduce<1, false>(s1, M.red);
        double m1[1] = {d3[1]}; block_reduce<1, true>(m1, M.red);
        if (t == 0) M.U[N - 1] = -s1[0];
        d3[1] = fmax(m1[0], fabs(s1[0]));
      }
    }
    __syncthreads();
    int itn = 0;
    for (int k = t; k < N; k += T) M.X[k] = 0.0;
    if (d3[1] > 1e-8) {
      // ================= LSQR on B = M' (Paige & Saunders; SciPy stopping rules, damp = 0) ====
      const double eps = 2.220446049250313e-16;
      const double atol = st.lsqr_atol, btol = st.lsqr_btol;
      const double ctol = st.lsqr_conlim > 0 ? 1.0 / st.lsqr_conlim : 0.0;
      const int iter_lim = st.lsqr_iter_lim < 0 ? 2 * N : st.lsqr_iter_lim;
#ifdef BC_REFINE
      const bool pc = true;   // (the tau column is masked by a zero column scaling; lsqr_precond = 0: otherwise identity)
#else
      const bool pc = st.lsqr_precond != 0;
#endif
      // row / column scaling of B: the equilibration is computed for M', so M takes it with the two sides swapped
      // (an inactive nonneg row zeroes column n+i of M, which is e_{n+i}, and row n+i: see jvp_inactive_rows)
      double *const Ls = JVP ? M.Rsc : M.Lsc, *const Rs = JVP ? M.Lsc : M.Rsc;
#ifdef BC_REFINE
      if (st.lsqr_precond != 0) equilibrate<DENSE>(a, M, Pg, xPx, st.ruiz_passes > 0 ? st.ruiz_passes : 10, plA, plN);
      for (int k = t; k < N; k += T) {
        if (st.lsqr_precond == 0) { M.Lsc[k] = 1.0; M.Rsc[k] = 1.0; }
        if (k == N - 1) M.Lsc[k] = 0.0;   // tau fixed at 1: its column of M is dropped
        M.U[k] *= Ls[k]; M.X[k] = 0.0;
      }
      __syncthreads();
#else
      if (pc) {
        equilibrate<DENSE>(a, M, Pg, xPx, st.ruiz_passes > 0 ? st.ruiz_passes : 10, plA, plN);
        for (int k = t; k < N; k += T) { M.U[k] *= Ls[k]; M.X[k] = 0.0; }
        __syncthreads();
      }
#endif
      // B = diag(Lsc) M' diag(Rsc), or diag(Rsc) M diag(Lsc) for the JVP  (identity scalings when lsqr_precond = 0);
      // both products accumulate
      auto acc_B = [&](const double *in, double *out) {   // out += B in
        const double *src = in;
        if (pc) { for (int k = t; k < N; k += T) M.tin[k] = Rs[k] * in[k]; src = M.tin; }
        __syncthreads();
        if constexpr (JVP) op_M<DENSE>(a, M, Pg, xPx, src, out, pc ? Ls : nullptr, plA, plN);
        else op_MT<DENSE>(a, M, Pg, xPx, src, out, pc ? Ls : nullptr, plA, plN);
      };
      auto acc_BT = [&](const double *in, double *out) {  // out += B' in
        const double *src = in;
        if (pc) { for (int k = t; k < N; k += T) M.tin[k] = Ls[k] * in[k]; src = M.tin; }
        __syncthreads();
        if constexpr (JVP) op_MT<DENSE>(a, M, Pg, xPx, src, out, pc ? Rs : nullptr, plA, plN);
        else op_M<DENSE>(a, M, Pg, xPx, src, out, pc ? Rs : nullptr, plA, plN);
      };
#ifdef BC_LSMR   // (not if constexpr: a scope around the LSQR code below changes the code of the forward-mode kernels)
      auto opB = [&](const double *in, double *out, double coef) {   // out <- B in + coef out, ||out||^2
        for (int k = t; k < N; k += T) out[k] *= coef;
        acc_B(in, out);
        double q[1] = {0};
        for (int k = t; k < N; k += T) q[0] = fma(out[k], out[k], q[0]);
        block_reduce<1, false>(q, M.red);
        return q[0];
      };
      auto opBT = [&](const double *in, double *out, double coef) {   // out <- B' in + coef out, ||out||^2
        for (int k = t; k < N; k += T) out[k] *= coef;
        acc_BT(in, out);
        double q[1] = {0};
        for (int k = t; k < N; k += T) q[0] = fma(out[k], out[k], q[0]);
        block_reduce<1, false>(q, M.red);
        return q[0];
      };
      itn = lsmr_block(N, M.U, M.V, M.W, M.t2 + m, M.X, M.red, st, iter_lim, opB, opBT);   // (u, v, h, h-bar, x)
#else
      double r1[1] = {0};
      for (int k = t; k < N; k += T) r1[0] = fma(M.U[k], M.U[k], r1[0]);
      block_reduce<1, false>(r1, M.red);
      const double bnorm = sqrt(r1[0]);
      double beta = bnorm, alfa = 0;
      // (beta = 0: the right-hand side vanished under the equilibration -- a forward-mode tangent that lives only in the
      //  dropped rows of inactive nonneg constraints.  As in SciPy's LSQR the solution is then 0; jvp_inactive_rows recovers
      //  those rows' unknowns from their own equations.  Dividing by it here turned the whole tangent into NaN.)
      for (int k = t; k < N; k += T) { M.U[k] = beta > 0 ? M.U[k] / beta : 0.0; M.V[k] = 0.0; }
      acc_BT(M.U, M.V);  // v = B' u
      r1[0] = 0;
      for (int k = t; k < N; k += T) r1[0] = fma(M.V[k], M.V[k], r1[0]);
      block_reduce<1, false>(r1, M.red);
      alfa = sqrt(r1[0]);
      if (alfa > 0) for (int k = t; k < N; k += T) { const double q = M.V[k] / alfa; M.V[k] = q; M.W[k] = q; }
      __syncthreads();
      double rhobar = alfa, phibar = beta, anorm = 0, ddnorm = 0, xxnorm = 0, z = 0, cs2 = -1, sn2 = 0;
      if (alfa * beta != 0.0) {
        while (itn < iter_lim) {
          itn++;
          for (int k = t; k < N; k += T) M.U[k] *= -alfa;   // u = B v - alfa u
          acc_B(M.V, M.U);
          r1[0] = 0;
          for (int k = t; k < N; k += T) r1[0] = fma(M.U[k], M.U[k], r1[0]);
          block_reduce<1, false>(r1, M.red);
          beta = sqrt(r1[0]);
          if (beta > 0) {
            for (int k = t; k < N; k += T) { M.U[k] /= beta; M.V[k] *= -beta; }   // v = B' u - beta v
            anorm = sqrt(anorm * anorm + alfa * alfa + beta * beta);
            acc_BT(M.U, M.V);
            r1[0] = 0;
            for (int k = t; k < N; k += T) r1[0] = fma(M.V[k], M.V[k], r1[0]);
            block_reduce<1, false>(r1, M.red);
            alfa = sqrt(r1[0]);
            if (alfa > 0) for (int k = t; k < N; k += T) M.V[k] /= alfa;
          }
          const double rho = hypot(rhobar, beta), cs = rhobar / rho, sn = beta / rho;
          const double theta = sn * alfa;
          rhobar = -cs * alfa;
          const double phi = cs * phibar;
          phibar = sn * phibar;
          const double tau = sn * phi;
          const double t1c = phi / rho, t2c = -theta / rho;
          __syncthreads();  // V normalised
          r1[0] = 0;
          for (int k = t; k < N; k += T) {
            const double wk = M.W[k], dk = wk / rho;
            r1[0] = fma(dk, dk, r1[0]);
            M.X[k] = fma(t1c, wk, M.X[k]);
            M.W[k] = fma(t2c, wk, M.V[k]);
          }
          block_reduce<1, false>(r1, M.red);
          ddnorm += r1[0];
          const double delta = sn2 * rho, gambar = -cs2 * rho, rhs = phi - delta * z, zbar = rhs / gambar;
          const double xnorm = sqrt(xxnorm + zbar * zbar);
          const double gamma = hypot(gambar, theta);
          cs2 = gambar / gamma; sn2 = theta / gamma; z = rhs / gamma; xxnorm += z * z;
          const double acond = anorm * sqrt(ddnorm), rnorm = phibar, arnorm = alfa * fabs(tau);
          const double test1 = rnorm / bnorm, test2 = arnorm / (anorm * rnorm + eps), test3 = 1.0 / (acond + eps);
          const double tt1 = test1 / (1.0 + anorm * xnorm / bnorm), rtol = btol + atol * anorm * xnorm / bnorm;
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
      }
#endif
      if (pc) { __syncthreads(); for (int k = t; k < N; k += T) M.X[k] *= Rs[k]; }
#ifdef BC_REFINE
      if (st.lsqr_precond != 0 && S.l > 0) { __syncthreads(); refine_inactive_rows<DENSE>(a, M, ryw); }
#else
      if constexpr (JVP) if (pc && S.l > 0) { __syncthreads(); jvp_inactive_rows<DENSE>(a, M, inst); }
#endif
    }
    __syncthreads();
#ifdef BC_REFINE
    alpha = 1.0;
    }   // (Newton loop)
    // ---- write-back: the candidate (x, pi_y, pi_y - v) replaces the input only if none of rp, rd, gap grows ----
    __syncthreads();
    for (int i = t; i < m; i += T) ryw[i] = yw[i] - vw[i];
    const RefMet r1 = refine_metrics<DENSE>(a, M, Pg, xw, yw, ryw, plA, plN);
    const bool accept = r1.r[0] <= r0.r[0] && r1.r[1] <= r0.r[1] && r1.r[2] <= r0.r[2];   // (false for a NaN)
    if (accept) {
      for (int j = t; j < n; j += T) a.tx[(size_t)inst * n + j] = xw[j];
      for (int i = t; i < m; i += T) { a.ty[(size_t)inst * m + i] = yw[i]; a.ts[(size_t)inst * m + i] = ryw[i]; }
      if (t == 0 && ra.resid) for (int q = 0; q < 3; q++) ra.resid[(size_t)inst * 3 + q] = r1.r[q];
    }
    if (t == 0) ra.flags[inst] = accept ? 1 : 0;
#else
    if constexpr (JVP) {   // ---- solution tangents: dx = z_x - x z_tau, dy = D z_y - y z_tau, ds = D z_y - z_y - s z_tau ----
      apply_D(S, M, M.X + n, M.t2);
      const double zt = M.X[N - 1];
      for (int j = t; j < n; j += T) a.tx[(size_t)inst * n + j] = M.X[j] - M.x[j] * zt;
      for (int i = t; i < m; i += T) {
        const size_t k = (size_t)inst * m + i;
        a.ty[k] = M.t2[i] - a.y[k] * zt;
        if (a.ts) a.ts[k] = M.t2[i] - M.X[n + i] - a.s[k] * zt;
      }
      if (t == 0 && a.lsqr_iters) a.lsqr_iters[inst] = itn;
    } else
    // ---- gradient assembly (every structural entry; SURVEY.md 8a B4 + the A.nonzero() hazard) ----
    {
      const double rt = M.X[N - 1];
      double *dAo = a.dA + (size_t)inst * S.nnzA;
      if (a.srec) {   // shared matrices: r and pi_y for the batch-summing reduction (shared.cu)
        put_srec(a.srec + (size_t)inst * bc_srec_doubles(n, m), M.X, M.X + n, rt, M.piy, n, m);
      } else if (DENSE) {
        for (int k = t; k < S.nnzA; k += T) { const int i = k / n, j = k % n; dAo[k] = M.x[j] * M.X[n + i] - M.piy[i] * M.X[j]; }
      } else {
        for (int k = t; k < S.nnzA; k += T) {
          const int i = __ldg(S.A_rowof + k), j = __ldg(S.A_indices + k);
          dAo[k] = M.x[j] * M.X[n + i] - M.piy[i] * M.X[j];
        }
      }
      for (int i = t; i < m; i += T) a.db[(size_t)inst * m + i] = M.piy[i] * rt - M.X[n + i];
      for (int j = t; j < n; j += T) a.dc[(size_t)inst * n + j] = M.x[j] * rt - M.X[j];
      if (a.dP && S.nnzP > 0 && !a.srec) {
        double *dPo = a.dP + (size_t)inst * S.nnzP;
        for (int k = t; k < S.nnzP; k += T) {
          const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);
          const double gij = (rt * M.x[i] - M.X[i]) * M.x[j], gji = (rt * M.x[j] - M.X[j]) * M.x[i];
          dPo[k] = (i == j) ? gij : gij + gji;
        }
      }
      if (t == 0 && a.lsqr_iters) a.lsqr_iters[inst] = itn;
    }
#endif
    __syncthreads();
  }
}

// The instantiations that exist: the adjoint and the forward-mode derivative (same kernel, same shared-memory layout, JVP = true)
// each as the 128-register build, the 4-CTA/SM build and the values-off-chip build (512-thread only); each with LSQR
// (bwd_kernel) and LSMR (bwd_lsmr_kernel).
template <bool JVP>
static const void *lsqr_kernel(int dense, int small_cta, int vals_global) {
  if (small_cta && vals_global) return nullptr;
  if (vals_global) return dense ? (const void *)BWD_KERNEL<true, false, JVP, true> : (const void *)BWD_KERNEL<false, false, JVP, true>;
  if (small_cta) return dense ? (const void *)BWD_KERNEL<true, true, JVP> : (const void *)BWD_KERNEL<false, true, JVP>;
  return dense ? (const void *)BWD_KERNEL<true, false, JVP> : (const void *)BWD_KERNEL<false, false, JVP>;
}
#if defined(BC_REFINE)
extern "C" size_t bc_refine_smem_bytes(int n, int m, int npoly, int nnzA, int nnzP_smem, int threads, int max_psd, int psd_total, int nexp,
                                       int vec_global, int vals_global) {
  return bwd_smem_doubles(n, m, npoly, nnzA, nnzP_smem, threads, max_psd, psd_total, nexp, vec_global, vals_global, 0, 1) * sizeof(double);
}
extern "C" size_t bc_refine_ws_doubles(int n, int m, int npoly) { return (bwd_vec_doubles(n, m, npoly, 0, 1) + 1) & ~(size_t)1; }
extern "C" const void *bc_refine_kernel(int dense, int small_cta, int vals_global) { return lsqr_kernel<true>(dense, small_cta, vals_global); }
#elif !defined(BC_LSMR)
extern "C" size_t bc_bwd_smem_bytes(int n, int m, int npoly, int nnzA, int nnzP_smem, int threads, int max_psd, int psd_total, int nexp, int vec_global,
                                    int vals_global, int lsmr) {
  return bwd_smem_doubles(n, m, npoly, nnzA, nnzP_smem, threads, max_psd, psd_total, nexp, vec_global, vals_global, lsmr) * sizeof(double);
}
extern "C" size_t bc_bwd_ws_doubles(int n, int m, int npoly, int lsmr) { return (bwd_vec_doubles(n, m, npoly, lsmr) + 1) & ~(size_t)1; }
extern "C" const void *bc_lsqr_kernel(int dense, int small_cta, int jvp, int vals_global, int lsmr) {
  if (lsmr) return bc_lsmr_kernel(dense, small_cta, jvp, vals_global);
  return jvp ? lsqr_kernel<true>(dense, small_cta, vals_global) : lsqr_kernel<false>(dense, small_cta, vals_global);
}
#else
extern "C" const void *bc_lsmr_kernel(int dense, int small_cta, int jvp, int vals_global) {
  return jvp ? lsqr_kernel<true>(dense, small_cta, vals_global) : lsqr_kernel<false>(dense, small_cta, vals_global);
}
#endif
