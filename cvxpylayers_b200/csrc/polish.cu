// polish.cu -- solution polishing for QPs and LPs with zero + nonneg cones (bcone_polish; NumPy twin: tests/polish_ref.py).
//
// The forward returns an operator-splitting iterate that meets eps, not the optimum.  Polishing (OSQP's `polish`) guesses the
// active set from it and solves the equality-constrained QP of that set exactly:
//   live rows L = the zero rows + the nonneg rows with y_i > s_i (the block adjoint's pi_y > 0),
//   [[P + d I, A_L'], [A_L, -d I]] [x; y_L] = [-c; b_L]
// through  P + d I = L L'  (chol_inv_packed: Pb <- L^{-1}),  W = L^{-1} A_L'  (in place over the staged rows of A),
// S = d I + W'W  (packed after W; Sb <- L_S^{-1}), then `refine` steps of iterative refinement against the unregularised
// KKT matrix, whose residuals read A and P from global memory (L2).  d = delta x the largest absolute entry of P and A_L (d
// scales with the data, so a whole instance multiplied by a constant polishes to the same x and y).  d makes the system
// quasi-definite: it also factorises for an LP (P = 0 or only semidefinite) and for dependent live rows.
// The candidate is completed to y = 0 off L, s = b - A x with s_L = 0, and s, y clipped at 0 on the nonneg rows (exactly
// complementary).  It replaces the input only if none of rp = |A x + s - b|_inf, rd = |P x + A'y + c|_inf and
// gap = |x'Px + c'x + b'y| is larger than the input's (same code for both); otherwise x, y, s are not written.  The status is
// never changed.  polished[i]: 1 accepted, 0 rejected (also: P + d I or S not positive definite), -1 not attempted (status
// not SOLVED / INACCURATE, a non-finite input, or W and S larger than the staging buffer of stage_cap doubles).
#include "common.cuh"

struct PolSmem {
  double *Pb, *Ab, *c, *bv, *x, *y, *s, *t, *r1, *dx, *ax, *aty, *px, *r2, *dyl, *yl, *tmp, *part, *red;
  int *live;
  uint64_t *bar;
  int *ibuf;
};

__host__ __device__ inline size_t pol_smem_doubles(int n, int m, int threads, long long stage_cap) {
  return 4 + (((size_t)n * (n + 1) / 2 + 1) & ~(size_t)1) + (((size_t)stage_cap + 1) & ~(size_t)1) + 7 * (size_t)n + 7 * (size_t)m +
         chol_scratch_doubles(n, threads) + threads + 4 * 32 + ((size_t)m + 2) / 2;
}

__device__ __forceinline__ void carve_pol(PolSmem &M, double *base, int n, int m, int threads, long long stage_cap) {
  double *q = base;
  M.bar = (uint64_t *)q; q += 2;
  M.ibuf = (int *)q; q += 2;
  M.Pb = q; q += (n * (n + 1) / 2 + 1) & ~1;
  M.Ab = q; q += (stage_cap + 1) & ~1LL;   // 16-byte aligned: the TMA destination
  M.c = q; q += n; M.x = q; q += n; M.t = q; q += n; M.r1 = q; q += n; M.dx = q; q += n; M.aty = q; q += n; M.px = q; q += n;
  M.bv = q; q += m; M.y = q; q += m; M.s = q; q += m; M.ax = q; q += m; M.r2 = q; q += m; M.dyl = q; q += m; M.yl = q; q += m;
  M.tmp = q; q += chol_scratch_doubles(n, threads);
  M.part = q; q += threads; M.red = q; q += 4 * 32;
  M.live = (int *)q;
}

template <bool DENSE>
__device__ __forceinline__ void polish_body(const PolishArgs &a) {
  extern __shared__ __align__(16) double smem[];
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = T >> 5;
  PolSmem M;
  carve_pol(M, smem, n, m, T, a.stage_cap);
  if (t == 0) { mbar_init(M.bar, 1); fence_mbar_init(); }
  __syncthreads();
  uint32_t tma_phase = 0;
  const int z = S.z;   // rows [0, z) zero cone, [z, m) nonneg (the only cones a polish plan exists for)
  const ColPlan plN = make_colplan(n, n), plA = make_colplan(m, n);

  for (;;) {
    if (t == 0) M.ibuf[0] = atomicAdd(a.counter, 1);
    __syncthreads();
    const int inst = M.ibuf[0];
    if (inst >= a.B) break;
    const double *Ag = a.A_vals + (size_t)inst * a.sA;
    const double *Pg = S.nnzP > 0 ? a.P_vals + (size_t)inst * a.sP : nullptr;
    double *xg = a.x + (size_t)inst * n, *yg = a.y + (size_t)inst * m, *sg = a.s + (size_t)inst * m;
    const int stat = a.status[inst];
    bool finite = true;
    for (int j = t; j < n; j += T) { const double v = xg[j]; M.x[j] = v; M.c[j] = a.c[(size_t)inst * n + j]; finite &= isfinite(v); }
    for (int i = t; i < m; i += T) {
      const double yi = yg[i], si = sg[i];
      M.y[i] = yi; M.s[i] = si; M.bv[i] = a.b[(size_t)inst * m + i];
      finite &= isfinite(yi) && isfinite(si);
    }
    finite = __syncthreads_and(finite);
    if ((stat != 1 && stat != 2) || !finite) {
      if (t == 0) a.polished[inst] = -1;
      continue;
    }

    // ax = A x, aty = A' y, px = P x of the point in M.x / M.y (A and P from global memory).  Ends synchronised.
    auto products = [&]() {
      for (int j = t; j < n; j += T) M.px[j] = 0.0;
      A_mul<DENSE>(S, Ag, M.x, [&](int i, double v) { M.ax[i] = v; });
      AT_mul<DENSE>(S, Ag, M.y, M.part, [&](int j, double v) { M.aty[j] = v; }, plA);   // (ends synchronised)
      if (S.nnzP > 0) P_mul(S, Pg, M.x, M.part, [&](int i, double v) { M.px[i] += v; }, plN);
    };
    // rp, rd, gap of the point in M.x / M.y / M.s; every thread gets the same bits
    auto metrics = [&](double (&r)[3]) {
      products();
      auto amax = [](double acc, double v) { const double e = fabs(v); return e == e ? fmax(acc, e) : INFINITY; };   // (NaN counts as inf)
      double mx[2] = {0, 0}, sm[1] = {0};
      for (int i = t; i < m; i += T) { mx[0] = amax(mx[0], M.ax[i] + M.s[i] - M.bv[i]); sm[0] = fma(M.bv[i], M.y[i], sm[0]); }
      for (int j = t; j < n; j += T) {
        mx[1] = amax(mx[1], M.px[j] + M.aty[j] + M.c[j]);
        sm[0] = fma(M.x[j], M.px[j] + M.c[j], sm[0]);
      }
      block_reduce<2, true>(mx, M.red);
      block_reduce<1, false>(sm, M.red);
      r[0] = mx[0]; r[1] = mx[1]; r[2] = fabs(sm[0]);
    };
    double r0[3];
    metrics(r0);

    // ---- live rows ----
    if (warp == 0) {
      int cnt = 0;
      for (int base = 0; base < m; base += 32) {
        const int i = base + lane;
        const bool lv = i < m && (i < z || M.y[i] > M.s[i]);
        const unsigned bal = __ballot_sync(0xffffffffu, lv);
        if (lv) M.live[cnt + __popc(bal & ((1u << lane) - 1))] = i;
        cnt += __popc(bal);
      }
      if (lane == 0) M.ibuf[1] = cnt;
    }
    __syncthreads();
    const int nl = M.ibuf[1];
    if (nl > n || (long long)nl * n + ((long long)nl * (nl + 1)) / 2 > a.stage_cap) {
      if (t == 0) a.polished[inst] = -1;
      continue;
    }
    // ---- stage A_L (dense: one TMA bulk copy per row, or plain loads; CSR: scattered into zeroed dense rows) and P ----
    double *Ws = M.Ab, *Sb = M.Ab + nl * n;
    const bool tma = DENSE && a.use_tma && nl > 0;
    if (tma && warp == 0) {
      if (lane == 0) { fence_proxy_async(); mbar_expect_tx(M.bar, (uint32_t)(nl * n * sizeof(double))); }
      __syncwarp();
      for (int l = lane; l < nl; l += 32) tma_bulk_g2s(Ws + l * n, Ag + (size_t)M.live[l] * n, (uint32_t)(n * sizeof(double)), M.bar);
    }
    if (DENSE && !tma) {
      for (int e = t; e < nl * n; e += T) { const int l = e / n, j = e - l * n; Ws[e] = Ag[(size_t)M.live[l] * n + j]; }
    } else if (!DENSE) {
      for (int e = t; e < nl * n; e += T) Ws[e] = 0.0;
    }
    for (int e = t; e < (n * (n + 1)) / 2; e += T) M.Pb[e] = 0.0;
    __syncthreads();
    if (!DENSE) {
      for (int l = warp; l < nl; l += nw) {
        const int i = M.live[l], e = __ldg(S.A_indptr + i + 1);
        for (int k = __ldg(S.A_indptr + i) + lane; k < e; k += 32) Ws[l * n + __ldg(S.A_indices + k)] = Ag[k];
      }
    }
    for (int k = t; k < S.nnzP; k += T) {   // upper row-major CSR -> lower row-major packed
      const int i = __ldg(S.P_rowof + k), cc = __ldg(S.P_indices + k);
      M.Pb[((cc * (cc + 1)) >> 1) + i] = Pg[k];
    }
    if (tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }
    __syncthreads();
    // ---- d = delta max(|P|_max, |A_L|_max); P + d I = L L' ----
    double dm[1] = {0.0};
    for (int e = t; e < (n * (n + 1)) / 2; e += T) dm[0] = fmax(dm[0], fabs(M.Pb[e]));
    for (int e = t; e < nl * n; e += T) dm[0] = fmax(dm[0], fabs(Ws[e]));
    block_reduce<1, true>(dm, M.red);
    const double d = a.delta * (dm[0] > 0.0 ? dm[0] : 1.0);
    for (int j = t; j < n; j += T) M.Pb[((j * (j + 1)) >> 1) + j] += d;
    __syncthreads();
    bool ok = chol_inv_packed(M.Pb, n, M.tmp);   // Pb <- L^{-1}
    __syncthreads();
    if (ok && nl > 0) {
      // ---- W = A_L L^{-T} in place on the tensor cores: one warp per 8 staged rows, their A fragments (n <= 128) in
      //      registers for every k-step ----
      {
        constexpr int KSMAX = 32;
        const int fr = lane >> 2, fc = lane & 3;
        const int ntl = (nl + 7) >> 3, nti = (n + 7) >> 3;
        for (int lt = warp; lt < ntl; lt += nw) {
          const int l = 8 * lt + fr;
          double af[KSMAX];
#pragma unroll
          for (int ks = 0; ks < KSMAX; ks++) { const int cidx = 4 * ks + fc; af[ks] = (l < nl && cidx < n) ? Ws[l * n + cidx] : 0.0; }
          __syncwarp();
          for (int it = 0; it < nti; it++) {
            const int i = 8 * it + fr;
            const double *Lrow = M.Pb + ((i * (i + 1)) >> 1);
            const int klim = 8 * it + 8;
            double c0 = 0.0, c1 = 0.0;
#pragma unroll
            for (int ks = 0; ks < KSMAX; ks++) {
              if (4 * ks < klim) {
                const int cidx = 4 * ks + fc;
                const double fb = (i < n && cidx <= i) ? Lrow[cidx] : 0.0;
                dmma884(c0, c1, af[ks], fb);
              }
            }
            const int col = 8 * it + 2 * fc;
            if (l < nl && col < n) Ws[l * n + col] = c0;        // (scalar stores: n may be odd)
            if (l < nl && col + 1 < n) Ws[l * n + col + 1] = c1;
          }
        }
      }
      __syncthreads();
      // ---- S = d I + W W' (packed lower) on 8 x 8 tiles ----
      {
        const int fr = lane >> 2, fc = lane & 3;
        const int ntl = (nl + 7) >> 3, ntile = (ntl * (ntl + 1)) >> 1, nks = (n + 3) >> 2;
        for (int e = warp; e < ntile; e += nw) {
          int ta = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
          while (((ta + 1) * (ta + 2)) >> 1 <= e) ta++;
          while ((ta * (ta + 1)) >> 1 > e) ta--;
          const int tb = e - ((ta * (ta + 1)) >> 1);
          const int la = 8 * ta + fr, lb = 8 * tb + fr;
          const double *pa = Ws + min(la, nl - 1) * n, *pb = Ws + min(lb, nl - 1) * n;
          double c0 = 0.0, c1 = 0.0;
          for (int ks = 0; ks < nks; ks++) {
            const int cidx = 4 * ks + fc;
            const double fa = (la < nl && cidx < n) ? pa[cidx] : 0.0, fb = (lb < nl && cidx < n) ? pb[cidx] : 0.0;
            dmma884(c0, c1, fa, fb);
          }
          const int r = 8 * ta + fr, q = 8 * tb + 2 * fc;
          if (r < nl && q <= r) Sb[((r * (r + 1)) >> 1) + q] = c0 + (q == r ? d : 0.0);
          if (r < nl && q + 1 <= r) Sb[((r * (r + 1)) >> 1) + q + 1] = c1 + (q + 1 == r ? d : 0.0);
        }
      }
      __syncthreads();
      ok = chol_inv_packed(Sb, nl, M.tmp);   // Sb <- L_S^{-1}
      __syncthreads();
    }
    if (!ok) {
      if (t == 0) a.polished[inst] = 0;
      continue;
    }
    const ColPlan plW = make_colplan(nl, n), plS = make_colplan(nl, nl);
    // [dx; dyl] = K_d^{-1} [r1; r2]:  S dyl = W' L^{-1} r1 - r2,  dx = L^{-T} (L^{-1} r1 - W dyl)   (r2 is overwritten)
    auto kkt_solve = [&]() {
      matvec_rows(M.Pb, PackedLowerLayout{}, n, n, M.r1, [&](int i, double v) { M.t[i] = v; });
      __syncthreads();
      if (nl > 0) {
        matvec_rows(Ws, DenseLayout{n}, nl, n, M.t, [&](int l, double v) { M.dyl[l] = v - M.r2[l]; });
        __syncthreads();
        matvec_rows(Sb, PackedLowerLayout{}, nl, nl, M.dyl, [&](int i, double v) { M.r2[i] = v; });
        __syncthreads();
        matvec_cols(Sb, PackedLowerLayout{}, nl, nl, M.r2, M.part, [&](int j, double v) { M.dyl[j] = v; }, plS);
        matvec_cols(Ws, DenseLayout{n}, nl, n, M.dyl, M.part, [&](int j, double v) { M.t[j] -= v; }, plW);
      }
      matvec_cols(M.Pb, PackedLowerLayout{}, n, n, M.t, M.part, [&](int j, double v) { M.dx[j] = v; }, plN);
    };
    // ---- regularised solve, then refinement against K = [[P, A_L'], [A_L, 0]] ----
    for (int j = t; j < n; j += T) M.r1[j] = -M.c[j];
    for (int l = t; l < nl; l += T) M.r2[l] = M.bv[M.live[l]];
    __syncthreads();
    kkt_solve();
    for (int j = t; j < n; j += T) M.x[j] = M.dx[j];
    for (int l = t; l < nl; l += T) M.yl[l] = M.dyl[l];
    for (int k = 0; k < a.refine; k++) {
      for (int i = t; i < m; i += T) M.y[i] = 0.0;
      __syncthreads();
      for (int l = t; l < nl; l += T) M.y[M.live[l]] = M.yl[l];
      __syncthreads();
      products();
      for (int j = t; j < n; j += T) M.r1[j] = -M.c[j] - M.px[j] - M.aty[j];
      for (int l = t; l < nl; l += T) M.r2[l] = M.bv[M.live[l]] - M.ax[M.live[l]];
      __syncthreads();
      kkt_solve();
      for (int j = t; j < n; j += T) M.x[j] += M.dx[j];
      for (int l = t; l < nl; l += T) M.yl[l] += M.dyl[l];
    }
    // ---- complete the point: y = 0 off L, clipped on the nonneg rows; s = b - A x, 0 on L, clipped ----
    for (int i = t; i < m; i += T) M.y[i] = 0.0;
    __syncthreads();
    for (int l = t; l < nl; l += T) { const int i = M.live[l]; M.y[i] = i < z ? M.yl[l] : fmax(M.yl[l], 0.0); }
    __syncthreads();
    A_mul<DENSE>(S, Ag, M.x, [&](int i, double v) { M.ax[i] = v; });
    __syncthreads();
    for (int i = t; i < m; i += T) M.s[i] = i < z ? 0.0 : fmax(M.bv[i] - M.ax[i], 0.0);
    __syncthreads();
    for (int l = t; l < nl; l += T) M.s[M.live[l]] = 0.0;
    __syncthreads();
    double r1v[3];
    metrics(r1v);
    const bool accept = r1v[0] <= r0[0] && r1v[1] <= r0[1] && r1v[2] <= r0[2];   // (false for a NaN)
    if (accept) {
      for (int j = t; j < n; j += T) xg[j] = M.x[j];
      for (int i = t; i < m; i += T) { yg[i] = M.y[i]; sg[i] = M.s[i]; }
      if (t == 0 && a.resid) { a.resid[inst * 3 + 0] = r1v[0]; a.resid[inst * 3 + 1] = r1v[1]; a.resid[inst * 3 + 2] = r1v[2]; }
    }
    if (t == 0) a.polished[inst] = accept ? 1 : 0;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(512, 1) polish_dense_kernel(const __grid_constant__ PolishArgs a) { polish_body<true>(a); }
__global__ void __launch_bounds__(512, 1) polish_csr_kernel(const __grid_constant__ PolishArgs a) { polish_body<false>(a); }

extern "C" size_t bc_polish_smem_bytes(int n, int m, int threads, long long stage_cap) {
  return pol_smem_doubles(n, m, threads, stage_cap) * sizeof(double);
}
extern "C" const void *bc_polish_kernel(int dense) { return dense ? (const void *)polish_dense_kernel : (const void *)polish_csr_kernel; }
