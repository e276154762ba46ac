// bwd_block.cu -- backward kernel for strongly convex QPs with polyhedral cones (the headline
// shape): LSQR right-preconditioned by the exact block factorisation of the reduced KKT matrix
// (settings.lsqr_precond = 2; oracle twin: vjp_block_precond in oracle/cone_oracle.c).
//
// With live rows L (zero rows + active nonneg rows; dead rows have r_i = dz_i = 0 exactly) the
// reduced adjoint system of diffcp (SURVEY.md 8a B2-B3, reference call site diffcp_if.py:86) is
//     B r = dz,   B = [[G, -h'], [g', x'Px]],   G = [[P, -A_L'], [A_L, 0]],  h' = (2Px+c ; b_L),  g = (c ; b_L).
// B blkdiag(G,1)^{-1} = [[I, -h'], [(G^{-T} g)', x'Px]] is the identity plus a rank-2 term, so LSQR needs
// ~3 iterations of O(N) work; its minimum-norm property still resolves the singular homogeneity
// direction.  G^{-1} is applied through  P = L L'  (packed Cholesky + explicit inverse, on chip),
// W = L^{-1} A_L'  (overwrites the staged rows of A in place) and  S = W'W = A_L P^{-1} A_L'  (Cholesky +
// inverse).  Only the live rows of A are staged (one TMA bulk copy per row).  Instances where the
// factorisation does not apply (P not positive definite, A_L rank deficient, more live rows than
// variables, or W and S together larger than the m n doubles the rows are staged in) are appended to a
// device-side list and re-run by bwd_fast_kernel with lsqr_precond = 1.
#include "common.cuh"

// W (nl x n) and then S (nl x nl, packed lower) are written into the buffer of m n doubles that stages the live rows.  With nl
// close to m and m < 1.5 n (e.g. every row an equality) S would run past it into the vectors and the factorisation scratch.
// (Staging the rows themselves always fits: nl <= m.)
__device__ __forceinline__ bool blk_fits(int nl, int n, int m) {
  return nl <= n && nl * n + ((nl * (nl + 1)) >> 1) <= ((m * n + 1) & ~1);
}

struct BlkSmem {
  double *Pb, *Ab, *x, *c, *px2c, *piy, *hp, *q, *rhs, *z, *U, *V, *W, *tn, *t2, *tL, *ry, *part, *red;
  int *live;
  uint64_t *bar;
  int *ibuf;
};

__host__ __device__ inline size_t bwdb_smem_doubles(int n, int m, int threads) {
  const size_t N = (size_t)n + m + 1;
  return 4 + (((size_t)n * (n + 1) / 2 + 1) & ~(size_t)1) + (((size_t)m * n + 1) & ~(size_t)1) + 3 * (size_t)n + 2 * (size_t)m + 7 * N + 2 * (size_t)n +
         (size_t)m + threads + 4 * 32 + ((size_t)m + 2) / 2;
}

__device__ __forceinline__ void carve_blk(BlkSmem &M, double *base, int n, int m, int threads) {
  const int N = n + m + 1;
  double *q = base;
  M.bar = (uint64_t *)q; q += 2;
  M.ibuf = (int *)q; q += 2;
  M.Pb = q; q += (n * (n + 1) / 2 + 1) & ~1;
  M.Ab = q; q += (m * n + 1) & ~1;
  M.x = q; q += n; M.c = q; q += n; M.px2c = q; q += n;
  M.piy = q; q += m; M.ry = q; q += m;
  M.rhs = q; q += N;
  M.hp = q; q += N; M.q = q; q += N; M.z = q; q += N; M.U = q; q += N; M.V = q; q += N; M.W = q; q += N;   // 6 N contiguous: factorisation scratch
  M.tn = q; q += n; M.t2 = q; q += n; M.tL = q; q += m;
  M.part = q; q += threads; M.red = q; q += 4 * 32;
  M.live = (int *)q;
}

// LSMR: diffcp's mode = "lsmr" (common.cuh lsmr_block) on the same preconditioned operator C, in the same shared memory (its
// u starts on the right-hand side in place and h-bar takes LSQR's u); the kernel bwd_block_lsmr_kernel below.  The instances
// it rejects go to an LSMR pass as well (api.cu).
template <bool LSMR>
__device__ __forceinline__ void bwd_block_body(const BwdArgs a) {   // (by value: by reference the LSQR kernel compiles to other code)
  extern __shared__ __align__(16) double smem[];
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, N = n + m + 1, T = blockDim.x, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = T >> 5;
  const bc_settings &st = a.st;
  BlkSmem M;
  carve_blk(M, smem, n, m, T);
  if (t == 0) { mbar_init(M.bar, 1); fence_mbar_init(); }
  __syncthreads();
  uint32_t tma_phase = 0;
  const int lo = S.z, hi = S.z + S.l;
  const ColPlan plN = make_colplan(n, n);

  for (;;) {
    if (t == 0) M.ibuf[0] = atomicAdd(a.counter, 1);
    __syncthreads();
    const int inst = M.ibuf[0];
    if (inst >= a.B) break;
    const double *Ag = a.A_vals + (size_t)inst * a.sA;
    const double *Pg = a.P_vals + (size_t)inst * a.sP;
    const double *dxg = a.dx + (size_t)inst * n, *dyg = a.dy + (size_t)inst * m;
    PhaseTimer pt; pt.start(a.prof);
    // ---- vectors, pi_y, dz ----
    double d2[2] = {0, 0};
    for (int j = t; j < n; j += T) {
      const double xj = a.x[(size_t)inst * n + j], d = dxg[j];
      M.x[j] = xj; M.c[j] = a.c[(size_t)inst * n + j]; M.rhs[j] = d;
      d2[0] = fma(xj, d, d2[0]); d2[1] = fmax(d2[1], fabs(d));
    }
    for (int i = t; i < m; i += T) {
      const double yi = a.y[(size_t)inst * m + i], si = a.s[(size_t)inst * m + i], vi = yi - si;
      const double pi = (i >= lo && i < hi) ? fmax(vi, 0.0) : vi;
      const double dy = dyg[i], ddy = (i < lo || pi > 0) ? dy : 0.0;
      M.piy[i] = pi; M.ry[i] = 0.0; M.tL[i] = ddy;   // tL: D dy by original row (compacted below)
      d2[0] = fma(yi, dy, d2[0]); d2[1] = fmax(d2[1], fabs(ddy));
    }
    {
      double s1[1] = {d2[0]}; block_reduce<1, false>(s1, M.red);
      double m1[1] = {d2[1]}; block_reduce<1, true>(m1, M.red);
      d2[0] = s1[0]; d2[1] = fmax(m1[0], fabs(s1[0]));
    }
    // ---- live rows; stage them with one TMA bulk copy per row ----
    if (warp == 0) {
      int cnt = 0;
      for (int base = 0; base < m; base += 32) {
        const int i = base + lane;
        const bool lv = i < m && (i < lo || i >= hi || M.piy[i] > 0);
        const unsigned bal = __ballot_sync(0xffffffffu, lv);
        if (lv) M.live[cnt + __popc(bal & ((1u << lane) - 1))] = i;
        cnt += __popc(bal);
      }
      if (lane == 0) M.ibuf[1] = cnt;
      __syncwarp();
      if (cnt <= n && a.use_tma) {
        if (lane == 0) { fence_proxy_async(); mbar_expect_tx(M.bar, (uint32_t)(cnt * n * sizeof(double))); }
        __syncwarp();
        for (int l = lane; l < cnt; l += 32) tma_bulk_g2s(M.Ab + l * n, Ag + (size_t)M.live[l] * n, (uint32_t)(n * sizeof(double)), M.bar);
      }
    }
    // P: upper row-major packed (CSR order) -> lower row-major packed
    for (int k = t; k < S.nnzP; k += T) {
      const int i = __ldg(S.P_rowof + k), cc = __ldg(S.P_indices + k);
      M.Pb[((cc * (cc + 1)) >> 1) + i] = Pg[k];
    }
    __syncthreads();
    const int nl = M.ibuf[1], nr = n + nl;
    bool applicable = blk_fits(nl, n, m);
    if (applicable && !a.use_tma) {
      for (int e = t; e < nl * n; e += T) { const int l = e / n, j = e - l * n; M.Ab[e] = Ag[(size_t)M.live[l] * n + j]; }
    }
    pt.stamp(8);   // load vectors, live list, P scatter
    // ---- 2Px + c and x'Px from the packed lower P (before it is overwritten by its factor) ----
    double xPx = 0;
    if (applicable) {
      matvec_rows(M.Pb, PackedLowerLayout{}, n, n, M.x, [&](int i, double v) { M.px2c[i] = v; });
      __syncthreads();
      matvec_cols(M.Pb, PackedLowerStrictLayout{}, n, n, M.x, M.part, [&](int j, double v) { M.px2c[j] += v; }, plN);
      double s1[1] = {0};
      for (int j = t; j < n; j += T) { const double px = M.px2c[j]; s1[0] = fma(M.x[j], px, s1[0]); M.px2c[j] = 2.0 * px + M.c[j]; }
      block_reduce<1, false>(s1, M.red);
      xPx = s1[0];
      applicable = chol_inv_packed(M.Pb, n, M.hp, a.prof);   // Pb <- L^{-1}   (scratch: hp..W are free here, 6 N >= 8 n + 72 checked on the host)
    }
    if (applicable && a.use_tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }
    if (!applicable && nl <= n && a.use_tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }  // drain the copies already issued
    __syncthreads();
    pt.stamp(9);   // Px + Cholesky/inverse of P (+ wait for the row copies)
    double *Ws = M.Ab, *Sb = M.Ab + nl * n;
    if (applicable && nl > 0) {
      // ---- W = A_L Linv' in place on the tensor cores (DMMA 8x8x4): one warp per 8 staged rows, whose A fragments
      //      (8 x n, n <= 128) are held in registers for every k-step, so the rows can be overwritten tile by tile ----
      {
        constexpr int KSMAX = 32;                 // k-steps of 4 columns: n <= 128
        const int fr = lane >> 2, fc = lane & 3;
        const int ntl = (nl + 7) >> 3, nti = (n + 7) >> 3;
        for (int lt = warp; lt < ntl; lt += nw) {
          const int l = 8 * lt + fr;
          double af[KSMAX];
#pragma unroll
          for (int ks = 0; ks < KSMAX; ks++) { const int cidx = 4 * ks + fc; af[ks] = (l < nl && cidx < n) ? Ws[l * n + cidx] : 0.0; }
          __syncwarp();
          for (int it = 0; it < nti; it++) {
            const int i = 8 * it + fr;            // row of Linv feeding output column i
            const double *Lrow = M.Pb + ((i * (i + 1)) >> 1);
            const int klim = 8 * it + 8;          // Linv[i][c] = 0 for c > i
            double c0 = 0.0, c1 = 0.0;
#pragma unroll
            for (int ks = 0; ks < KSMAX; ks++) {
              if (4 * ks < klim) {                // warp-uniform
                const int cidx = 4 * ks + fc;
                const double fb = (i < n && cidx <= i) ? Lrow[cidx] : 0.0;
                dmma884(c0, c1, af[ks], fb);
              }
            }
            const int col = 8 * it + 2 * fc;
            if (l < nl && col < n) *reinterpret_cast<double2 *>(Ws + l * n + col) = make_double2(c0, c1);   // n is even
          }
        }
      }
      __syncthreads();
      pt.stamp(10);  // W = L^{-1} A_L'
      // ---- S = W W' (nl x nl, packed lower): 8 x 8 tiles of the lower triangle, one DMMA per 4 columns of W ----
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
          if (r < nl && q <= r) Sb[((r * (r + 1)) >> 1) + q] = c0;
          if (r < nl && q + 1 <= r) Sb[((r * (r + 1)) >> 1) + q + 1] = c1;
        }
      }
      __syncthreads();
      pt.stamp(11);  // S = W W'
      applicable = chol_inv_packed(Sb, nl, M.hp);   // Sb <- L_S^{-1}  (scratch: hp..W)
      pt.stamp(12);  // Cholesky/inverse of S
    }
    if (!applicable) {   // hand the instance to the fallback pass (block-uniform branch)
      if (t == 0) { const int k = atomicAdd(a.fail_count, 1); a.fail_list[k] = inst; }
      __syncthreads();
      continue;
    }
    const ColPlan plW = make_colplan(nl, n), plS = make_colplan(nl, nl);
    // solve with S = L_S L_S':  v <- L_S^{-T} (L_S^{-1} v)   (in/out in M.tL, scratch M.W)
    auto S_solve = [&]() {
      if (nl == 0) return;
      matvec_rows(Sb, PackedLowerLayout{}, nl, nl, M.tL, [&](int i, double v) { M.W[i] = v; });
      __syncthreads();
      matvec_cols(Sb, PackedLowerLayout{}, nl, nl, M.W, M.part, [&](int j, double v) { M.tL[j] = v; }, plS);
    };
    // ---- hp = (2Px+c ; b_L), q = G^{-T} (c ; b_L):  P qx + A_L' qL = c, -A_L qx = b_L ----
    for (int j = t; j < n; j += T) M.hp[j] = M.px2c[j];
    for (int l = t; l < nl; l += T) { const double bl = a.b[(size_t)inst * m + M.live[l]]; M.hp[n + l] = bl; M.rhs[n + l] = M.tL[M.live[l]]; }
    __syncthreads();
    matvec_rows(M.Pb, PackedLowerLayout{}, n, n, M.c, [&](int i, double v) { M.tn[i] = v; });          // tn = L^{-1} c
    __syncthreads();
    if (nl > 0) {
      matvec_rows(Ws, DenseLayout{n}, nl, n, M.tn, [&](int l, double v) { M.tL[l] = M.hp[n + l] + v; });   // b_L + A_L P^{-1} c
      __syncthreads();
      S_solve();                                                                                              // qL
      for (int l = t; l < nl; l += T) M.q[n + l] = M.tL[l];
      matvec_cols(Ws, DenseLayout{n}, nl, n, M.tL, M.part, [&](int j, double v) { M.tn[j] -= v; }, plW);   // tn -= W qL
    }
    matvec_cols(M.Pb, PackedLowerLayout{}, n, n, M.tn, M.part, [&](int j, double v) { M.q[j] = v; }, plN);   // qx = L^{-T} tn
    if (t == 0) M.rhs[nr] = -d2[0];
    __syncthreads();
    // ---- LSQR on C = [[I, -hp], [q', x'Px]]  (size nr + 1), SciPy stopping rules ----
    int itn = 0;
    const int NR = nr + 1;
    for (int k = t; k < NR; k += T) M.z[k] = 0.0;
    if (d2[1] > 1e-8) {
      const double eps = 2.220446049250313e-16, atol = st.lsqr_atol, btol = st.lsqr_btol;
      const double ctol = st.lsqr_conlim > 0 ? 1.0 / st.lsqr_conlim : 0.0;
      const int iter_lim = st.lsqr_iter_lim < 0 ? 2 * N : st.lsqr_iter_lim;
      // out = C in  /  out = C' in ; returns ||out||^2 (one block reduction each)
      auto C_mul = [&](const double *in, double *out, double coef) {   // out <- C in + coef * out
        const double it_ = in[nr];
        double r2[2] = {0, 0};
        for (int k = t; k < nr; k += T) { const double o = fma(-M.hp[k], it_, in[k]) + coef * out[k]; out[k] = o; r2[0] = fma(o, o, r2[0]); r2[1] = fma(M.q[k], in[k], r2[1]); }
        const double ot_old = out[nr];
        block_reduce<2, false>(r2, M.red);
        const double ot = r2[1] + xPx * it_ + coef * ot_old;
        if (t == 0) out[nr] = ot;
        __syncthreads();
        return r2[0] + ot * ot;
      };
      auto CT_mul = [&](const double *in, double *out, double coef) {  // out <- C' in + coef * out
        const double it_ = in[nr];
        double r2[2] = {0, 0};
        for (int k = t; k < nr; k += T) { const double o = fma(M.q[k], it_, in[k]) + coef * out[k]; out[k] = o; r2[0] = fma(o, o, r2[0]); r2[1] = fma(M.hp[k], in[k], r2[1]); }
        const double ot_old = out[nr];
        block_reduce<2, false>(r2, M.red);
        const double ot = -r2[1] + xPx * it_ + coef * ot_old;
        if (t == 0) out[nr] = ot;
        __syncthreads();
        return r2[0] + ot * ot;
      };
      if constexpr (LSMR) {
        itn = lsmr_block(NR, M.rhs, M.V, M.W, M.U, M.z, M.red, st, iter_lim, C_mul, CT_mul);   // (u, v, h, h-bar, x)
      } else {
        double r1[1] = {0};
        for (int k = t; k < NR; k += T) { const double u = M.rhs[k]; M.U[k] = u; r1[0] = fma(u, u, r1[0]); M.V[k] = 0.0; }
        block_reduce<1, false>(r1, M.red);
        const double bnorm = sqrt(r1[0]);
        double beta = bnorm, alfa = 0;
        if (beta > 0) {
          for (int k = t; k < NR; k += T) M.U[k] /= beta;
          __syncthreads();
          alfa = sqrt(CT_mul(M.U, M.V, 0.0));
        }
        if (alfa > 0) for (int k = t; k < NR; k += T) { const double v = M.V[k] / alfa; M.V[k] = v; M.W[k] = v; }
        __syncthreads();
        double rhobar = alfa, phibar = beta, anorm = 0, ddnorm = 0, xxnorm = 0, zz = 0, cs2 = -1, sn2 = 0;
        if (alfa * beta != 0.0) {
          while (itn < iter_lim) {
            itn++;
            beta = sqrt(C_mul(M.V, M.U, -alfa));
            if (beta > 0) {
              for (int k = t; k < NR; k += T) M.U[k] /= beta;
              anorm = sqrt(anorm * anorm + alfa * alfa + beta * beta);
              __syncthreads();
              alfa = sqrt(CT_mul(M.U, M.V, -beta));
              if (alfa > 0) for (int k = t; k < NR; k += T) M.V[k] /= alfa;
            }
            const double rho = hypot(rhobar, beta), cs = rhobar / rho, sn = beta / rho;
            const double theta = sn * alfa;
            rhobar = -cs * alfa;
            const double phi = cs * phibar;
            phibar = sn * phibar;
            const double tau = sn * phi, t1c = phi / rho, t2c = -theta / rho;
            __syncthreads();
            r1[0] = 0;
            for (int k = t; k < NR; k += T) {
              const double wk = M.W[k], dk = wk / rho;
              r1[0] = fma(dk, dk, r1[0]);
              M.z[k] = fma(t1c, wk, M.z[k]);
              M.W[k] = fma(t2c, wk, M.V[k]);
            }
            block_reduce<1, false>(r1, M.red);
            ddnorm += r1[0];
            const double delta = sn2 * rho, gambar = -cs2 * rho, rhs_ = phi - delta * zz, zbar = rhs_ / gambar;
            const double xnorm = sqrt(xxnorm + zbar * zbar);
            const double gamma = hypot(gambar, theta);
            cs2 = gambar / gamma; sn2 = theta / gamma; zz = rhs_ / gamma; xxnorm += zz * zz;
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
      }
    }
    __syncthreads();
    pt.stamp(13);  // q, LSQR
    // ---- r = blkdiag(G,1)^{-1} z :  S rL = zL - A_L P^{-1} zx,  rx = P^{-1}(zx + A_L' rL) ----
    const double rt = M.z[nr];
    matvec_rows(M.Pb, PackedLowerLayout{}, n, n, M.z, [&](int i, double v) { M.tn[i] = v; });              // tn = L^{-1} zx
    __syncthreads();
    if (nl > 0) {
      matvec_rows(Ws, DenseLayout{n}, nl, n, M.tn, [&](int l, double v) { M.tL[l] = M.z[n + l] - v; });
      __syncthreads();
      S_solve();                                                                                              // rL
      for (int l = t; l < nl; l += T) M.ry[M.live[l]] = M.tL[l];
      matvec_cols(Ws, DenseLayout{n}, nl, n, M.tL, M.part, [&](int j, double v) { M.tn[j] += v; }, plW);
    }
    matvec_cols(M.Pb, PackedLowerLayout{}, n, n, M.tn, M.part, [&](int j, double v) { M.t2[j] = v; }, plN);  // rx
    // ---- gradient assembly on every structural entry (SURVEY.md 8a B4) ----
    {
      double *dAo = a.dA + (size_t)inst * S.nnzA;
      if (a.srec) {   // shared matrices: r and pi_y for the batch-summing reduction (shared.cu)
        put_srec(a.srec + (size_t)inst * bc_srec_doubles(n, m), M.t2, M.ry, rt, M.piy, n, m);
      } else {
        for (int k = t; k < S.nnzA; k += T) {
          const int i = k / n, j = k - i * n;
          dAo[k] = M.x[j] * M.ry[i] - M.piy[i] * M.t2[j];
        }
      }
      for (int i = t; i < m; i += T) a.db[(size_t)inst * m + i] = M.piy[i] * rt - M.ry[i];
      for (int j = t; j < n; j += T) a.dc[(size_t)inst * n + j] = M.x[j] * rt - M.t2[j];
      if (a.dP && !a.srec) {
        double *dPo = a.dP + (size_t)inst * S.nnzP;
        for (int k = t; k < S.nnzP; k += T) {
          const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);
          const double gij = (rt * M.x[i] - M.t2[i]) * M.x[j], gji = (rt * M.x[j] - M.t2[j]) * M.x[i];
          dPo[k] = (i == j) ? gij : gij + gji;
        }
      }
      if (t == 0 && a.lsqr_iters) a.lsqr_iters[inst] = itn;
    }
    __syncthreads();
    pt.stamp(14);  // final solve + gradient write
  }
}

#ifndef BC_LSMR
__global__ void __launch_bounds__(512, 1) bwd_block_kernel(const __grid_constant__ BwdArgs a) { bwd_block_body<false>(a); }

extern "C" size_t bc_bwdb_smem_bytes(int n, int m, int threads) { return bwdb_smem_doubles(n, m, threads) * sizeof(double); }
extern "C" const void *bc_bwdb_kernel(int lsmr) { return lsmr ? bc_bwdb_lsmr_kernel() : (const void *)bwd_block_kernel; }
#else
// bwd_block_lsmr.cu: the LSMR kernel, in a translation unit of its own (next to it the LSQR kernel compiles to other code)
__global__ void __launch_bounds__(512, 1) bwd_block_lsmr_kernel(const __grid_constant__ BwdArgs a) { bwd_block_body<true>(a); }

extern "C" const void *bc_bwdb_lsmr_kernel(void) { return (const void *)bwd_block_lsmr_kernel; }
#endif
