// bwd_fast.cu -- backward kernel, fast path for the headline shape: dense A (n <= 128), zero +
// nonneg cones only, P absent or a dense upper triangle resident in shared memory.
// Same mathematics as bwd.cu (diffcp's adjoint, SURVEY.md 8a B1-B4; reference call site
// src/cvxpylayers/interfaces/diffcp_if.py:86), different schedule:
//
//  * FUSED OPERATOR PASS.  Every application of M or M' needs A x_part and A' y_part of the same
//    input vector.  One pass over the instance's rows computes both: each A element is read from
//    shared memory once and feeds two FMAs (row dot product -> butterfly reduce inside the warp,
//    column partial -> private registers, combined across warps through 8 slots).  The rows of the
//    symmetric P (upper triangle) ride in the same pass.
//  * LIVE ROWS ONLY.  With the equilibrated LSQR the inactive nonneg rows are eliminated exactly
//    (their unknown is dz_i = 0), so the pass walks a per-instance list of live rows.
//  * MERGED REDUCTIONS.  LSQR's u, v are kept un-normalised (their norms ride as scalars), the
//    tau-row dot products, ||out||^2 and ||w||^2 share one block reduction per operator: two
//    block reductions per LSQR iteration instead of five, ~10 barriers instead of ~30.
#include "common.cuh"

struct FastSmem {
  double *Av, *Pv, *x, *c, *px2c, *piy, *b, *U, *V, *W, *X, *Lsc, *Rsc, *ein, *prow, *part, *red;
  double *Hb;   // LSMR only: its h-bar (U, V, W, X are u, v, h, x)
  int *rows;
  uint64_t *bar;
  int *ibuf;
};

// lsmr: the LSMR variant keeps one more N-vector
__host__ __device__ inline size_t bwdf_smem_doubles(int n, int m, int nnzA, int nnzP, int threads, int lsmr = 0) {
  const size_t N = (size_t)n + m + 1;
  const size_t part = (size_t)8 * n > (size_t)threads ? (size_t)8 * n : (size_t)threads;
  return 4 + (((size_t)nnzA + 1) & ~(size_t)1) + (((size_t)nnzP + 1) & ~(size_t)1) + 3 * (size_t)n + 2 * (size_t)m + (lsmr ? 7 : 6) * N + ((N + 1) & ~(size_t)1) + n +
         part + 3 * 32 + ((size_t)m + n + 2) / 2 + 4;
}

template <bool LSMR = false>
__device__ __forceinline__ void carve_f(FastSmem &M, double *base, int n, int m, int nnzA, int nnzP, int threads) {
  const int N = n + m + 1;
  double *q = base;
  M.bar = (uint64_t *)q; q += 2;
  M.ibuf = (int *)q; q += 2;
  M.Av = q; q += (nnzA + 1) & ~1;
  M.Pv = q; q += (nnzP + 1) & ~1;
  M.ein = q; q += (N + 1) & ~1;                     // 16-byte aligned (double2 loads)
  M.part = q; q += (8 * n > threads ? 8 * n : threads);
  M.x = q; q += n; M.c = q; q += n; M.px2c = q; q += n;
  M.piy = q; q += m; M.b = q; q += m;
  M.U = q; q += N; M.V = q; q += N; M.W = q; q += N; M.X = q; q += N; M.Lsc = q; q += N; M.Rsc = q; q += N;
  if (LSMR) { M.Hb = q; q += N; }
  M.prow = q; q += n;
  M.red = q; q += 3 * 32;
  M.rows = (int *)q;
}

// One fused pass over the row list.  ex = x-part of the effective input in shared memory
// (16-byte aligned); lanes own column PAIRS (2*lane + 64k, +1): A rows are read with 128-bit
// loads, P rows (packed upper triangle, row starts not 16-byte aligned) with 64-bit loads.
// ymul(i) = multiplier of A row i in the column accumulation; P row i uses ex[i].
// repi(row_code, value) is called by one lane per listed row (row_code < m: A row, else P row m+i);
// cepi(j, column_total) once per column by thread j (P's row part is added by the caller via prow).
// n must be even and <= 64*NCH.
template <bool SQ, int NCH, class YMul, class RowEpi, class ColEpi>
__device__ __forceinline__ void fused_pass(const FastSmem &M, int n, int m, int nlist, const double *ex, YMul ymul, RowEpi repi, ColEpi cepi) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5, t = threadIdx.x;
  double2 xr[NCH], acc[NCH];
  const bool tail_ok = 2 * lane + 64 * (NCH - 1) < n;   // the last chunk may be partial
#pragma unroll
  for (int k = 0; k < NCH; k++) {
    acc[k] = make_double2(0.0, 0.0);
    xr[k] = (k < NCH - 1 || tail_ok) ? *reinterpret_cast<const double2 *>(ex + 2 * lane + 64 * k) : make_double2(0.0, 0.0);
  }
  const int ngroups = (nlist + 3) >> 2;
  for (int g = warp; g < ngroups; g += nw) {
    double a[4] = {0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int idx = 4 * g + r;
      if (idx < nlist) {
        const int row = M.rows[idx];
        if (row < m) {
          const double mul = ymul(row);
          const double2 *p2 = reinterpret_cast<const double2 *>(M.Av + row * n) + lane;
#pragma unroll
          for (int k = 0; k < NCH; k++) {
            if (k < NCH - 1 || tail_ok) {
              double2 q = p2[32 * k];
              if (SQ) { q.x *= q.x; q.y *= q.y; }
              a[r] = fma(q.x, xr[k].x, a[r]); a[r] = fma(q.y, xr[k].y, a[r]);
              acc[k].x = fma(q.x, mul, acc[k].x); acc[k].y = fma(q.y, mul, acc[k].y);
            }
          }
        } else {
          const int i = row - m;
          const double mul = ex[i];
          const double *p = M.Pv + (i * n - ((i * (i + 1)) >> 1));
#pragma unroll
          for (int k = 0; k < NCH; k++) {
            const int c0 = 2 * lane + 64 * k, c1 = c0 + 1;
            if (c1 >= i && (k < NCH - 1 || tail_ok)) {
              double q1 = p[c1]; if (SQ) q1 *= q1;
              a[r] = fma(q1, xr[k].y, a[r]);
              if (c1 > i) acc[k].y = fma(q1, mul, acc[k].y);
              if (c0 >= i) {
                double q0 = p[c0]; if (SQ) q0 *= q0;
                a[r] = fma(q0, xr[k].x, a[r]);
                if (c0 > i) acc[k].x = fma(q0, mul, acc[k].x);
              }
            }
          }
        }
      }
    }
    const double tot = butterfly4(a[0], a[1], a[2], a[3], lane);
    if ((lane & 7) == 0) {
      const int idx = 4 * g + ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
      if (idx < nlist) repi(M.rows[idx], tot);
    }
  }
  // column partials: 8 slots, warps w and w+8 share a slot in two phases
  const int slot = warp & 7;
  if (warp < 8) {
#pragma unroll
    for (int k = 0; k < NCH; k++)
      if (k < NCH - 1 || tail_ok) *reinterpret_cast<double2 *>(M.part + slot * n + 2 * lane + 64 * k) = acc[k];
  }
  __syncthreads();
  if (warp >= 8) {
#pragma unroll
    for (int k = 0; k < NCH; k++)
      if (k < NCH - 1 || tail_ok) {
        double2 *q = reinterpret_cast<double2 *>(M.part + slot * n + 2 * lane + 64 * k);
        double2 v = *q; v.x += acc[k].x; v.y += acc[k].y; *q = v;
      }
  }
  __syncthreads();
  if (t < n) {
    const int ns = nw < 8 ? nw : 8;
    double s = 0;
    for (int q = 0; q < ns; q++) s += M.part[q * n + t];
    cepi(t, s);
  }
}

// out <- osc o (Op e) + coef * out, with e = in o isc * iscal (the effective input);
// TRANS: Op = M' (the LSQR system matrix B), else Op = M.  Returns ||out||^2; wn2 is block-summed in place.
// D = diag(d): d_i = 1 on zero rows, [pi_y,i > 0] on nonneg rows.
template <bool TRANS, int NCH>
__device__ __forceinline__ double fast_op(const FastSmem &M, const DevStruct &S, int nlist, double xPx, const double *in,
                                          const double *isc, double iscal, double *out, const double *osc, double coef,
                                          double &wn2) {
  const int n = S.n, m = S.m, N = n + m + 1, t = threadIdx.x, T = blockDim.x;
  for (int k = t; k < N; k += T) M.ein[k] = in[k] * (isc ? isc[k] : 1.0) * iscal;   // effective input
  const double out_t = out[N - 1];
  __syncthreads();
  const double *e = M.ein;
  const double et = e[N - 1];
  double dot = 0, nrm = 0;
  auto ymul = [&](int i) {
    if (TRANS) return -e[n + i];
    return (i < S.z || M.piy[i] > 0) ? e[n + i] : 0.0;
  };
  auto repi = [&](int row, double v) {
    if (row < m) {
      const int i = row, k = n + i;
      const double ey = e[k], bi = M.b[i];
      const bool d = (i < S.z || M.piy[i] > 0);
      double val;
      if (TRANS) { val = d ? v - bi * et : ey; dot = fma(bi, ey, dot); }
      else { const double dey = d ? ey : 0.0; val = -v + bi * et - dey + ey; dot = fma(-bi, dey, dot); }
      const double o = fma(osc ? osc[k] : 1.0, val, coef * out[k]);
      out[k] = o; nrm = fma(o, o, nrm);
    } else {
      M.prow[row - m] = v;
    }
  };
  const bool hasP = S.nnzP > 0;
  auto cepi = [&](int j, double s) {
    double val = s + (hasP ? M.prow[j] : 0.0);
    if (TRANS) { val -= M.px2c[j] * et; dot = fma(M.c[j], e[j], dot); }
    else { val += M.c[j] * et; dot = fma(-M.px2c[j], e[j], dot); }
    const double o = fma(osc ? osc[j] : 1.0, val, coef * out[j]);
    out[j] = o; nrm = fma(o, o, nrm);
  };
  fused_pass<false, NCH>(M, n, m, nlist, e, ymul, repi, cepi);
  double r3[3] = {dot, nrm, wn2};
  block_reduce<3, false>(r3, M.red);
  const double ot = fma(osc ? osc[N - 1] : 1.0, r3[0] + xPx * et, coef * out_t);
  if (t == 0) out[N - 1] = ot;
  wn2 = r3[2];
  return r3[1] + ot * ot;
}

// LSMR: diffcp's mode = "lsmr" (common.cuh lsmr_block) on the same operator, scalings and right-hand side; the kernel
// bwd_fast_lsmr_kernel below.
template <int NCH, bool LSMR>
__device__ __forceinline__ void bwd_fast_body(const BwdArgs &a) {   // (by reference: by value the LSQR kernels compile to other code)
  extern __shared__ __align__(16) double smem[];
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, N = n + m + 1, T = blockDim.x, t = threadIdx.x;
  const bc_settings &st = a.st;
  FastSmem M;
  carve_f<LSMR>(M, smem, n, m, S.nnzA, S.nnzP, T);
  if (t == 0) { mbar_init(M.bar, 1); fence_mbar_init(); }
  __syncthreads();
  uint32_t tma_phase = 0;
  const bool hasP = a.P_vals && S.nnzP > 0;
  const bool pc = st.lsqr_precond != 0;
  const int lo = S.z, hi = S.z + S.l;

  for (;;) {
    if (t == 0) {
      const int k = atomicAdd(a.counter, 1), nwork = a.B_dev ? *a.B_dev : a.B;
      M.ibuf[0] = k < nwork ? (a.inst_list ? a.inst_list[k] : k) : -1;
    }
    __syncthreads();
    const int inst = M.ibuf[0];
    if (inst < 0) break;
    const double *Ag = a.A_vals + (size_t)inst * a.sA;
    const double *Pglob = hasP ? a.P_vals + (size_t)inst * a.sP : nullptr;
    const bool tmaP = a.use_tma && hasP && (S.nnzP % 2 == 0) && (((uintptr_t)a.P_vals & 15) == 0);   // bulk copies need 16-byte aligned sources
    if (a.use_tma) {
      if (t == 0) {
        fence_proxy_async();
        mbar_expect_tx(M.bar, (uint32_t)((S.nnzA + (tmaP ? S.nnzP : 0)) * sizeof(double)));
        tma_bulk_g2s(M.Av, Ag, (uint32_t)(S.nnzA * sizeof(double)), M.bar);
        if (tmaP) tma_bulk_g2s(M.Pv, Pglob, (uint32_t)(S.nnzP * sizeof(double)), M.bar);
      }
    } else {
      for (int k = t; k < S.nnzA; k += T) M.Av[k] = Ag[k];
    }
    if (hasP && !tmaP) for (int k = t; k < S.nnzP; k += T) M.Pv[k] = Pglob[k];
    const double *dxg = a.dx + (size_t)inst * n, *dyg = a.dy + (size_t)inst * m;
    double d2[2] = {0, 0};  // x'dx + y'dy, max |dz|
    for (int j = t; j < n; j += T) {
      const double xj = a.x[(size_t)inst * n + j], d = dxg[j];
      M.x[j] = xj; M.c[j] = a.c[(size_t)inst * n + j]; M.U[j] = d; M.X[j] = 0.0; M.prow[j] = 0.0;
      d2[0] = fma(xj, d, d2[0]); d2[1] = fmax(d2[1], fabs(d));
    }
    for (int i = t; i < m; i += T) {
      const double yi = a.y[(size_t)inst * m + i], si = a.s[(size_t)inst * m + i], vi = yi - si;
      const double pi = (i >= lo && i < hi) ? fmax(vi, 0.0) : vi;
      const double dy = dyg[i], ddy = (i < lo || pi > 0) ? dy : 0.0;   // D dy
      M.b[i] = a.b[(size_t)inst * m + i]; M.piy[i] = pi; M.U[n + i] = ddy; M.X[n + i] = 0.0;
      d2[0] = fma(yi, dy, d2[0]); d2[1] = fmax(d2[1], fabs(ddy));
    }
    {
      double s1[1] = {d2[0]}; block_reduce<1, false>(s1, M.red);
      double m1[1] = {d2[1]}; block_reduce<1, true>(m1, M.red);
      if (t == 0) { M.U[N - 1] = -s1[0]; M.X[N - 1] = 0.0; }
      d2[1] = fmax(m1[0], fabs(s1[0]));
    }
    // ---- live-row list: zero rows + active nonneg rows (all rows in plain mode), then P rows ----
    if (t < 32) {
      int cnt = 0;
      for (int base = 0; base < m; base += 32) {
        const int i = base + t;
        const bool live = i < m && (!pc || i < lo || i >= hi || M.piy[i] > 0);
        const unsigned bal = __ballot_sync(0xffffffffu, live);
        if (live) M.rows[cnt + __popc(bal & ((1u << t) - 1))] = i;
        cnt += __popc(bal);
      }
      if (hasP) for (int i = t; i < n; i += 32) M.rows[cnt + i] = m + i;
      if (t == 0) M.ibuf[1] = cnt + (hasP ? n : 0);
    }
    if (a.use_tma) { mbar_wait(M.bar, tma_phase); tma_phase ^= 1; }
    __syncthreads();
    const int nlist = M.ibuf[1];
    // ---- 2Px + c and x'Px (one fused pass over the P rows only: skip A rows via a zero multiplier) ----
    double xPx = 0;
    if (hasP) {
      const int nA = nlist - n;
      // temporarily walk only the P rows: they are the tail of the list
      const int *saved = M.rows;
      M.rows = (int *)saved + nA;
      double acc1 = 0;
      for (int j = t; j < n; j += T) M.ein[j] = M.x[j];
      __syncthreads();
      fused_pass<false, NCH>(M, n, m, n, M.ein, [&](int) { return 0.0; },
                             [&](int row, double v) { M.prow[row - m] = v; },
                             [&](int j, double s) { const double px = s + M.prow[j]; M.px2c[j] = 2.0 * px + M.c[j]; acc1 = fma(M.x[j], px, acc1); });
      M.rows = (int *)saved;
      double s1[1] = {acc1}; block_reduce<1, false>(s1, M.red);
      xPx = s1[0];
    } else {
      for (int j = t; j < n; j += T) M.px2c[j] = M.c[j];
      __syncthreads();
    }
    int itn = 0;
    if (d2[1] > 1e-8) {
      // ---- diagonal equilibration (2-norm Ruiz on the 0/1-skeleton of M'; oracle: lsqr_equilibrate) ----
      if (pc) {
        double *L = M.Lsc, *R = M.Rsc, *rs = M.V, *cs = M.W;
        for (int k = t; k < N; k += T) {
          double v = 1.0;
          if (k >= n && k < n + m) { const int i = k - n; if (i >= lo && i < hi && !(M.piy[i] > 0)) v = 0.0; }
          L[k] = v; R[k] = v; rs[k] = 0.0; cs[k] = 0.0;
        }
        __syncthreads();
        const int passes = st.ruiz_passes > 0 ? st.ruiz_passes : 10;
        for (int pass = 0; pass < passes; pass++) {
          const double Lt = L[N - 1], Rt = R[N - 1];
          double s2[2] = {0, 0};  // rs[tau], cs[tau]
          // pass 1: in = R.^2  -> row sums of squares (x rows via columns, y rows via row results)
          for (int k = t; k < N; k += T) M.ein[k] = R[k] * R[k];
          __syncthreads();
          fused_pass<true, NCH>(M, n, m, nlist, M.ein, [&](int i) { return M.ein[n + i]; },
                           [&](int row, double v) {
                             if (row < m) { const int k = n + row; const double e1 = M.b[row] * M.b[row] * L[k] * L[k] * Rt * Rt;
                               rs[k] = v * L[k] * L[k] + e1; s2[1] += e1; }
                             else M.prow[row - m] = v; },
                           [&](int j, double s) { const double e1 = M.px2c[j] * M.px2c[j] * L[j] * L[j] * Rt * Rt;
                             rs[j] = (s + (hasP ? M.prow[j] : 0.0)) * L[j] * L[j] + e1; s2[1] += e1; });
          __syncthreads();
          // pass 2: in = L.^2  -> column sums of squares
          for (int k = t; k < N; k += T) M.ein[k] = L[k] * L[k];
          __syncthreads();
          fused_pass<true, NCH>(M, n, m, nlist, M.ein, [&](int i) { return M.ein[n + i]; },
                           [&](int row, double v) {
                             if (row < m) { const int k = n + row; const double e2 = M.b[row] * M.b[row] * Lt * Lt * R[k] * R[k];
                               cs[k] = v * R[k] * R[k] + e2; s2[0] += e2; }
                             else M.prow[row - m] = v; },
                           [&](int j, double s) { const double e2 = M.c[j] * M.c[j] * Lt * Lt * R[j] * R[j];
                             cs[j] = (s + (hasP ? M.prow[j] : 0.0)) * R[j] * R[j] + e2; s2[0] += e2; });
          block_reduce<2, false>(s2, M.red);
          const double ett = xPx * xPx * Lt * Lt * Rt * Rt;
          for (int k = t; k < N; k += T) {
            const double r = (k == N - 1) ? s2[0] + ett : rs[k], c = (k == N - 1) ? s2[1] + ett : cs[k];
            if (L[k] > 0 && r > 1e-300) L[k] /= sqrt(sqrt(r));
            if (R[k] > 0 && c > 1e-300) R[k] /= sqrt(sqrt(c));
          }
          __syncthreads();
        }
        for (int k = t; k < N; k += T) M.U[k] *= L[k];
        __syncthreads();
      }
      const double *Ls = pc ? M.Lsc : nullptr, *Rs = pc ? M.Rsc : nullptr;
      if constexpr (LSMR) {
        // ---- LSMR on B = diag(L) M' diag(R); u, v normalised ----
        const int iter_lim = st.lsqr_iter_lim < 0 ? 2 * N : st.lsqr_iter_lim;
        auto opB = [&](const double *in, double *out, double coef) {   // out <- B in + coef out, ||out||^2
          double dummy = 0;
          const double r = fast_op<true, NCH>(M, S, nlist, xPx, in, Rs, 1.0, out, Ls, coef, dummy);
          __syncthreads();
          return r;
        };
        auto opBT = [&](const double *in, double *out, double coef) {   // out <- B' in + coef out, ||out||^2
          double dummy = 0;
          const double r = fast_op<false, NCH>(M, S, nlist, xPx, in, Ls, 1.0, out, Rs, coef, dummy);
          __syncthreads();
          return r;
        };
        itn = lsmr_block(N, M.U, M.V, M.W, M.Hb, M.X, M.red, st, iter_lim, opB, opBT);   // (u, v, h, h-bar, x)
      } else {
        // ---- LSQR on B = diag(L) M' diag(R); u, v stored un-normalised (u = U/beta, v = V/alfa) ----
        const double eps = 2.220446049250313e-16;
        const double atol = st.lsqr_atol, btol = st.lsqr_btol;
        const double ctol = st.lsqr_conlim > 0 ? 1.0 / st.lsqr_conlim : 0.0;
        const int iter_lim = st.lsqr_iter_lim < 0 ? 2 * N : st.lsqr_iter_lim;
        double r1[1] = {0};
        for (int k = t; k < N; k += T) { r1[0] = fma(M.U[k], M.U[k], r1[0]); M.V[k] = 0.0; }
        block_reduce<1, false>(r1, M.red);
        const double bnorm = sqrt(r1[0]), ibnorm = bnorm > 0 ? 1.0 / bnorm : 0.0;
        double beta = bnorm, alfa = 0, wn2 = 0;
        if (beta > 0) {
          __syncthreads();
          alfa = sqrt(fast_op<false, NCH>(M, S, nlist, xPx, M.U, Ls, 1.0 / beta, M.V, Rs, 0.0, wn2));   // V = B' u
          __syncthreads();
        }
        if (alfa > 0) for (int k = t; k < N; k += T) M.W[k] = M.V[k] / alfa;
        wn2 = (t == 0) ? 1.0 : 0.0;  // ||w_1||^2 = ||v_1||^2 = 1, carried through the next block reduction
        __syncthreads();
        double rhobar = alfa, phibar = beta, anorm = 0, ddnorm = 0, xxnorm = 0, z = 0, cs2 = -1, sn2 = 0;
        if (alfa * beta != 0.0) {
          while (itn < iter_lim) {
            itn++;
            // U = B v - alfa u
            const double nb2 = fast_op<true, NCH>(M, S, nlist, xPx, M.V, Rs, 1.0 / alfa, M.U, Ls, -alfa / beta, wn2);
            const double wnorm2 = wn2;   // ||w_k||^2 of the current w
            beta = sqrt(nb2);
            __syncthreads();
            if (beta > 0) {
              anorm = sqrt(anorm * anorm + alfa * alfa + beta * beta);
              double dummy = 0;
              const double na2 = fast_op<false, NCH>(M, S, nlist, xPx, M.U, Ls, 1.0 / beta, M.V, Rs, -beta / alfa, dummy);  // V = B' u - beta v
              alfa = sqrt(na2);
              __syncthreads();
            }
            // scalar recurrences of LSQR (same quantities as SciPy's; reciprocals shared, stopping
            // ratios compared by cross-multiplication to keep fp64 divisions off the critical path)
            const double rho = sqrt(fma(rhobar, rhobar, beta * beta)), irho = 1.0 / rho;
            const double cs = rhobar * irho, sn = beta * irho;
            const double theta = sn * alfa;
            rhobar = -cs * alfa;
            const double phi = cs * phibar;
            phibar = sn * phibar;
            const double tau = sn * phi;
            const double t1c = phi * irho, t2c = -theta * irho, ialfa = alfa > 0 ? 1.0 / alfa : 0.0;
            wn2 = 0;
            for (int k = t; k < N; k += T) {
              const double wk = M.W[k];
              M.X[k] = fma(t1c, wk, M.X[k]);
              const double wnew = fma(t2c, wk, M.V[k] * ialfa);
              M.W[k] = wnew; wn2 = fma(wnew, wnew, wn2);
            }
            ddnorm = fma(wnorm2, irho * irho, ddnorm);
            const double delta = sn2 * rho, gambar = -cs2 * rho, rhs = phi - delta * z, zbar = rhs / gambar;
            const double xnorm = sqrt(fma(zbar, zbar, xxnorm));
            const double gamma = sqrt(fma(gambar, gambar, theta * theta)), igamma = 1.0 / gamma;
            cs2 = gambar * igamma; sn2 = theta * igamma; z = rhs * igamma; xxnorm = fma(z, z, xxnorm);
            const double acond = anorm * sqrt(ddnorm), rnorm = phibar, arnorm = alfa * fabs(tau);
            const double test1 = rnorm * ibnorm, den2 = fma(anorm, rnorm, eps), den3 = acond + eps;
            const double axb = anorm * xnorm * ibnorm, rtol = fma(atol, axb, btol);
            const double u = 1.1102230246251565e-16;   // 1 + t <= 1  <=>  t <= 2^-53
            int istop = 0;
            if (itn >= iter_lim) istop = 7;
            if (1.0 <= u * den3) istop = 6;
            if (arnorm <= u * den2) istop = 5;
            if (test1 <= u * (1.0 + axb)) istop = 4;
            if (1.0 <= ctol * den3) istop = 3;
            if (arnorm <= atol * den2) istop = 2;
            if (test1 <= rtol) istop = 1;
            if (istop || !(alfa > 0) || !(beta > 0)) break;
          }
        }
      }
      __syncthreads();
      if (pc) { for (int k = t; k < N; k += T) M.X[k] *= M.Rsc[k]; __syncthreads(); }
    }
    // ---- gradient assembly on every structural entry (SURVEY.md 8a B4) ----
    {
      const double rt = M.X[N - 1];
      double *dAo = a.dA + (size_t)inst * S.nnzA;
      if (a.srec) {   // shared matrices: r and pi_y for the batch-summing reduction (shared.cu)
        put_srec(a.srec + (size_t)inst * bc_srec_doubles(n, m), M.X, M.X + n, rt, M.piy, n, m);
      } else {
        for (int k = t; k < S.nnzA; k += T) {   // coalesced stores along the row-major CSR order
          const int i = k / n, j = k - i * n;
          dAo[k] = M.x[j] * M.X[n + i] - M.piy[i] * M.X[j];
        }
      }
      for (int i = t; i < m; i += T) a.db[(size_t)inst * m + i] = M.piy[i] * rt - M.X[n + i];
      for (int j = t; j < n; j += T) a.dc[(size_t)inst * n + j] = M.x[j] * rt - M.X[j];
      if (a.dP && hasP && !a.srec) {
        double *dPo = a.dP + (size_t)inst * S.nnzP;
        for (int k = t; k < S.nnzP; k += T) {
          const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);
          const double gij = (rt * M.x[i] - M.X[i]) * M.x[j], gji = (rt * M.x[j] - M.X[j]) * M.x[i];
          dPo[k] = (i == j) ? gij : gij + gji;
        }
      }
      if (t == 0 && a.lsqr_iters) a.lsqr_iters[inst] = itn;
    }
    __syncthreads();
  }
}

#ifndef BC_LSMR
template <int NCH>
__global__ void __launch_bounds__(512, 1) bwd_fast_kernel(const __grid_constant__ BwdArgs a) { bwd_fast_body<NCH, false>(a); }

extern "C" size_t bc_bwdf_smem_bytes(int n, int m, int nnzA, int nnzP, int threads, int lsmr) {
  return bwdf_smem_doubles(n, m, nnzA, nnzP, threads, lsmr) * sizeof(double);
}
extern "C" const void *bc_bwdf_kernel(int n, int lsmr) {
  if (lsmr) return bc_bwdf_lsmr_kernel(n);
  return n <= 64 ? (const void *)bwd_fast_kernel<1> : (const void *)bwd_fast_kernel<2>;
}
#else
// bwd_fast_lsmr.cu: the LSMR kernels, in a translation unit of their own (next to them the LSQR kernels compile to other code)
template <int NCH>
__global__ void __launch_bounds__(512, 1) bwd_fast_lsmr_kernel(const __grid_constant__ BwdArgs a) { bwd_fast_body<NCH, true>(a); }

extern "C" const void *bc_bwdf_lsmr_kernel(int n) { return n <= 64 ? (const void *)bwd_fast_lsmr_kernel<1> : (const void *)bwd_fast_lsmr_kernel<2>; }
#endif
