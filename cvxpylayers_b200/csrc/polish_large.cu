// polish_large.cu -- solution polishing for zero + nonneg structures that polish.cu cannot hold on chip (n > 128, or the
// staging buffer does not fit next to the rest): the slab tier of bcone_polish (NumPy twin: tests/polish_ref.py).
//
// The rule and the arithmetic are polish.cu's: live rows L = the zero rows + the nonneg rows with y_i > s_i (nl > n: not
// attempted), d = delta x the largest absolute entry of P and A_L, P + d I = L_P L_P', W = A_L L_P^{-T}, S = d I + W W', then
// `refine` steps of iterative refinement against the unregularised KKT matrix, the same completion, the same acceptance test on
// rp / rd / gap and the same flags.  What differs is where the data lives and how the O(n^3) work is laid out:
//   * One persistent CTA per instance, as in polish.cu, but everything of the instance -- the live-row list, the n- and
//     m-vectors, L_P^{-1}, W and S -- sits in the CTA's slab of global memory (bc_polish_large_slab_doubles); only the reduction
//     scratch and the two GEMM panels are in shared memory.
//   * Without P, or with only diagonal P entries (decided at bcone_create), L_P^{-1} is the vector 1 / sqrt(P_jj + d) and W is
//     A_L with its columns scaled; no n x n factor is formed.  Otherwise P + d I is factorised and inverted in place by
//     chol_inv_packed (the on-chip kernel's routine, here on the slab).
//   * W = A_L L_P^{-T} (in place over the staged rows) and S = W W' run as 64 x 64 output blocks on DMMA tiles, their operands
//     staged through shared memory in panels of 32 columns, so each slab element is read O(size / 64) times instead of once per
//     8 x 8 tile.  S is factorised and inverted in place by chol_inv_packed, and the KKT solves are products with the explicit
//     inverses, as on chip.
// The file is self-contained apart from common.cuh's unchanged helpers: polish.cu's live-row, completion and metrics code is
// written out again here rather than shared, because moving it into common.cuh would change the SASS of polish.cu's kernels
// (the precedent is the LSMR translation units, DESIGN.md section 3).  The slab's matrices are read with plain loads (never
// through the read-only path: the kernel writes them).
#include "common.cuh"

namespace {
constexpr int PL_THREADS = 512;            // 16 warps: each owns 4 of the 64 8 x 8 tiles of an output block
constexpr int PL_KP = 32, PL_LD = PL_KP + 4;   // panel width; row pitch of a staged panel (conflict-free fragment reads)

__host__ __device__ inline long long pl_even(long long v) { return (v + 1) & ~1LL; }

struct PlSlab {
  int *live;
  double *c, *x, *tv, *r1, *dx, *aty, *px, *bv, *y, *s, *ax, *r2, *dyl, *yl, *tmp, *Pb, *W, *Sb;
};

// Slab of one CTA: live list | c x tv r1 dx aty px (n) | bv y s ax r2 dyl yl (m) | chol scratch | L_P^{-1} (packed, or n) |
// W (min(m, n) x n) | S (packed, min(m, n))
__host__ __device__ inline long long pl_slab_doubles(int n, int m, int threads, int p_diag) {
  const long long k = n < m ? n : m;
  return pl_even((m + 1) / 2) + 7LL * n + 7LL * m + pl_even(chol_scratch_doubles(n, threads)) +
         pl_even(p_diag ? (long long)n : (long long)n * (n + 1) / 2) + k * n + pl_even(k * (k + 1) / 2);
}

__device__ __forceinline__ PlSlab carve_slab(double *q, int n, int m, int threads, int p_diag) {
  PlSlab M;
  const long long k = n < m ? n : m;
  M.live = (int *)q; q += pl_even((m + 1) / 2);
  M.c = q; q += n; M.x = q; q += n; M.tv = q; q += n; M.r1 = q; q += n; M.dx = q; q += n; M.aty = q; q += n; M.px = q; q += n;
  M.bv = q; q += m; M.y = q; q += m; M.s = q; q += m; M.ax = q; q += m; M.r2 = q; q += m; M.dyl = q; q += m; M.yl = q; q += m;
  M.tmp = q; q += pl_even(chol_scratch_doubles(n, threads));
  M.Pb = q; q += pl_even(p_diag ? (long long)n : (long long)n * (n + 1) / 2);
  M.W = q; q += k * n;
  M.Sb = q;
  return M;
}

// out_i = sum_c M(i, c) x_c for a row-oriented matrix of the slab: one warp per row.  ep(i, v) is called by one lane.
template <class Layout, class Epi>
__device__ __forceinline__ void slab_rows(const double *M, Layout lay, int nrows, const double *x, Epi ep) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int i = warp; i < nrows; i += nw) {
    const double *p = M + lay.base(i);
    double acc = 0.0;
    for (int c = lay.beg(i) + lane; c < lay.end(i); c += 32) acc = fma(p[c], x[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) ep(i, acc);
  }
}

// out_j = sum_i M(i, j) y_i: a thread per (column, chunk of rows), the chunk partials combined through part (blockDim.x
// doubles) in a fixed order.  ep(j, v) is called once per column.  Ends synchronised.
template <class Layout, class Epi>
__device__ __forceinline__ void slab_cols(const double *M, Layout lay, int nrows, int ncols, const double *y, double *part, Epi ep) {
  const int T = blockDim.x, t = threadIdx.x;
  if (ncols <= T) {
    const int CH = T / ncols, j = t % ncols, c = t / ncols;
    double acc = 0.0;
    if (c < CH) {
      const int hi = min((int)(((long long)(c + 1) * nrows) / CH), lay.row_hi(j, nrows));
      for (int i = max((int)(((long long)c * nrows) / CH), lay.row_lo(j)); i < hi; i++) acc = fma(M[lay.base(i) + j], y[i], acc);
    }
    part[t] = acc;
    __syncthreads();
    if (t < ncols) {
      double v = 0.0;
      for (int cc = 0; cc < CH; cc++) v += part[cc * ncols + t];
      ep(t, v);
    }
  } else {
    for (int j = t; j < ncols; j += T) {
      double acc = 0.0;
      const int hi = lay.row_hi(j, nrows);
      for (int i = lay.row_lo(j); i < hi; i++) acc = fma(M[lay.base(i) + j], y[i], acc);
      ep(j, acc);
    }
  }
  __syncthreads();
}

// One 64 x 64 output block C[r][q] = sum_{k < klim} X(r, k) Y(q, k), r in [r0, r0 + 64), q in [q0, q0 + 64), on DMMA tiles
// with both operands staged through shared memory (Xs, Ys: 64 x PL_LD doubles each) in panels of PL_KP columns.  xat / yat
// return the operand entries (0 outside the matrices).  ep(r, q, v) is called once per entry of the block, after every read of
// the operands (so it may overwrite them).
template <class FX, class FY, class Epi>
__device__ __forceinline__ void block64(int r0, int q0, int klim, FX xat, FY yat, double *Xs, double *Ys, Epi ep) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, fr = lane >> 2, fc = lane & 3;
  double acc[4][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
  for (int k0 = 0; k0 < klim; k0 += PL_KP) {
    for (int e = t; e < 64 * PL_KP; e += PL_THREADS) {
      const int r = e / PL_KP, kk = e % PL_KP, k = k0 + kk;
      Xs[r * PL_LD + kk] = k < klim ? xat(r0 + r, k) : 0.0;
      Ys[r * PL_LD + kk] = k < klim ? yat(q0 + r, k) : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int tile = warp + 16 * u, ti = tile >> 3, tj = tile & 7;
      const double *xa = Xs + (8 * ti + fr) * PL_LD + fc, *yb = Ys + (8 * tj + fr) * PL_LD + fc;
#pragma unroll
      for (int ks = 0; ks < PL_KP / 4; ks++) dmma884(acc[u][0], acc[u][1], xa[4 * ks], yb[4 * ks]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; u++) {
    const int tile = warp + 16 * u, ti = tile >> 3, tj = tile & 7;
    const int r = r0 + 8 * ti + fr, q = q0 + 8 * tj + 2 * fc;
    ep(r, q, acc[u][0]);
    ep(r, q + 1, acc[u][1]);
  }
}

template <bool DENSE>
__device__ __forceinline__ void polish_large_body(const PolishLargeArgs &g) {
  extern __shared__ __align__(16) double smem[];
  const PolishArgs &a = g.a;
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, T = blockDim.x, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = T >> 5;
  const int pdg = g.p_diag;
  int *ibuf = (int *)smem;
  double *red = smem + 2, *part = red + 4 * 32, *Xs = part + T, *Ys = Xs + 64 * PL_LD;
  PlSlab M = carve_slab(g.ws + (size_t)blockIdx.x * g.ws_stride, n, m, T, pdg);
  const int z = S.z;   // rows [0, z) zero cone, [z, m) nonneg
  const ColPlan plN = make_colplan(n, n), plA = make_colplan(m, n);

  for (;;) {
    if (t == 0) ibuf[0] = atomicAdd(a.counter, 1);
    __syncthreads();
    const int inst = ibuf[0];
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
      AT_mul<DENSE>(S, Ag, M.y, part, [&](int j, double v) { M.aty[j] = v; }, plA);   // (ends synchronised)
      if (S.nnzP > 0) P_mul(S, Pg, M.x, part, [&](int i, double v) { M.px[i] += v; }, plN);
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
      block_reduce<2, true>(mx, red);
      block_reduce<1, false>(sm, red);
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
      if (lane == 0) ibuf[1] = cnt;
    }
    __syncthreads();
    const int nl = ibuf[1];
    if (nl > n) {
      if (t == 0) a.polished[inst] = -1;
      continue;
    }
    // ---- stage A_L into W (dense: coalesced row loads; CSR: scattered into zeroed dense rows, one warp per row) and P ----
    double *W = M.W, *Sb = M.Sb, *Pb = M.Pb;
    const int np = pdg ? n : (n * (n + 1)) / 2;
    if (DENSE) {
      for (int e = t; e < nl * n; e += T) { const int l = e / n, j = e - l * n; W[e] = Ag[(size_t)M.live[l] * n + j]; }
    } else {
      for (int e = t; e < nl * n; e += T) W[e] = 0.0;
    }
    for (int e = t; e < np; e += T) Pb[e] = 0.0;
    __syncthreads();
    if (!DENSE) {
      for (int l = warp; l < nl; l += nw) {
        const int i = M.live[l], e = __ldg(S.A_indptr + i + 1);
        for (int k = __ldg(S.A_indptr + i) + lane; k < e; k += 32) W[l * n + __ldg(S.A_indices + k)] = Ag[k];
      }
    }
    for (int k = t; k < S.nnzP; k += T) {   // upper row-major CSR -> lower row-major packed (or the diagonal)
      const int i = __ldg(S.P_rowof + k), cc = __ldg(S.P_indices + k);
      Pb[pdg ? i : ((cc * (cc + 1)) >> 1) + i] = Pg[k];
    }
    __syncthreads();
    // ---- d = delta max(|P|_max, |A_L|_max); P + d I = L L' (diagonal: L^{-1} = 1 / sqrt(P_jj + d)) ----
    double dm[1] = {0.0};
    for (int e = t; e < np; e += T) dm[0] = fmax(dm[0], fabs(Pb[e]));
    for (int e = t; e < nl * n; e += T) dm[0] = fmax(dm[0], fabs(W[e]));
    block_reduce<1, true>(dm, red);
    const double d = a.delta * (dm[0] > 0.0 ? dm[0] : 1.0);
    bool ok;
    if (pdg) {
      bool pd = true;
      for (int j = t; j < n; j += T) { const double v = Pb[j] + d; pd &= v > 0.0; Pb[j] = 1.0 / sqrt(v); }
      ok = __syncthreads_and(pd);
    } else {
      for (int j = t; j < n; j += T) Pb[((j * (j + 1)) >> 1) + j] += d;
      __syncthreads();
      ok = chol_inv_packed(Pb, n, M.tmp);   // Pb <- L^{-1}
      __syncthreads();
    }
    if (ok && nl > 0) {
      // ---- W = A_L L^{-T} in place ----
      if (pdg) {
        for (int e = t; e < nl * n; e += T) W[e] *= Pb[e % n];
      } else {
        // 64-row blocks of W; within one, column blocks from the right: block (rb, cb) reads columns < 64 cb + 64 of its rows
        // and then overwrites columns [64 cb, 64 cb + 64), which no block to its left reads
        const int nrb = (nl + 63) >> 6, ncb = (n + 63) >> 6;
        for (int rb = 0; rb < nrb; rb++)
          for (int cb = ncb - 1; cb >= 0; cb--)
            block64(
                64 * rb, 64 * cb, min(n, 64 * cb + 64),
                [&](int r, int k) { return r < nl ? W[r * n + k] : 0.0; },
                [&](int q, int k) { return q < n && k <= q ? Pb[((q * (q + 1)) >> 1) + k] : 0.0; }, Xs, Ys,
                [&](int r, int q, double v) { if (r < nl && q < n) W[r * n + q] = v; });
      }
      __syncthreads();
      // ---- S = d I + W W' (packed lower) in 64 x 64 blocks on and below the diagonal ----
      {
        const int nb = (nl + 63) >> 6;
        auto wat = [&](int r, int k) { return r < nl ? W[r * n + k] : 0.0; };
        for (int ab = 0; ab < nb; ab++)
          for (int bb = 0; bb <= ab; bb++)
            block64(64 * ab, 64 * bb, n, wat, wat, Xs, Ys,
                    [&](int r, int q, double v) { if (r < nl && q <= r) Sb[((r * (r + 1)) >> 1) + q] = v + (q == r ? d : 0.0); });
      }
      __syncthreads();
      ok = chol_inv_packed(Sb, nl, M.tmp);   // Sb <- L_S^{-1}
      __syncthreads();
    }
    if (!ok) {
      if (t == 0) a.polished[inst] = 0;
      continue;
    }
    // [dx; dyl] = K_d^{-1} [r1; r2]:  S dyl = W L^{-1} r1 - r2,  dx = L^{-T} (L^{-1} r1 - W' dyl)   (r2 is overwritten)
    auto kkt_solve = [&]() {
      if (pdg) for (int j = t; j < n; j += T) M.tv[j] = Pb[j] * M.r1[j];
      else slab_rows(Pb, PackedLowerLayout{}, n, M.r1, [&](int i, double v) { M.tv[i] = v; });
      __syncthreads();
      if (nl > 0) {
        slab_rows(W, DenseLayout{n}, nl, M.tv, [&](int l, double v) { M.dyl[l] = v - M.r2[l]; });
        __syncthreads();
        slab_rows(Sb, PackedLowerLayout{}, nl, M.dyl, [&](int i, double v) { M.r2[i] = v; });
        __syncthreads();
        slab_cols(Sb, PackedLowerLayout{}, nl, nl, M.r2, part, [&](int j, double v) { M.dyl[j] = v; });
        slab_cols(W, DenseLayout{n}, nl, n, M.dyl, part, [&](int j, double v) { M.tv[j] -= v; });
      }
      if (pdg) { for (int j = t; j < n; j += T) M.dx[j] = Pb[j] * M.tv[j]; __syncthreads(); }
      else slab_cols(Pb, PackedLowerLayout{}, n, n, M.tv, part, [&](int j, double v) { M.dx[j] = v; });
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
}  // namespace

__global__ void __launch_bounds__(PL_THREADS, 1) polish_large_dense_kernel(const __grid_constant__ PolishLargeArgs g) { polish_large_body<true>(g); }
__global__ void __launch_bounds__(PL_THREADS, 1) polish_large_csr_kernel(const __grid_constant__ PolishLargeArgs g) { polish_large_body<false>(g); }

extern "C" long long bc_polish_large_slab_doubles(int n, int m, int threads, int p_diag) { return pl_slab_doubles(n, m, threads, p_diag); }
extern "C" size_t bc_polish_large_smem_bytes(int threads) { return (2 + 4 * 32 + (size_t)threads + 2 * 64 * PL_LD) * sizeof(double); }
extern "C" int bc_polish_large_threads(void) { return PL_THREADS; }
extern "C" const void *bc_polish_large_kernel(int dense) {
  return dense ? (const void *)polish_large_dense_kernel : (const void *)polish_large_csr_kernel;
}
