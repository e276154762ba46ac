// fwd_fast.cu -- forward solve for dense A with polyhedral cones (zero + nonneg rows): the same operator
// splitting as fwd.cu (same formulas, same termination rules; SURVEY.md 8a F3-F6, the work diffcp/SCS do
// at src/cvxpylayers/interfaces/diffcp_if.py:365,369), re-laid out around what the shared-memory
// micro-benchmarks of tools/microbench.cu showed: the per-iteration products with A were
// bound by shared-memory bandwidth and shuffle throughput, not by FP64 issue.
//
//   * A LIVES IN REGISTERS: thread (R, C) of the 512 keeps the 4 x 10 tile A[4R..4R+3, 10C..10C+9] of the
//     equilibrated matrix for the whole solve (80 of its 128 registers; m n <= 20480).  A x is 40 FMAs per
//     thread + a 10-term partial sum per row through shared memory, A' y is 40 FMAs + a (m/4)-term partial
//     sum per column; neither touches the 160 KB of A again and neither uses a shuffle.
//   * K^{-1} IS EXPLICIT: after the packed Cholesky + inverse (common.cuh) the symmetric n x n inverse
//     Linv' Linv is formed once into the shared memory that staged A, so the linear solve of an iteration is
//     ONE dense product (2 x 10 tiles, same partial-sum scheme) instead of two packed triangular ones.
//   * Ruiz passes run on the register tiles too (row / column maxima through the same partial buffers);
//     P sits in shared memory as a packed symmetric matrix during equilibration and K formation.
//   * The four dot products of the tau root are reduced only over the warps that own an output.
// Everything else (metric, tau root, over-relaxation, adaptive checks, certificates, adaptive scale with
// on-chip re-factorisation, write-back) is the algorithm of fwd.cu verbatim.
#include "common.cuh"

// Sub-phase cycle counters (tools/phase_profile.py) cost registers in the hot loop: compiled in only with -DBC_SUBPROF.
#ifdef BC_SUBPROF
#define SUB_DECL(name) PhaseTimer name; name.start(a.prof)
#define SUB_SKIP(name) name.skip()
#define SUB_STAMP(name, k) name.stamp(k)
#else
#define SUB_DECL(name)
#define SUB_SKIP(name)
#define SUB_STAMP(name, k)
#endif

namespace {

constexpr int FT = 512;          // threads per CTA
constexpr int TR = 4, TC = 10;   // tile of A per thread: columns [0, TCR) in registers, [TCR, TC) in a private shared-memory slot
constexpr int TCR = 8;

// Tile geometry.  CT column tiles x RTu row tiles; with non-zero template arguments every shared-memory offset
// below is a compile-time constant (addresses fold into instruction immediates, reduction loops unroll), which
// is what keeps the iteration loop inside 128 registers next to the 80 of the tile; <0, 0> is the runtime
// fallback for other shapes.
template <int CT_, int RTU_>
struct Geo {
  int ct, rtu;
  __host__ __device__ Geo(int n, int m) : ct((n + TC - 1) / TC), rtu((m + TR - 1) / TR) {}
  __host__ __device__ __forceinline__ int CT() const { return CT_ ? CT_ : ct; }
  __host__ __device__ __forceinline__ int RTu() const { return RTU_ ? RTU_ : rtu; }
  __host__ __device__ __forceinline__ int npad() const { return CT() * TC; }
  __host__ __device__ __forceinline__ int mpad() const { return RTu() * TR; }
  __host__ __device__ __forceinline__ int KR() const { return (npad() / 2) * CT() <= FT ? 2 : 4; }
  __host__ __device__ __forceinline__ int npk() const { return (npad() * (npad() + 1) / 2 + 1) & ~1; }
  __host__ __device__ __forceinline__ int rowsR() const { return mpad() > npad() ? mpad() : npad(); }
  // X region during the iterations: [Kinv npad x kst | partial sums (column partials RTu x npad and row partials
  // rowsR x CT take turns) | private tile slots TR x FT double2]; it also stages A (m x n) for the K formation,
  // and during the Ruiz passes (no Kinv yet) it holds their row partials (oRz).
  // Row stride of Kinv.  The 2 x 10 tiles of kinv_rows are read as double2 by quarter-warps that straddle two tile rows
  // (10 tiles per row, 8 lanes per quarter); with 16-byte units u = KR R kst / 2 + 5 C + c / 2 the two halves collide unless
  // KR kst / 2 = 2 (mod 8): stride 100 costs 60 % extra wavefronts on the 80 KB that every iteration reads, 106 none.
  // (Compile-time geometries only: in the runtime-geometry instantiation one more loop-invariant value pushed the tile products of
  //  the iteration loop into local memory, which costs more than the conflicts do.)
  __host__ __device__ __forceinline__ int kst() const { return (CT_ != 0 && KR() == 2) ? npad() + ((10 - (npad() & 7)) & 7) : npad(); }
  __host__ __device__ __forceinline__ int oXC() const { return npad() * kst(); }
  __host__ __device__ __forceinline__ int szPart() const { const int a = RTu() * npad(), b = rowsR() * CT(); return ((a > b ? a : b) + 1) & ~1; }
  __host__ __device__ __forceinline__ int oPS() const { return oXC() + szPart(); }
  __host__ __device__ __forceinline__ int XD() const { const int it = oPS() + TR * FT * (TC - TCR), stg = mpad() * npad(); return ((it > stg ? it : stg) + 1) & ~1; }
  // Row partials of the Ruiz passes (rowsR x CT), written in the same phase as the column partials at oXC: in the Kinv area,
  // unused then, unless they would reach oXC (m >> n); then behind the private tile slots, where A was staged (ok() checks
  // that they end inside X; XD itself is left alone: its formula feeds every vector offset of the iteration loop).
  __host__ __device__ __forceinline__ int oRz() const { return rowsR() * CT() <= oXC() ? 0 : oPS() + TR * FT * (TC - TCR); }
  // whole block (doubles): [bar, ibuf (4) | X | Li | 9 x-vectors | 7 y-vectors | red (8 x 32) | scalars (64) | Cholesky scratch]
  __host__ __device__ __forceinline__ int oX() const { return 4; }
  __host__ __device__ __forceinline__ int oLi() const { return oX() + XD(); }
  __host__ __device__ __forceinline__ int oVx() const { return oLi() + npk(); }
  __host__ __device__ __forceinline__ int oVy() const { return oVx() + 9 * npad(); }
  __host__ __device__ __forceinline__ int oRed() const { return oVy() + 7 * mpad(); }
  __host__ __device__ __forceinline__ int oCh() const { return oRed() + 256 + 64; }   // Cholesky scratch
  // Its size, 26 ceil(npad / 4) + 2 doubles rounded up to even, is fixed so that the kernel's shared memory (and with it which
  // shapes the kernel accepts) does not depend on the Cholesky routine; ok() checks that the routine's need at FT threads fits.
  __host__ __device__ __forceinline__ int szCh() const { return (26 * ((npad() + 3) >> 2) + 3) & ~1; }
  __host__ __device__ __forceinline__ int total() const { return oCh() + szCh(); }
  // cached set-up of one instance (global memory): [header 8 | E npad | D mpad | Kinv npad x kst]; header = {scale of the
  // stored Kinv, 1.0 once Kinv is stored, rho_x it was built with, ...}
  __host__ __device__ __forceinline__ int cE() const { return 8; }
  __host__ __device__ __forceinline__ int cD() const { return cE() + npad(); }
  __host__ __device__ __forceinline__ int cK() const { return cD() + mpad(); }
  __host__ __device__ __forceinline__ int cTotal() const { return (cK() + npad() * kst() + 1) & ~1; }
  __host__ __device__ __forceinline__ bool ok(int n, int m) const {
    return n <= FT && m <= FT && CT() * RTu() <= FT && ((npad() + KR() - 1) / KR()) * CT() <= FT && chol_scratch_doubles(npad(), FT) <= szCh() &&
           oRz() + rowsR() * CT() <= XD();
  }
};

// Vector slots (x-space: k * npad from oVx; y-space: k * mpad from oVy)
enum { VX_W = 0, VX_U, VX_UT, VX_G, VX_CH, VX_EN, VX_TN, VX_TN2, VX_TN3 };
enum { VY_W = 0, VY_U, VY_UT, VY_G, VY_BH, VY_DM, VY_TM };

__device__ __forceinline__ double inv_ry_f(int z, int i, double scale) { return i < z ? BC_ZERO_CONE_FACTOR * scale : scale; }
__device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }

// ---------------------------------------------------------------- register-tile products
// out_j = sum_i A_ij y_i.  Every active thread folds its 4 rows into 10 column partials, thread j < n adds
// the RTu partials of its column.  ep(j, value) runs on thread j.  One barrier inside, none at the end.
template <class G, class Epi>
__device__ __forceinline__ void rt_cols(const double (&ar)[TR][TCR], const double2 *ps, const G &g, bool act, int R, int C, const double *y,
                                        double *XC, int n, Epi ep, int t = threadIdx.x) {
  if (act) {
    const double2 y01 = *reinterpret_cast<const double2 *>(y + TR * R), y23 = *reinterpret_cast<const double2 *>(y + TR * R + 2);
    double2 *dst = reinterpret_cast<double2 *>(XC + R * g.npad() + TC * C);
    {   // the slot columns first: their loads overlap the register part
      const double2 s0 = ps[0], s1 = ps[FT], s2 = ps[2 * FT], s3 = ps[3 * FT];
      dst[TCR >> 1] = make_double2(fma(s3.x, y23.y, fma(s2.x, y23.x, fma(s1.x, y01.y, s0.x * y01.x))),
                                   fma(s3.y, y23.y, fma(s2.y, y23.x, fma(s1.y, y01.y, s0.y * y01.x))));
    }
#pragma unroll
    for (int c = 0; c < TCR; c += 2) {
      const double q0 = fma(ar[3][c], y23.y, fma(ar[2][c], y23.x, fma(ar[1][c], y01.y, ar[0][c] * y01.x)));
      const double q1 = fma(ar[3][c + 1], y23.y, fma(ar[2][c + 1], y23.x, fma(ar[1][c + 1], y01.y, ar[0][c + 1] * y01.x)));
      dst[c >> 1] = make_double2(q0, q1);
    }
  }
  __syncthreads();
  if (t < n) {
    const double *p = XC + t;
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    int Rr = 0;
#pragma unroll 4
    for (; Rr + 3 < g.RTu(); Rr += 4) {
      s0 += p[Rr * g.npad()]; s1 += p[(Rr + 1) * g.npad()]; s2 += p[(Rr + 2) * g.npad()]; s3 += p[(Rr + 3) * g.npad()];
    }
    for (; Rr < g.RTu(); Rr++) s0 += p[Rr * g.npad()];
    ep(t, (s0 + s1) + (s2 + s3));
  }
}
// out_i = sum_j A_ij x_j.  ep(i, value) runs on thread i < m.  One barrier inside, none at the end.
template <class G, class Epi>
__device__ __forceinline__ void rt_rows(const double (&ar)[TR][TCR], const double2 *ps, const G &g, bool act, int R, int C, const double *x,
                                        double *XR, int m, Epi ep, int t = threadIdx.x) {
  if (act) {
    double s[TR];
    {
      const double2 v = *reinterpret_cast<const double2 *>(x + TC * C + TCR);
#pragma unroll
      for (int r = 0; r < TR; r++) { const double2 q = ps[r * FT]; s[r] = fma(q.y, v.y, q.x * v.x); }
    }
#pragma unroll
    for (int c = 0; c < TCR; c += 2) {
      const double2 v = *reinterpret_cast<const double2 *>(x + TC * C + c);
#pragma unroll
      for (int r = 0; r < TR; r++) s[r] = fma(ar[r][c + 1], v.y, fma(ar[r][c], v.x, s[r]));
    }
#pragma unroll
    for (int r = 0; r < TR; r++) XR[(TR * R + r) * g.CT() + C] = s[r];
  }
  __syncthreads();
  if (t < m) {
    const double *p = XR + t * g.CT();
    double s0 = 0, s1 = 0;
    int c = 0;
#pragma unroll
    for (; c + 1 < g.CT(); c += 2) { s0 += p[c]; s1 += p[c + 1]; }
    if (c < g.CT()) s0 += p[c];
    ep(t, s0 + s1);
  }
}
// out_i = sum_j Kinv_ij x_j for the symmetric inverse stored with row stride npad (KR x 10 tiles read from
// shared memory).  ep(i, value) runs on thread i < n.  One barrier inside, none at the end.
template <int KR, class G, class Epi>
__device__ __forceinline__ void kinv_rows(const double *Kinv, const G &g, int n, int R, int C, const double *x, double *XR, Epi ep, int t) {
  if (KR * R < n) {
    double s[KR];
#pragma unroll
    for (int r = 0; r < KR; r++) s[r] = 0.0;
    const double2 *row = reinterpret_cast<const double2 *>(Kinv + (KR * R) * g.kst() + TC * C);
    const int rs = g.kst() >> 1;   // row stride in double2
#pragma unroll
    for (int c = 0; c < TC; c += 2) {
      const double2 v = *reinterpret_cast<const double2 *>(x + TC * C + c);
#pragma unroll
      for (int r = 0; r < KR; r++) {
        if (KR * R + r < n) { const double2 q = row[r * rs + (c >> 1)]; s[r] = fma(q.y, v.y, fma(q.x, v.x, s[r])); }
      }
    }
#pragma unroll
    for (int r = 0; r < KR; r++) if (KR * R + r < n) XR[(KR * R + r) * g.CT() + C] = s[r];
  }
  __syncthreads();
  if (t < n) {
    const double *p = XR + t * g.CT();
    double s0 = 0, s1 = 0;
    int c = 0;
#pragma unroll
    for (; c + 1 < g.CT(); c += 2) { s0 += p[c]; s1 += p[c + 1]; }
    if (c < g.CT()) s0 += p[c];
    ep(t, s0 + s1);
  }
}
template <class G, class Epi>
__device__ __forceinline__ void kinv_mul(const double *Kinv, const G &g, int n, int R, int C, const double *x, double *XR, Epi ep, int t = threadIdx.x) {
  if (g.KR() == 2) kinv_rows<2>(Kinv, g, n, R, C, x, XR, ep, t); else kinv_rows<4>(Kinv, g, n, R, C, x, XR, ep, t);
}

// Sum of four per-thread values over the block when only the first `nwc` warps hold non-zero terms.
// Two barriers; every thread ends with the same bits.
__device__ __forceinline__ void reduce4_lead(double (&v)[4], double *red, int nwc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp < nwc) {
    const double k = butterfly4(v[0], v[1], v[2], v[3], lane);   // lane 8 q holds the warp sum of value order[q]
    if ((lane & 7) == 0) red[(((lane >> 4) & 1) * 2 + ((lane >> 3) & 1)) * 16 + warp] = k;
  }
  __syncthreads();
  // second stage: lane = 16 * (value >> 1) ... keep it simple: lanes 0..15 sum values 0/1, all lanes read two partials
  {
    const int w = lane & 15;
    double a0 = w < nwc ? red[(lane >> 4) * 16 + w] : 0.0;          // value 0 (lanes 0-15) / value 1 (lanes 16-31)
    double a1 = w < nwc ? red[(2 + (lane >> 4)) * 16 + w] : 0.0;    // value 2 / value 3
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) { a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o); }
    v[0] = __shfl_sync(0xffffffffu, a0, 0); v[1] = __shfl_sync(0xffffffffu, a0, 16);
    v[2] = __shfl_sync(0xffffffffu, a1, 0); v[3] = __shfl_sync(0xffffffffu, a1, 16);
  }
#ifndef BC_OPT_BAR7
  __syncthreads();   // red may be rewritten by the next reduction
#endif
  // (BC_OPT_BAR7: the caller's next barrier -- the one that closes the iteration -- precedes every later write of red)
}

// K = rho_x I + sum_i r_i a_i a_i' (r_i = scale, x 1000 on zero-cone rows) (+ P^ when haveP: K then holds the
// unscaled packed P on entry) for the staged, equilibrated A (row-major m x n in shared memory), packed lower.
// Tensor-core SYRK: a warp owns a 16 x 32 strip of 8 x 8 tiles (two A fragments feed four B fragments per
// k-step of 4 rows), strips touching the lower triangle are dealt round-robin; tiles above the diagonal are
// skipped.  Fragments of the next k-step are loaded while the current DMMAs issue.
__device__ __noinline__ void form_K(const double *Av, int m, int n, int z, double scale, double rho_x, double *K, bool haveP, const double *En) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int fr = lane >> 2, fc = lane & 3;
  const int nb = (n + 7) >> 3, nJP = (nb + 1) >> 1, nKQ = (nb + 3) >> 2;
  const double wz = BC_ZERO_CONE_FACTOR * scale, wl = scale;
  int cnt = 0;
  for (int JP = 0; JP < nJP; JP++)
    for (int KQ = 0; KQ < nKQ; KQ++) {
      if (4 * KQ > 2 * JP + 1) continue;        // strip entirely above the diagonal
      if ((cnt++ % nw) != warp) continue;
      double acc[2][4][2];
      bool need[2][4];
#pragma unroll
      for (int u = 0; u < 2; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) { acc[u][v][0] = acc[u][v][1] = 0.0; need[u][v] = (4 * KQ + v <= 2 * JP + u) && (2 * JP + u < nb); }
      const int jr = 16 * JP + fr, kc = 32 * KQ + fr;
      double fa[2], fb[4], ga[2], gb[4];
      auto load = [&](int i, double (&xa)[2], double (&xb)[4]) {
        const int ii = i + fc;
        const bool valid = ii < m;
        const double *row = Av + ii * n;
        const double w = ii < z ? wz : wl;
#pragma unroll
        for (int u = 0; u < 2; u++) { const int j = jr + 8 * u; xa[u] = (valid && j < n) ? row[j] * w : 0.0; }
#pragma unroll
        for (int v = 0; v < 4; v++) { const int k = kc + 8 * v; xb[v] = (valid && k < n) ? row[k] : 0.0; }
      };
      load(0, fa, fb);
      for (int i = 0; i < m; i += 8) {
        load(i + 4, ga, gb);                      // rows past m load zeros
#pragma unroll
        for (int u = 0; u < 2; u++)
#pragma unroll
          for (int v = 0; v < 4; v++) if (need[u][v]) dmma884(acc[u][v][0], acc[u][v][1], fa[u], fb[v]);
        load(i + 8, fa, fb);
#pragma unroll
        for (int u = 0; u < 2; u++)
#pragma unroll
          for (int v = 0; v < 4; v++) if (need[u][v]) dmma884(acc[u][v][0], acc[u][v][1], ga[u], gb[v]);
      }
#pragma unroll
      for (int u = 0; u < 2; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) {
          if (!need[u][v]) continue;
          const int j = 16 * JP + 8 * u + fr, k = 32 * KQ + 8 * v + 2 * fc;
          if (j < n && k <= j) {
            const int e0 = ((j * (j + 1)) >> 1) + k;
            double v0 = acc[u][v][0] + (j == k ? rho_x : 0.0);
            if (haveP) v0 += K[e0] * En[k] * En[j];
            K[e0] = v0;
            if (k + 1 <= j) {
              double v1 = acc[u][v][1] + (j == k + 1 ? rho_x : 0.0);
              if (haveP) v1 += K[e0 + 1] * En[k + 1] * En[j];
              K[e0 + 1] = v1;
            }
          }
        }
    }
  __syncthreads();
}

// Kinv = X' X for the packed lower-triangular X = L^{-1}: full symmetric n x n with row stride kst (columns [n, npad) zero).
// Tensor-core tiles: Kinv(I, J) = sum over k >= 8 I of X(k, I)' X(k, J) in steps of four rows k (DMMA 8 x 8 x 4); a warp owns
// one block row I (the A fragment) and up to eight tiles J <= I of it, rows dealt round-robin; entries above the diagonal of
// X (not stored) and rows past n enter as zeros.  The mirror image is written with the tile.
#ifdef BC_KINV_SCALAR   // the round-1 version (2 x 2 register tiles on the DFMA pipe), kept for A/B timing
__device__ __noinline__ void form_Kinv(const double *Xp, int n, int npad, int kst, double *Kinv) {
  const int T = blockDim.x, t = threadIdx.x;
  const int nb = (n + 1) >> 1, ntile = (nb * (nb + 1)) >> 1;
  for (int e = t; e < ntile; e += T) {
    int I = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
    while (((I + 1) * (I + 2)) >> 1 <= e) I++;
    while ((I * (I + 1)) >> 1 > e) I--;
    const int J = e - ((I * (I + 1)) >> 1);
    const int i0 = 2 * I, j0 = 2 * J;
    double c00 = 0, c01 = 0, c10 = 0, c11 = 0;
    {   // k = i0: X[k][i0 + 1] is above the diagonal
      const double *row = Xp + ((i0 * (i0 + 1)) >> 1);
      const double a0 = row[i0], b0 = row[j0], b1 = (j0 + 1 <= i0) ? row[j0 + 1] : 0.0;
      c00 = a0 * b0; c01 = a0 * b1;
    }
    for (int k = i0 + 1; k < n; k++) {
      const double *row = Xp + ((k * (k + 1)) >> 1);
      const double a0 = row[i0], a1 = row[i0 + 1], b0 = row[j0], b1 = row[j0 + 1];
      c00 = fma(a0, b0, c00); c01 = fma(a0, b1, c01); c10 = fma(a1, b0, c10); c11 = fma(a1, b1, c11);
    }
    const bool i1 = i0 + 1 < n, j1 = j0 + 1 < n;
    Kinv[i0 * kst + j0] = c00; Kinv[j0 * kst + i0] = c00;
    if (j1) { Kinv[i0 * kst + j0 + 1] = c01; Kinv[(j0 + 1) * kst + i0] = c01; }
    if (i1) { Kinv[(i0 + 1) * kst + j0] = c10; Kinv[j0 * kst + i0 + 1] = c10; }
    if (i1 && j1) { Kinv[(i0 + 1) * kst + j0 + 1] = c11; Kinv[(j0 + 1) * kst + i0 + 1] = c11; }
  }
  __syncthreads();
  for (int k = t; k < n * (npad - n); k += T) { const int i = k / (npad - n), c = n + k % (npad - n); Kinv[i * kst + c] = 0.0; }
  __syncthreads();
}
#else
__device__ __noinline__ void form_Kinv(const double *Xp, int n, int npad, int kst, double *Kinv) {
  const int T = blockDim.x, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = T >> 5;
  const int fr = lane >> 2, fc = lane & 3;
  const int nb = (n + 7) >> 3;
  constexpr int KJ = 4;   // tiles per work item: 8 accumulator registers (this runs with the A tile of the caller live)
  int cnt = 0;
  for (int I = 0; I < nb; I++)
    for (int J0 = 0; J0 <= I; J0 += KJ) {
      if ((cnt++ % nw) != warp) continue;
      const int nJ = min(I - J0 + 1, KJ);
      double acc[KJ][2];
#pragma unroll
      for (int v = 0; v < KJ; v++) acc[v][0] = acc[v][1] = 0.0;
      const int ia = 8 * I + fr;
      for (int k0 = 8 * I; k0 < n; k0 += 4) {
        const int k = k0 + fc;
        const bool kv = k < n;
        const double *row = Xp + ((k * (k + 1)) >> 1);
        const double fa = (kv && ia <= k) ? row[ia] : 0.0;
#pragma unroll
        for (int v = 0; v < KJ; v++)
          if (v < nJ) {   // (warp-uniform)
            const int jb = 8 * (J0 + v) + fr;
            const double fb = (kv && jb <= k) ? row[jb] : 0.0;
            dmma884(acc[v][0], acc[v][1], fa, fb);
          }
      }
#pragma unroll
      for (int v = 0; v < KJ; v++)
        if (v < nJ && ia < n) {
          const int j = 8 * (J0 + v) + 2 * fc;
          const bool mirror = (J0 + v) != I;   // a diagonal tile is complete by itself
          if (j < n) { Kinv[ia * kst + j] = acc[v][0]; if (mirror) Kinv[j * kst + ia] = acc[v][0]; }
          if (j + 1 < n) { Kinv[ia * kst + j + 1] = acc[v][1]; if (mirror) Kinv[(j + 1) * kst + ia] = acc[v][1]; }
        }
    }
  __syncthreads();
  // padding columns [n, npad) must stay finite: the tile products multiply them by zeros of the vectors
  for (int k = t; k < n * (npad - n); k += T) { const int i = k / (npad - n), c = n + k % (npad - n); Kinv[i * kst + c] = 0.0; }
  __syncthreads();
}
#endif

__device__ __noinline__ bool chol_cold(double *K, int n, double *tmp) { return chol_inv_packed(K, n, tmp); }

// Slots of the shared scalar block sc[] (= red + 256): values every thread agrees on but only the cold paths
// need, kept out of the register file.
enum { SC_SIGMA = 0, SC_NB0, SC_NC0, SC_SUMLOG, SC_PREVLR, SC_RP, SC_RD, SC_GAP, SC_UTAU, SC_NLOG, SC_LASTUP, SC_PREVIT,
       SC_NEXT, SC_STATUS, SC_DONE, SC_NEWSCALE, SC_RYZ, SC_RYL, SC_GRG, SC_COUNT, SC_AATAU, SC_AADT, SC_NEXTREAL, SC_AASCR };   // SC_AASCR: 17 slots

// Everything of a termination check after the two products with A (A u_x in tm, A' u_y in tn): P^ u_x, the
// residual norms on the un-normalised data (SURVEY.md 8a F6), termination and certificates, the adaptive
// check schedule and the adaptive-scale decision (including the w_y correction that keeps R (w + u - 2 u~)
// invariant).  A handful of calls per solve and deliberately NOT inlined: the register allocation of the
// iteration loop belongs to the tiles.  Results travel through sc[]; ends with a barrier.
__device__ __noinline__ void check_tail(const FwdArgs &a, double *vx, double *vy, double *red, double *scratch, const double *Pv,
                                        int npad, int mpad, int it, double scale, double tau) {
  const DevStruct &S = a.S;
  const bc_settings &st = a.st;
  const int n = S.n, m = S.m, t = threadIdx.x, z = S.z;
  double *sc = red + 256;
  const double *ux = vx + npad, *ch = vx + 4 * npad, *En = vx + 5 * npad, *tn = vx + 6 * npad;
  double *tn2 = vx + 7 * npad, *tn3 = vx + 8 * npad;
  double *wy = vy;
  const double *uy = vy + mpad, *uty = vy + 2 * mpad, *bh = vy + 4 * mpad, *Dm = vy + 5 * mpad, *tm = vy + 6 * mpad;
  const double sigma = sc[SC_SIGMA], nb0 = sc[SC_NB0], nc0 = sc[SC_NC0];
  double sum_log = sc[SC_SUMLOG], prev_lr = sc[SC_PREVLR];
  int n_log = (int)sc[SC_NLOG], last_up = (int)sc[SC_LASTUP], prev_it = (int)sc[SC_PREVIT], next_check = (int)sc[SC_NEXT];
  int status = BCONE_INACCURATE;
  double rp = sc[SC_RP], rd = sc[SC_RD], gap = sc[SC_GAP], new_scale = 0.0;
  double pxu = 0;
  if (t < n) { tn2[t] = 0.0; tn3[t] = En[t] * ux[t]; }
  __syncthreads();
  if (Pv) {  // P^ u_x = E (P (E u_x))
    const ColPlan plN = make_colplan(n, n);
    P_mul(S, Pv, tn3, scratch, [&](int j, double v) { tn2[j] += v; }, plN);
    if (t < n) pxu = tn2[t] * En[t];
  }
  double sm[3] = {0, 0, 0};   // xPx_u, ctx_u, bty_u
  double mx[7] = {0, 0, 0, 0, 0, 0, 0};  // rp, nAx, nS, nAxs, rd, nPx, nATy
  if (t < m) {
    const double ax = tm[t];
    const double rsk = (uy[t] - (2.0 * uty[t] - wy[t])) / inv_ry_f(z, t, scale);
    const double sc_ = 1.0 / (Dm[t] * sigma);
    mx[0] = fabs(ax + rsk - bh[t] * tau) * sc_;
    mx[1] = fabs(ax) * sc_; mx[2] = fabs(rsk) * sc_;
    mx[3] = fabs(ax + rsk) * sc_;
    sm[2] = bh[t] * uy[t];
  }
  if (t < n) {
    const double aty = tn[t];
    const double sc_ = 1.0 / (En[t] * sigma);
    mx[4] = fabs(pxu + aty + ch[t] * tau) * sc_;
    mx[5] = fabs(pxu) * sc_; mx[6] = fabs(aty) * sc_;
    sm[0] = ux[t] * pxu; sm[1] = ch[t] * ux[t];
  }
  block_reduce<3, false>(sm, red);
  block_reduce<7, true>(mx, red);
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
  if (!done && st.adaptive_scale && n_log > 0 && it - last_up >= BC_RESCALE_MIN_ITERS) {
    const double fac = sqrt(exp(sum_log / n_log));
    if (fac > 3.1622776601683795 || fac < 0.31622776601683794) {
      const double ns = fmin(fmax(scale * fac, BC_MIN_SCALE), BC_MAX_SCALE);
      if (ns != scale) {
        const double ratio = ns / scale;  // r_old / r_new
        if (t < m) wy[t] = ratio * (wy[t] + uy[t] - 2.0 * uty[t]) + 2.0 * uty[t] - uy[t];
        new_scale = ns;
        sum_log = 0; n_log = 0; last_up = it;
      }
    }
  }
  if (t == 0) {
    sc[SC_SUMLOG] = sum_log; sc[SC_PREVLR] = prev_lr; sc[SC_RP] = rp; sc[SC_RD] = rd; sc[SC_GAP] = gap; sc[SC_UTAU] = tau;
    sc[SC_NLOG] = n_log; sc[SC_LASTUP] = last_up; sc[SC_PREVIT] = prev_it; sc[SC_NEXT] = next_check;
    sc[SC_STATUS] = status; sc[SC_DONE] = done ? 1.0 : 0.0; sc[SC_NEWSCALE] = new_scale;
  }
  __syncthreads();
}

// Column maxima of |P^| for one Ruiz pass: four lanes per index over the packed symmetric matrix, folded into tn.
// (A variant with separate row / column walks, running addresses and the factor e_j applied once was slower:
// the pass is bound by the dependent max chain of each lane, not by the index arithmetic.)
__device__ __noinline__ void ruiz_P_part(const double *Pl, const double *En, double *tn, int n) {
  const int t = threadIdx.x, q = t & 3;
  for (int j0 = 0; j0 < n; j0 += blockDim.x >> 2) {   // (block-uniform trip count: the shuffles below see full warps)
    const int j = j0 + (t >> 2);
    double mx = 0;
    if (j < n) {
      const double ej = En[j];
      for (int i = q; i < n; i += 4) {
        const int lo = min(i, j), hi = max(i, j);
        const double p = Pl[((hi * (hi + 1)) >> 1) + lo];
        const double elo = i < j ? En[i] : ej, ehi = i < j ? ej : En[i];
        mx = dmax(mx, fabs(p * elo * ehi));
      }
    }
    mx = dmax(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = dmax(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    if (q == 0 && j < n) tn[j] = dmax(tn[j], mx);
  }
  __syncthreads();
}

// P as a packed symmetric matrix (lower, row j at j(j+1)/2) in the factor's buffer; ends with a barrier.
__device__ __noinline__ void scatter_P(const DevStruct &S, const double *Pg, double *Pl, int npk) {
  const int t = threadIdx.x, T = blockDim.x;
  if (!S.p_dense) { for (int e = t; e < npk; e += T) Pl[e] = 0.0; __syncthreads(); }
  for (int k = t; k < S.nnzP; k += T) {
    const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);   // j >= i
    Pl[((j * (j + 1)) >> 1) + i] = Pg[k];
  }
  __syncthreads();
}

// Cached set-up (global memory, one record per instance; layout in Geo): cold, out of line.
template <bool PUT>
__device__ __noinline__ void cache_vectors(double *rec, double *En, int n, int npad, double *Dm, int m) {
  const int t = threadIdx.x;
  if (PUT) { if (t < n) rec[t] = En[t]; if (t < m) rec[npad + t] = Dm[t]; }
  else { if (t < n) En[t] = rec[t]; if (t < m) Dm[t] = rec[npad + t]; __syncthreads(); }
}
__device__ __noinline__ void cache_put_kinv(double *hd, int offK, const double *Kinv, int n2, double scale, double rho_x) {
  double2 *dst = reinterpret_cast<double2 *>(hd + offK);
  const double2 *src = reinterpret_cast<const double2 *>(Kinv);
  for (int k = threadIdx.x; k < n2; k += blockDim.x) dst[k] = src[k];
  if (threadIdx.x == 0) { hd[0] = scale; hd[1] = 1.0; hd[2] = rho_x; }
}

// Anderson acceleration hooks of the register-tiled kernel.  Events happen at the END of iteration j (w complete),
// which is the oracle's top of iteration j + 1 (nothing happens in between):
//   j = 0 (mod iv): accelerate.  The iterate the last step started from is rebuilt as w - alpha (u - u~) (u, u~ are
//                   still in shared memory), so no event is needed one iteration earlier just to remember it.
//   j = 1 (mod iv): safeguard the step taken from an accelerated point -- scheduled only after a step was taken.
// While the window fills (the first `lookback` events) an event is a few vector copies to the slab in L2.
// ibuf[1] holds the next event's iteration; w_tau travels through sc[SC_AATAU], alpha (u_tau - tau~) through sc[SC_AADT].
__device__ __noinline__ void aa_begin(const FwdArgs &a, int *ibuf) {
  if (threadIdx.x == 0) {
    const int iv = a.st.acceleration_interval > 0 ? a.st.acceleration_interval : 1;
    const bool on = a.aa_ws != nullptr && a.st.acceleration_lookback != 0;
    ibuf[1] = on ? iv : 0x7fffffff;
    ibuf[2] = 0;   // pairs recorded since the last reset (mirror of the slab header)
    if (on) { double *ws = a.aa_ws + (size_t)blockIdx.x * a.aa_stride; ws[0] = 0.0; ws[1] = 0.0; ws[2] = 0.0; ws[3] = 0.0; }
  }
  __syncthreads();
}
// Fill-phase event (fewer than `lookback` pairs recorded, nothing to safeguard): store the raw pair -- x = the iterate the
// last step started from, rebuilt as w - alpha (u - u~); f = w -- into column k of S / D (common.cuh aa_apply_dev turns
// them into difference columns at the first solve).  A dozen registers: cheap to call from the iteration loop.
__device__ __noinline__ void aa_fill_light(const FwdArgs &a, int j, const double *vxb, const double *vyb, int npad, int mpad, const double *sc, int *ibuf) {
  const int iv = a.st.acceleration_interval > 0 ? a.st.acceleration_interval : 1, lb = a.st.acceleration_lookback, mem = lb > 0 ? lb : -lb;
  const int n = a.S.n, m = a.S.m, N = n + m + 1, Np = (N + 1) & ~1, t = threadIdx.x, k = ibuf[2];
  double *ws = a.aa_ws + (size_t)blockIdx.x * a.aa_stride;
  double *Sx = ws + BC_AA_HDR + (size_t)(4 + mem + k) * Np, *Df = Sx + (size_t)mem * Np;
  const double al = a.st.alpha;
  if (t < n) { const double f = vxb[VX_W * npad + t]; Df[t] = f; Sx[t] = f - al * (vxb[VX_U * npad + t] - vxb[VX_UT * npad + t]); }
  if (t < m) { const double f = vyb[VY_W * mpad + t]; Df[n + t] = f; Sx[n + t] = f - al * (vyb[VY_U * mpad + t] - vyb[VY_UT * mpad + t]); }
  __syncthreads();   // everybody has read ibuf[2]
  if (t == 0) { Df[N - 1] = sc[SC_AATAU]; Sx[N - 1] = sc[SC_AATAU] - sc[SC_AADT]; ws[0] = k + 1; ibuf[2] = k + 1; ibuf[1] = j + iv - j % iv; }
  __syncthreads();
}
__device__ __noinline__ void aa_event(const FwdArgs &a, int j, double *vxb, double *vyb, int npad, int mpad, double *sc, double *red, int *ibuf, double *lu) {
  const int iv = a.st.acceleration_interval > 0 ? a.st.acceleration_interval : 1, lb = a.st.acceleration_lookback;
  const int n = a.S.n, m = a.S.m, N = n + m + 1, Np = (N + 1) & ~1, t = threadIdx.x;
  double *ws = a.aa_ws + (size_t)blockIdx.x * a.aa_stride;
  const AaIter w{vxb + VX_W * npad, n, vyb + VY_W * mpad, m, sc + SC_AATAU};
  __syncthreads();   // sc[SC_AATAU], sc[SC_AADT] written by thread 0
  bool pending = false;
  if (j < a.st.max_iters) {
    bool rejected = false;
    if (ws[1] != 0.0) rejected = aa_safeguard_dev(ws, lb, w, red);
    if (j % iv == 0) {
      if (!rejected) {   // w_prev = the iterate this step started from
        double *wprev = ws + BC_AA_HDR + 3 * Np;
        const double *ux = vxb + VX_U * npad, *utx = vxb + VX_UT * npad, *uy = vyb + VY_U * mpad, *uty = vyb + VY_UT * mpad;
        for (int e = t; e < N; e += FT)
          wprev[e] = e < n ? w.wx[e] - a.st.alpha * (ux[e] - utx[e]) : (e < n + m ? w.wy[e - n] - a.st.alpha * (uy[e - n] - uty[e - n]) : sc[SC_AATAU] - sc[SC_AADT]);
      }
      if (aa_apply_dev(ws, lb, w, sc + SC_AASCR, red, lu) > 0.0) { aa_store_prev(ws, lb, w, sc[SC_AATAU]); pending = true; }
    }
  }
  __syncthreads();
  if (t == 0) { ibuf[1] = pending ? j + 1 : j + iv - j % iv; ibuf[2] = (int)ws[0]; }
  __syncthreads();
}

}  // namespace

template <int CT_, int RTU_>
__global__ void __launch_bounds__(FT, 1) fwd_fast_kernel(const __grid_constant__ FwdArgs a) {
  extern __shared__ __align__(16) double sm[];
  const DevStruct &S = a.S;
  const int n = S.n, m = S.m, t = threadIdx.x, z = S.z;
  const bc_settings &st = a.st;
  const Geo<CT_, RTU_> g(n, m);
  uint64_t *bar = (uint64_t *)sm;
  int *ibuf = (int *)(sm + 2);
  double *const X = sm + g.oX(), *const Li = sm + g.oLi(), *const red = sm + g.oRed(), *const sc = red + 256;
  auto vx = [&](int k) { return sm + g.oVx() + k * g.npad(); };
  auto vy = [&](int k) { return sm + g.oVy() + k * g.mpad(); };
  double *const Kinv = X, *const XC = X + g.oXC(), *const XR = XC;   // column / row partials take turns in one buffer
  double2 *const ps = reinterpret_cast<double2 *>(X + g.oPS()) + t;   // private slot r: ps[r * FT] = tile columns 8, 9 of row r
  if (t == 0) { mbar_init(bar, 1); fence_mbar_init(); }
  // vectors: the padding entries are read by the tile products (against zero matrix entries) and must stay finite
  for (int k = t; k < 9 * g.npad() + 7 * g.mpad(); k += FT) sm[g.oVx() + k] = 0.0;
  __syncthreads();
  uint32_t tma_phase = 0;
  const int R = t / g.CT(), C = t - R * g.CT();
  const bool act = R < g.RTu();
  const int nwc = (max(m, n) + 31) >> 5;   // warps owning an output of the products
  const bool p_tma = (S.nnzP % 2 == 0) && (((uintptr_t)a.P_vals & 15) == 0) && ((size_t)S.nnzP * 8 < (1u << 20));
  double ar[TR][TCR];

  for (;;) {
    if (t == 0) {
      const int k = atomicAdd(a.counter, 1);
      ibuf[0] = k;
      int ru = 0;   // cached set-up usable: written by a completed factorisation with the same rho_x
      if (k < a.B && a.cache) {
        double *hd = a.cache + (size_t)k * a.cache_stride;
        ru = a.cache_reuse && hd[1] == 1.0 && hd[2] == a.st.rho_x;
        if (!ru && a.cache_stride) hd[1] = 0.0;   // (a shared record, cache_stride = 0, is never written by the batch)
      }
      ibuf[3] = ru;
    }
    __syncthreads();
    const int inst = ibuf[0];
    if (inst >= a.B) break;
    const double *Pg = (a.P_vals && S.nnzP > 0) ? a.P_vals + (size_t)inst * a.sP : nullptr;
    long long *pt_t0 = reinterpret_cast<long long *>(sc + SC_COUNT);
    if (a.prof && t == 0) *pt_t0 = clock64();
    auto pt_stamp = [&](int k) { if (a.prof && t == 0) { const long long now = clock64(); atomicAdd(a.prof + k, (unsigned long long)(now - *pt_t0)); *pt_t0 = now; } };
    SUB_DECL(pi);

    // ---- stage the instance ----
    {
      const double *Ag = a.A_vals + (size_t)inst * a.sA;
      if (a.use_tma) {
        if (t == 0) {
          fence_proxy_async();
          mbar_expect_tx(bar, (uint32_t)(S.nnzA * sizeof(double)));
          tma_bulk_g2s(X, Ag, (uint32_t)(S.nnzA * sizeof(double)), bar);
        }
      } else {
        for (int k = t; k < S.nnzA; k += FT) X[k] = Ag[k];
      }
    }
    {
      const double *bg = a.b + (size_t)inst * m, *cg = a.c + (size_t)inst * n;
      double v4[2] = {0, 0};
      if (t < m) { const double v = bg[t]; vy(VY_BH)[t] = v; vy(VY_DM)[t] = 1.0; v4[0] = fabs(v); }
      if (t < n) { const double v = cg[t]; vx(VX_CH)[t] = v; vx(VX_EN)[t] = 1.0; v4[1] = fabs(v); }
      block_reduce<2, true>(v4, red);
      if (t == 0) {
        sc[SC_NB0] = v4[0]; sc[SC_NC0] = v4[1];
        sc[SC_SUMLOG] = 0; sc[SC_PREVLR] = 0; sc[SC_NLOG] = 0; sc[SC_LASTUP] = 0; sc[SC_PREVIT] = 0; sc[SC_NEXT] = 0;
        sc[SC_RP] = nan(""); sc[SC_RD] = nan(""); sc[SC_GAP] = nan(""); sc[SC_UTAU] = 0; sc[SC_STATUS] = BCONE_INACCURATE;
      }
    }
    if (Pg && !ibuf[3]) scatter_P(S, Pg, Li, g.npk());   // (a cached set-up needs P only in CSR order, for the checks)
    if (a.use_tma) { mbar_wait(bar, tma_phase); tma_phase ^= 1; }
    __syncthreads();
    // ---- register tiles ----
    auto load_tile = [&]() {   // registers + slots from the staged m x n copy in X (ends with a barrier)
      double2 sl[TR];
#pragma unroll
      for (int r = 0; r < TR; r++) {
        const int i = TR * R + r;
#pragma unroll
        for (int c = 0; c < TCR; c++) { const int j = TC * C + c; ar[r][c] = (act && i < m && j < n) ? X[i * n + j] : 0.0; }
        const int j8 = TC * C + TCR;
        sl[r].x = (act && i < m && j8 < n) ? X[i * n + j8] : 0.0;
        sl[r].y = (act && i < m && j8 + 1 < n) ? X[i * n + j8 + 1] : 0.0;
      }
      __syncthreads();   // every read of the staged copy is done: X is free (partial buffers, slots, later Kinv)
#pragma unroll
      for (int r = 0; r < TR; r++) ps[r * FT] = sl[r];
    };
    load_tile();
    double *const XRz = X + g.oRz();   // row partials of the Ruiz passes
    pt_stamp(0);

    // ---- Ruiz equilibration: A^ = D A E, P^ = E P E (SURVEY.md 8a F4) ----
    if (ibuf[3]) cache_vectors<false>(a.cache + (size_t)inst * a.cache_stride + g.cE(), vx(VX_EN), n, g.npad(), vy(VY_DM), m);   // E and D of the solve that wrote it
    if (st.normalize) {
      for (int pass = ibuf[3] ? st.ruiz_passes : 0; pass < st.ruiz_passes; pass++) {
        SUB_SKIP(pi);
        if (act) {
          double e[TC], d[TR], rowp[TR];
#pragma unroll
          for (int c = 0; c < TC; c += 2) { const double2 v = *reinterpret_cast<const double2 *>(vx(VX_EN) + TC * C + c); e[c] = v.x; e[c + 1] = v.y; }
#pragma unroll
          for (int r = 0; r < TR; r += 2) { const double2 v = *reinterpret_cast<const double2 *>(vy(VY_DM) + TR * R + r); d[r] = v.x; d[r + 1] = v.y; }
          double2 *dst = reinterpret_cast<double2 *>(XC + R * g.npad() + TC * C);
          {
            double c0 = 0, c1 = 0;
#pragma unroll
            for (int r = 0; r < TR; r++) {
              const double2 q = ps[r * FT];
              const double v0 = fabs(q.x) * e[TCR] * d[r], v1 = fabs(q.y) * e[TCR + 1] * d[r];
              c0 = dmax(c0, v0); c1 = dmax(c1, v1);
              rowp[r] = dmax(v0, v1);
            }
            dst[TCR >> 1] = make_double2(c0, c1);
          }
#pragma unroll
          for (int c = 0; c < TCR; c += 2) {
            double c0 = 0, c1 = 0;
#pragma unroll
            for (int r = 0; r < TR; r++) {
              const double v0 = fabs(ar[r][c]) * e[c] * d[r], v1 = fabs(ar[r][c + 1]) * e[c + 1] * d[r];
              c0 = dmax(c0, v0); c1 = dmax(c1, v1);
              rowp[r] = dmax(rowp[r], dmax(v0, v1));
            }
            dst[c >> 1] = make_double2(c0, c1);
          }
#pragma unroll
          for (int r = 0; r < TR; r++) XRz[(TR * R + r) * g.CT() + C] = rowp[r];
        }
        __syncthreads();
        if (t < m) {
          const double *p = XRz + t * g.CT(); double r = 0;
#pragma unroll
          for (int c = 0; c < g.CT(); c++) r = dmax(r, p[c]);
          vy(VY_TM)[t] = r;
        }
        {
          const int j = (n <= 128) ? t - (FT - 128) : t;   // the upper warps take the column maxima when they suffice
          if (j >= 0 && j < n) {
            const double *p = XC + j; double r0 = 0, r1 = 0;
            int Rr = 0;
#pragma unroll 4
            for (; Rr + 1 < g.RTu(); Rr += 2) { r0 = dmax(r0, p[Rr * g.npad()]); r1 = dmax(r1, p[(Rr + 1) * g.npad()]); }
            if (Rr < g.RTu()) r0 = dmax(r0, p[Rr * g.npad()]);
            vx(VX_TN)[j] = dmax(r0, r1);
          }
        }
        __syncthreads();
        SUB_STAMP(pi, 16);
        if (Pg) ruiz_P_part(Li, vx(VX_EN), vx(VX_TN), n);
        SUB_STAMP(pi, 17);
        if (t < m) { const double r = vy(VY_TM)[t]; vy(VY_DM)[t] *= fmin(fmax(r < 1e-8 ? 1.0 : rsqrt(r), BC_EQ_MIN), BC_EQ_MAX); }
        if (t < n) { const double r = vx(VX_TN)[t]; vx(VX_EN)[t] *= fmin(fmax(r < 1e-8 ? 1.0 : rsqrt(r), BC_EQ_MIN), BC_EQ_MAX); }
        __syncthreads();
        SUB_STAMP(pi, 18);
      }
      if (st.ruiz_passes > 0 && act) {   // A^ = D A E on the tiles
        double e[TC], d[TR];
#pragma unroll
        for (int c = 0; c < TC; c += 2) { const double2 v = *reinterpret_cast<const double2 *>(vx(VX_EN) + TC * C + c); e[c] = v.x; e[c + 1] = v.y; }
#pragma unroll
        for (int r = 0; r < TR; r += 2) { const double2 v = *reinterpret_cast<const double2 *>(vy(VY_DM) + TR * R + r); d[r] = v.x; d[r + 1] = v.y; }
#pragma unroll
        for (int r = 0; r < TR; r++) {
#pragma unroll
          for (int c = 0; c < TCR; c++) ar[r][c] *= d[r] * e[c];
          double2 q = ps[r * FT];
          q.x *= d[r] * e[TCR]; q.y *= d[r] * e[TCR + 1];
          ps[r * FT] = q;
        }
      }
    }
    if (a.cache && a.cache_stride && !ibuf[3]) cache_vectors<true>(a.cache + (size_t)inst * a.cache_stride + g.cE(), vx(VX_EN), n, g.npad(), vy(VY_DM), m);
    {
      double v[2] = {0, 0};
      if (t < m) { const double q = vy(VY_DM)[t] * vy(VY_BH)[t]; vy(VY_BH)[t] = q; v[0] = fabs(q); }
      if (t < n) { const double q = vx(VX_EN)[t] * vx(VX_CH)[t]; vx(VX_CH)[t] = q; v[1] = fabs(q); }
      block_reduce<2, true>(v, red);
      double sigma = fmax(v[0], v[1]);
      sigma = (!st.normalize || sigma < 1e-6) ? 1.0 : 1.0 / sigma;
      if (t < m) vy(VY_BH)[t] *= sigma;
      if (t < n) vx(VX_CH)[t] *= sigma;
      if (t == 0) sc[SC_SIGMA] = sigma;
      __syncthreads();
    }
    pt_stamp(1);

    double scale = ibuf[3] ? a.cache[(size_t)inst * a.cache_stride] : st.scale, w_tau = 1.0;
    int it = 0, next_check = st.adaptive_check ? (st.check_interval < 10 ? st.check_interval : 10) : st.check_interval;
    if (t < n) { vx(VX_W)[t] = 0; vx(VX_U)[t] = 0; vx(VX_UT)[t] = 0; }
    if (t < m) { vy(VY_W)[t] = 0; vy(VY_U)[t] = 0; vy(VY_UT)[t] = 0; }
    if (a.x0) {   // warm start: w = u + R^{-1} v at the previous solution; a row with a non-finite value starts cold (see fwd.cu)
      const double sg = sc[SC_SIGMA];
      const double x0 = t < n ? a.x0[(size_t)inst * n + t] : 0.0, y0 = t < m ? a.y0[(size_t)inst * m + t] : 0.0,
                   s0 = t < m ? a.s0[(size_t)inst * m + t] : 0.0;
      if (!__syncthreads_or(!isfinite(x0) || !isfinite(y0) || !isfinite(s0))) {
        if (t < n) vx(VX_W)[t] = x0 * sg / vx(VX_EN)[t];
        if (t < m) { const double d = vy(VY_DM)[t]; vy(VY_W)[t] = y0 * sg / d + s0 * d * sg * inv_ry_f(z, t, scale); }
      }
    }
    __syncthreads();
    bool refactor = true, first = true;
    // Anderson acceleration of w (common.cuh): everything about it lives in aa_event(); the loop only compares the
    // iteration counter with the next event kept in shared memory (ibuf[1]), so the hot path carries no extra state.
    aa_begin(a, ibuf);
    if (t == 0) sc[SC_NEXTREAL] = next_check;
    __syncthreads();
    next_check = min(next_check, ibuf[1]);

    for (it = 1; it <= st.max_iters; it++) {
      if (refactor) {
        // Factorisation at the current scale (the one place it is written, so the tiles stay in registers):
        // stage A^ from the tiles -> K -> Cholesky -> Linv -> Kinv; then g = (R_z + M)^{-1} h and g'Rg.
        SUB_DECL(pf);
        const bool from_cache = first && ibuf[3];   // Kinv at this scale comes from the cached set-up: no staging, K, Cholesky
        const bool c_tma = from_cache && a.use_tma && (((uintptr_t)a.cache & 15) == 0);
        // (the record's address is derived HERE, from a value the compiler cannot prove loop-invariant: hoisted out of the iteration
        //  loop it cost the runtime-geometry instantiation three tile values in local memory)
        int inst_c = ibuf[0];
        asm volatile("" : "+r"(inst_c));
        double *const rec = a.cache ? a.cache + (size_t)inst_c * a.cache_stride : nullptr;
        if (!from_cache) {
        if (!first && Pg) scatter_P(S, Pg, Li, g.npk());   // the factor's buffer held P in CSR order for the checks
        {
          double2 sl[TR];
#pragma unroll
          for (int r = 0; r < TR; r++) sl[r] = ps[r * FT];
          __syncthreads();   // the staged copy overwrites the slots (and Kinv, partials)
          if (act) {
#pragma unroll
            for (int r = 0; r < TR; r++) {
              const int i = TR * R + r;
              if (i < m) {
#pragma unroll
                for (int c = 0; c < TCR; c++) { const int j = TC * C + c; if (j < n) X[i * n + j] = ar[r][c]; }
                const int j8 = TC * C + TCR;
                if (j8 < n) X[i * n + j8] = sl[r].x;
                if (j8 + 1 < n) X[i * n + j8 + 1] = sl[r].y;
              }
            }
          }
        }
        __syncthreads();
        form_K(X, m, n, z, scale, st.rho_x, Li, Pg != nullptr, vx(VX_EN));
        SUB_STAMP(pf, 19);
        const bool okf = chol_cold(Li, n, sm + g.oCh());
#ifdef BC_SUBPROF
        if (a.prof && t == 0) atomicAdd(a.prof + 29, 1ull);   // factorisations (tools/phase_profile.py)
#endif
        if (!okf) { if (t == 0) sc[SC_STATUS] = BCONE_FAILED; if (first) it = 0; break; }
        SUB_STAMP(pf, 21);
        // the tiles come back from the staged copy: nothing has to stay live across the factorisation
        load_tile();
        __syncthreads();
        form_Kinv(Li, n, g.npad(), g.kst(), Kinv);
        if (rec && a.cache_stride) cache_put_kinv(rec, g.cK(), Kinv, (n * g.kst()) >> 1, scale, st.rho_x);   // (shared record: private re-factorisation)
        }
        {   // asynchronous loads behind one barrier phase: P in CSR order into the factor's buffer (for the termination
            // checks) and, with a cached set-up, Kinv
          const double *ck = from_cache ? rec + g.cK() : nullptr;
          const uint32_t pb = (Pg && p_tma) ? (uint32_t)(S.nnzP * sizeof(double)) : 0u, kb = c_tma ? (uint32_t)(n * g.kst() * sizeof(double)) : 0u;
          if (t == 0 && pb + kb) {
            fence_proxy_async();
            mbar_expect_tx(bar, pb + kb);
            if (pb) tma_bulk_g2s(Li, Pg, pb, bar);
            if (kb) tma_bulk_g2s(Kinv, ck, kb, bar);
          }
          if (Pg && !p_tma) for (int k = t; k < S.nnzP; k += FT) Li[k] = Pg[k];
          if (from_cache && !c_tma) for (int k = t; k < n * g.kst(); k += FT) Kinv[k] = ck[k];
        }
        SUB_STAMP(pf, 20);
        if (t == 0) { sc[SC_RYZ] = 1.0 / (BC_ZERO_CONE_FACTOR * scale); sc[SC_RYL] = 1.0 / scale; }
        if (t < m) vy(VY_TM)[t] = vy(VY_BH)[t] * inv_ry_f(z, t, scale);
        __syncthreads();
        rt_cols(ar, ps, g, act, R, C, vy(VY_TM), XC, n, [&](int j, double v) { vx(VX_TN)[j] = vx(VX_CH)[j] - v; });
        if (c_tma) { mbar_wait(bar, tma_phase); tma_phase ^= 1; }   // Kinv (and P) have landed
        __syncthreads();
        kinv_mul(Kinv, g, n, R, C, vx(VX_TN), XR, [&](int j, double v) { vx(VX_G)[j] = v; });
        __syncthreads();
        double acc[1] = {0};
        rt_rows(ar, ps, g, act, R, C, vx(VX_G), XR, m, [&](int i, double v) {
          const double iry = inv_ry_f(z, i, scale), gi = (vy(VY_BH)[i] + v) * iry;
          vy(VY_G)[i] = gi; acc[0] = fma((1.0 / iry) * gi, gi, acc[0]); });
        if (t < n) acc[0] = fma(st.rho_x * vx(VX_G)[t], vx(VX_G)[t], acc[0]);
        block_reduce<1, false>(acc, red);
        if (t == 0) sc[SC_GRG] = acc[0];
        if (Pg && p_tma && !c_tma) { mbar_wait(bar, tma_phase); tma_phase ^= 1; }
        __syncthreads();
        SUB_STAMP(pf, 22);
        pt_stamp(2);
        refactor = false; first = false;
      }
      SUB_SKIP(pi);
      // thread-dependent addresses are re-derived every iteration instead of being kept (and spilled) as loop invariants
      int Ri = R, Ci = C, ti = t;
      asm volatile("" : "+r"(Ri), "+r"(Ci), "+r"(ti));
      const double2 *psi = reinterpret_cast<const double2 *>(X + g.oPS()) + ti;
      rt_cols(ar, psi, g, act, Ri, Ci, vy(VY_W), XC, n, [&](int j, double v) { vx(VX_TN)[j] = st.rho_x * vx(VX_W)[j] - v; }, ti);
      __syncthreads();
      SUB_STAMP(pi, 23);
      // (p_x, p_y go through shared memory and the dot products are taken after the last product: nothing but the
      //  tiles is live across the three products)
      kinv_mul(Kinv, g, n, Ri, Ci, vx(VX_TN), XR, [&](int j, double v) { vx(VX_UT)[j] = v; }, ti);
      __syncthreads();
      SUB_STAMP(pi, 24);
      double d4[4] = {0, 0, 0, 0};   // mu'g, p'Rg, p'Rp, p'mu (R-weighted)
      auto dots = [&](double r, double pk, double wk, double gk) {
        d4[0] = fma(r * wk, gk, d4[0]); d4[1] = fma(r * pk, gk, d4[1]);
        d4[2] = fma(r * pk, pk, d4[2]); d4[3] = fma(r * pk, wk, d4[3]);
      };
      rt_rows(ar, psi, g, act, Ri, Ci, vx(VX_UT), XR, m, [&](int i, double v) {
        const bool zr = i < z;
        const double iry = zr ? BC_ZERO_CONE_FACTOR * scale : scale, wk = vy(VY_W)[i];
        const double py = wk + v * iry;
        vy(VY_UT)[i] = py;
        dots(sc[zr ? SC_RYZ : SC_RYL], py, wk, vy(VY_G)[i]); }, ti);
      if (ti < n) dots(st.rho_x, vx(VX_UT)[ti], vx(VX_W)[ti], vx(VX_G)[ti]);
      SUB_STAMP(pi, 26);
      reduce4_lead(d4, red, nwc);
      SUB_STAMP(pi, 27);
      const double qa = BC_TAU_FACTOR + sc[SC_GRG], qb = d4[0] - 2.0 * d4[1] - BC_TAU_FACTOR * w_tau, qc = d4[2] - d4[3];
      double disc = qb * qb - 4.0 * qa * qc;
      if (disc < 0) disc = 0;
      const double tau_t = (-qb + sqrt(disc)) / (2.0 * qa);
      const bool check = it >= next_check || it == st.max_iters;
      // cone step + relaxation (the relaxation is fused here unless a check needs the plain iterate)
      if (ti < n) {
        const double utk = vx(VX_UT)[ti] - tau_t * vx(VX_G)[ti], wk = vx(VX_W)[ti], uk = 2.0 * utk - wk;
        vx(VX_UT)[ti] = utk; vx(VX_U)[ti] = uk;
        if (!check) vx(VX_W)[ti] = wk + st.alpha * (uk - utk);
      }
      if (ti < m) {
        const double utk = vy(VY_UT)[ti] - tau_t * vy(VY_G)[ti], wk = vy(VY_W)[ti];
        double uk = 2.0 * utk - wk;
        if (ti >= z && ti < z + S.l) uk = fmax(uk, 0.0);
        vy(VY_UT)[ti] = utk; vy(VY_U)[ti] = uk;
        if (!check) vy(VY_W)[ti] = wk + st.alpha * (uk - utk);
      }
      const double u_tau = fmax(2.0 * tau_t - w_tau, 0.0);
      if (!check) w_tau += st.alpha * (u_tau - tau_t);
      __syncthreads();
      SUB_STAMP(pi, 28);
      if (check) {   // an event: a termination check and / or an acceleration event (both rare, both cold)
        if (it >= (int)sc[SC_NEXTREAL] || it == st.max_iters) {
          pt_stamp(3);
          rt_rows(ar, ps, g, act, R, C, vx(VX_U), XR, m, [&](int i, double v) { vy(VY_TM)[i] = v; });
          __syncthreads();   // row and column partials share one buffer
          rt_cols(ar, ps, g, act, R, C, vy(VY_U), XC, n, [&](int j, double v) { vx(VX_TN)[j] = v; });
          __syncthreads();
          {   // the check's register footprint would otherwise keep part of the tile in local memory for the whole loop
            double *pk = a.park + (size_t)blockIdx.x * (TR * TCR * FT) + t;
#pragma unroll
            for (int r = 0; r < TR; r++)
#pragma unroll
              for (int c = 0; c < TCR; c++) pk[(r * TCR + c) * FT] = ar[r][c];
            check_tail(a, vx(0), vy(0), red, XC, Pg ? Li : nullptr, g.npad(), g.mpad(), it, scale, u_tau);
#pragma unroll
            for (int r = 0; r < TR; r++)
#pragma unroll
              for (int c = 0; c < TCR; c++) ar[r][c] = pk[(r * TCR + c) * FT];
          }
          if (t == 0) sc[SC_NEXTREAL] = st.adaptive_check ? sc[SC_NEXT] : (double)(it + st.check_interval);
          const bool done = sc[SC_DONE] != 0.0;
          const double ns = sc[SC_NEWSCALE];
          pt_stamp(4);
          if (done) break;
          if (ns != 0.0) { scale = ns; refactor = true; if (a.aa_ws) { aa_reset_dev(a.aa_ws + (size_t)blockIdx.x * a.aa_stride); if (t == 0) ibuf[2] = 0; } }
        }
        if (it < st.max_iters) {  // (the last iterate keeps w so that s = R(u - t) is recoverable)
          if (t < n) vx(VX_W)[t] += st.alpha * (vx(VX_U)[t] - vx(VX_UT)[t]);
          if (t < m) vy(VY_W)[t] += st.alpha * (vy(VY_U)[t] - vy(VY_UT)[t]);
          w_tau += st.alpha * (u_tau - tau_t);
          __syncthreads();
        }
        if (it >= ibuf[1] && it < st.max_iters && ibuf[2] < abs(st.acceleration_lookback) && it % (st.acceleration_interval > 0 ? st.acceleration_interval : 1) == 0) {
          // acceleration window still filling: record the pair (cheap callee, the tile stays in registers)
          if (t == 0) { sc[SC_AATAU] = w_tau; sc[SC_AADT] = st.alpha * (u_tau - tau_t); }
          __syncthreads();
          aa_fill_light(a, it, vx(0), vy(0), g.npad(), g.mpad(), sc, ibuf);
        } else if (it >= ibuf[1]) {   // acceleration event (every acceleration_interval iterations; never when it is off)
          // The callee chain needs more registers than the tile leaves free.  Parking the tile in the slab for the
          // duration of the call (128 KB per CTA, L2) keeps it out of the call's live set, so the register allocation
          // of the iteration loop is the one without acceleration; the compiler's own answer was to keep a third of
          // the tile in local memory for the whole loop, which slows every iteration.
          double *park = a.park + (size_t)blockIdx.x * (TR * TCR * FT) + t;
#pragma unroll
          for (int r = 0; r < TR; r++)
#pragma unroll
            for (int c = 0; c < TCR; c++) park[(r * TCR + c) * FT] = ar[r][c];
          if (t == 0) { sc[SC_AATAU] = w_tau; sc[SC_AADT] = st.alpha * (u_tau - tau_t); }
          aa_event(a, it, vx(0), vy(0), g.npad(), g.mpad(), sc, red, ibuf, XC);   // (the partial-sum buffer is idle between iterations)
          w_tau = sc[SC_AATAU];
#pragma unroll
          for (int r = 0; r < TR; r++)
#pragma unroll
            for (int c = 0; c < TCR; c++) ar[r][c] = park[(r * TCR + c) * FT];
        }
        next_check = min((int)sc[SC_NEXTREAL], ibuf[1]);
      }
    }
    if (it > st.max_iters) it = st.max_iters;
    __syncthreads();
    pt_stamp(4);
    // ---- write back ----
    {
      int status = (int)sc[SC_STATUS];
      if (status == BCONE_INACCURATE && !(sc[SC_UTAU] > 1e-12)) status = BCONE_FAILED;   // (see fwd.cu: no positive tau at the iteration limit)
      double *xo = a.x + (size_t)inst * n, *yo = a.y + (size_t)inst * m, *so = a.s + (size_t)inst * m;
      if (status == BCONE_SOLVED || status == BCONE_INACCURATE) {
        double tau = sc[SC_UTAU];
        if (!(tau > 1e-12)) tau = 1e-12;
        const double k0 = 1.0 / (sc[SC_SIGMA] * tau);
        if (t < n) xo[t] = vx(VX_EN)[t] * vx(VX_U)[t] * k0;
        if (t < m) {
          const double rsk = (vy(VY_U)[t] - (2.0 * vy(VY_UT)[t] - vy(VY_W)[t])) / inv_ry_f(z, t, scale);
          yo[t] = vy(VY_DM)[t] * vy(VY_U)[t] * k0;
          so[t] = rsk * k0 / vy(VY_DM)[t];
        }
      } else {
        const double qn = nan("");
        if (t < n) xo[t] = qn;
        if (t < m) { yo[t] = qn; so[t] = qn; }
      }
      if (t == 0) {
        a.status[inst] = status; a.iters[inst] = it;
        if (a.resid) { a.resid[inst * 3 + 0] = sc[SC_RP]; a.resid[inst * 3 + 1] = sc[SC_RD]; a.resid[inst * 3 + 2] = sc[SC_GAP]; }
      }
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------- host entry points
// Specialised geometries (compile-time offsets); anything else runs the <0, 0> instantiation.
extern "C" const void *bc_fwdf_kernel(int n, int m) {
  const Geo<0, 0> g0(n, m);
  return g0.CT() == 10 && g0.RTu() == 50 ? (const void *)fwd_fast_kernel<10, 50> : (const void *)fwd_fast_kernel<0, 0>;
}

// (sizes come from the geometry type the launch will instantiate: the padded Kinv stride exists only in the compile-time one)
#define FWDF_GEO(n, m, EXPR)                                                                 \
  do {                                                                                       \
    const Geo<0, 0> g0(n, m);                                                                \
    if (g0.CT() == 10 && g0.RTu() == 50) { const Geo<10, 50> g(n, m); EXPR; }                \
    else { const Geo<0, 0> g(n, m); EXPR; }                                                  \
  } while (0)
extern "C" size_t bc_fwdf_smem_bytes(int n, int m) {
  const Geo<0, 0> g0(n, m);
  if (!g0.ok(n, m)) return (size_t)1 << 40;
  size_t r = 0;
  FWDF_GEO(n, m, r = (size_t)g.total() * sizeof(double));
  return r;
}
extern "C" int bc_fwdf_threads(void) { return FT; }
extern "C" size_t bc_fwdf_cache_doubles(int n, int m) { size_t r = 0; FWDF_GEO(n, m, r = (size_t)g.cTotal()); return r; }
// Eligibility beyond "dense A, polyhedral cones, direct mode" (checked by the caller): the tile grid has to
// cover the matrix with at least half of the threads busy.
extern "C" int bc_fwdf_eligible(int n, int m) {
  const Geo<0, 0> g(n, m);
  return g.ok(n, m) && g.CT() * g.RTu() >= FT / 2;
}
