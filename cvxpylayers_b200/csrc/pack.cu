// pack.cu -- boundary layout <-> engine layout.
//
// The reference hands its solver interface value matrices with the BATCH AXIS CONTIGUOUS
// (A_eval[nnz_aug, B], q_eval[n+1, B]; src/cvxpylayers/torch/cvxpylayer.py:441-451) and then
// walks them in a per-instance Python loop (diffcp_if.py:57-68).  The engine wants one
// instance's values contiguous so a CTA can stage them with a single TMA bulk copy.  These two
// kernels are that re-packing, fused with the sign flip (A = -A_cvx), the CSC->CSR gather and
// the b_idx scatter: HBM-bound tiled transposes, 128-bit loads along the batch axis.
#include <cuda_runtime.h>
#include "common.cuh"

#define TK 32  // rows of the boundary matrix per tile
#define TI 64  // batch entries per tile

// out[i * ldo + dmap(k)] = sign * in[(roff + smap(k)) * B + i],  k in [0,K), i in [0,B)
// (ldb: row pitch of the boundary tensor in doubles -- B for a whole tensor, the full batch when `in` points at a column
//  slice [lo, lo + B) of it)
__global__ void __launch_bounds__(256) b2e_kernel(const double *__restrict__ in, double *__restrict__ out, int K, int B,
                                                  int ldo, int roff, const int *__restrict__ smap,
                                                  const int *__restrict__ dmap, double sign, long long ldb) {
  __shared__ double tile[TK][TI + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k0 = blockIdx.x * TK, i0 = blockIdx.y * TI;
  const bool vec = ((B & 1) == 0) && ((ldb & 1) == 0) && (((uintptr_t)in & 15) == 0);   // 128-bit accesses need an aligned base (the C ABI takes any pointer)
  for (int kk = ty; kk < TK; kk += 8) {
    const int k = k0 + kk;
    if (k >= K) continue;
    const int r = roff + (smap ? __ldg(smap + k) : k);
    const int i = i0 + 2 * tx;
    const double *p = in + (size_t)r * ldb + i;
    if (vec && i + 1 < B) {
      const double2 v = *reinterpret_cast<const double2 *>(p);
      tile[kk][2 * tx] = v.x; tile[kk][2 * tx + 1] = v.y;
    } else {
      if (i < B) tile[kk][2 * tx] = p[0];
      if (i + 1 < B) tile[kk][2 * tx + 1] = p[1];
    }
  }
  __syncthreads();
  const int k = k0 + tx;
  if (k < K) {
    const int d = dmap ? __ldg(dmap + k) : k;
    for (int ii = ty; ii < TI; ii += 8) {
      const int i = i0 + ii;
      if (i < B) out[(size_t)i * ldo + d] = sign * tile[tx][ii];
    }
  }
}

// out[(roff + dmap(k)) * B + i] = sign * in[i * ldi + smap(k)]
__global__ void __launch_bounds__(256) e2b_kernel(const double *__restrict__ in, double *__restrict__ out, int K, int B,
                                                  int ldi, int roff, const int *__restrict__ smap,
                                                  const int *__restrict__ dmap, double sign, long long ldb) {
  __shared__ double tile[TK][TI + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k0 = blockIdx.x * TK, i0 = blockIdx.y * TI;
  const int k = k0 + tx;
  if (k < K) {
    const int s = smap ? __ldg(smap + k) : k;
    for (int ii = ty; ii < TI; ii += 8) {
      const int i = i0 + ii;
      if (i < B) tile[tx][ii] = in[(size_t)i * ldi + s];
    }
  }
  __syncthreads();
  const bool vec = ((B & 1) == 0) && ((ldb & 1) == 0) && (((uintptr_t)out & 15) == 0);
  for (int kk = ty; kk < TK; kk += 8) {
    const int kq = k0 + kk;
    if (kq >= K) continue;
    const int r = roff + (dmap ? __ldg(dmap + kq) : kq);
    const int i = i0 + 2 * tx;
    double *p = out + (size_t)r * ldb + i;
    if (vec && i + 1 < B) {
      *reinterpret_cast<double2 *>(p) = make_double2(sign * tile[kk][2 * tx], sign * tile[kk][2 * tx + 1]);
    } else {
      if (i < B) p[0] = sign * tile[kk][2 * tx];
      if (i + 1 < B) p[1] = sign * tile[kk][2 * tx + 1];
    }
  }
}

// ---- parameter -> matrix affine map fused into the load stage (SURVEY.md 8f.1) ------------------------------------------
// The reference materialises A_eval = A_param @ p_stack ([nnz_aug, P1] sparse x [P1, B] dense; forward at
// src/cvxpylayers/torch/cvxpylayer.py:443-451, transpose at :33-37) in memory only for the solver interface to read it
// once.  p2e_kernel evaluates the map straight into the engine's instance-contiguous tiles: same tile geometry as
// b2e_kernel, but a tile row is sum_e val_e p_stack[col_e, i] over the CSR row of the parameter matrix (lanes along the
// batch axis: every p_stack read is coalesced) instead of a copy.
//   out[i * ldo + dmap(k)] = sign * sum_{e in row (roff + smap(k))} val[e] * p[col[e] * ldp + i]
// (ldp: row pitch of p_stack -- B, or the full batch when only its first columns are read, as for shared matrices)
__global__ void __launch_bounds__(256) p2e_kernel(const double *__restrict__ p, const int *__restrict__ rptr, const int *__restrict__ cols,
                                                  const double *__restrict__ vals, double *__restrict__ out, int K, int B, int ldo, int roff,
                                                  const int *__restrict__ smap, const int *__restrict__ dmap, double sign, long long ldp) {
  __shared__ double tile[TK][TI + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k0 = blockIdx.x * TK, i0 = blockIdx.y * TI;
  for (int kk = ty; kk < TK; kk += 8) {
    const int k = k0 + kk;
    if (k >= K) continue;
    const int r = roff + (smap ? __ldg(smap + k) : k);
    const int e0 = __ldg(rptr + r), e1 = __ldg(rptr + r + 1);
    const int i = i0 + tx;
    double a0 = 0.0, a1 = 0.0;
    for (int e = e0; e < e1; e++) {
      const double v = __ldg(vals + e);
      const double *col = p + (size_t)(__ldg(cols + e) & 0x3fffffff) * ldp;   // (bit 30: exclusive-column flag of the way back)
      if (i < B) a0 = fma(v, col[i], a0);
      if (i + 32 < B) a1 = fma(v, col[i + 32], a1);
    }
    tile[kk][tx] = a0; tile[kk][tx + 32] = a1;
  }
  __syncthreads();
  const int k = k0 + tx;
  if (k < K) {
    const int d = dmap ? __ldg(dmap + k) : k;
    for (int ii = ty; ii < TI; ii += 8) {
      const int i = i0 + ii;
      if (i < B) out[(size_t)i * ldo + d] = sign * tile[tx][ii];
    }
  }
}
// Transposed map on the way back: dp[col * ldp + i] += sign * val[e] * in[i * ldi + smap(k)] for every entry e of row
// (roff + dmap(k)) of the parameter matrix.  One pass over the engine-layout gradient (tile transposed through shared
// memory exactly like e2b_kernel), then lanes along the batch axis update dp: entries flagged exclusive (the only entry
// of their parameter column, the usual "this matrix entry IS a parameter" case; flag = bit 30 of col) are plain stores,
// the others are fp64 atomic adds (dp is zeroed by the caller).  Column `skip` (the constant 1 row of p_stack) is dropped.
__global__ void __launch_bounds__(256) e2p_kernel(const double *__restrict__ in, const int *__restrict__ rptr, const int *__restrict__ cols,
                                                  const double *__restrict__ vals, double *__restrict__ dp, int K, int B, int ldi, int roff,
                                                  const int *__restrict__ smap, const int *__restrict__ dmap, double sign, int skip, long long ldp) {
  __shared__ double tile[TK][TI + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k0 = blockIdx.x * TK, i0 = blockIdx.y * TI;
  const int k = k0 + tx;
  if (k < K) {
    const int s = smap ? __ldg(smap + k) : k;
    for (int ii = ty; ii < TI; ii += 8) {
      const int i = i0 + ii;
      if (i < B) tile[tx][ii] = in[(size_t)i * ldi + s];
    }
  }
  __syncthreads();
  for (int kk = ty; kk < TK; kk += 8) {
    const int kq = k0 + kk;
    if (kq >= K) continue;
    const int r = roff + (dmap ? __ldg(dmap + kq) : kq);
    const int e0 = __ldg(rptr + r), e1 = __ldg(rptr + r + 1);
    for (int e = e0; e < e1; e++) {
      const int cf = __ldg(cols + e), c = cf & 0x3fffffff;
      if (c == skip) continue;
      const double v = sign * __ldg(vals + e);
      double *row = dp + (size_t)c * ldp + i0;
      if (cf & 0x40000000) {
        if (i0 + tx < B) row[tx] = v * tile[kk][tx];
        if (i0 + tx + 32 < B) row[tx + 32] = v * tile[kk][tx + 32];
      } else {
        if (i0 + tx < B) atomicAdd(row + tx, v * tile[kk][tx]);
        if (i0 + tx + 32 < B) atomicAdd(row + tx + 32, v * tile[kk][tx + 32]);
      }
    }
  }
}
// ---- layer prologue / epilogue on the device (SURVEY.md 8f.3) ----------------------------------------------------------------
// The reference builds p_stack with a chain of expand / permute / reshape / cat / transpose per call
// (_flatten_and_batch_params, src/cvxpylayers/torch/cvxpylayer.py:84-141) and takes the requested variables apart with slices,
// Fortran reshapes and a symmetric scatter (_recover_results, :225-282).  Both are index maps; one launch each:
//   rows_from_param : p_stack[(row0 + k), b] = f(param[b * stride + map[k]])   (stride = 0: an unbatched parameter is broadcast;
//                     map = the Fortran-order flattening; f = log for GP parameters)
//   param_from_rows : its adjoint (sum over the batch for an unbatched parameter; x 1/p for log)
//   gather_cols     : out[b, k] = f(scale[k] * in[b * ld + map[k]])   (slice + svec unpack + reshape of one variable; f = exp for GP)
//   scatter_cols    : its adjoint (atomic: the two triangles of a symmetric variable read the same entry)
__global__ void __launch_bounds__(256) rows_from_param_kernel(const double *__restrict__ param, long long stride, const int *__restrict__ map,
                                                             int K, int B, int op, double *__restrict__ rows) {
  __shared__ double tile[TK][TI + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k0 = blockIdx.x * TK, i0 = blockIdx.y * TI;
  const int k = k0 + tx;
  if (k < K) {
    const int src = map ? __ldg(map + k) : k;
    for (int ii = ty; ii < TI; ii += 8) {
      const int i = i0 + ii;
      if (i < B) { const double v = param[(size_t)i * stride + src]; tile[tx][ii] = op == 2 ? log(v) : v; }
    }
  }
  __syncthreads();
  for (int kk = ty; kk < TK; kk += 8) {
    const int kq = k0 + kk;
    if (kq >= K) continue;
    for (int ii = tx; ii < TI; ii += 32) { const int i = i0 + ii; if (i < B) rows[(size_t)kq * B + i] = tile[kk][ii]; }
  }
}
__global__ void __launch_bounds__(256) param_from_rows_kernel(const double *__restrict__ grows, const double *__restrict__ param, long long stride,
                                                             const int *__restrict__ map, int K, int B, int op, double *__restrict__ gparam) {
  // one thread per (k, b) with b fastest: coalesced reads of the gradient rows; writes are strided (parameters are small) and,
  // for an unbatched parameter (stride 0), reduced over the batch with atomics
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)K * B) return;
  const int k = (int)(e / B), b = (int)(e - (long long)k * B);
  const int dst = map ? __ldg(map + k) : k;
  double g = grows[e];
  if (op == 2) g /= param[(size_t)b * stride + dst];
  if (stride == 0) atomicAdd(gparam + dst, g); else gparam[(size_t)b * stride + dst] = g;
}
__global__ void __launch_bounds__(256) gather_cols_kernel(const double *__restrict__ in, long long ld, const int *__restrict__ map,
                                                         const double *__restrict__ scale, int K, int B, int op, double *__restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)K * B) return;
  const int b = (int)(e / K), k = (int)(e - (long long)b * K);
  double v = in[(size_t)b * ld + __ldg(map + k)] * (scale ? __ldg(scale + k) : 1.0);
  out[e] = op == 1 ? exp(v) : v;
}
__global__ void __launch_bounds__(256) scatter_cols_kernel(const double *__restrict__ gout, const double *__restrict__ out, long long ld,
                                                          const int *__restrict__ map, const double *__restrict__ scale, int K, int B, int op,
                                                          double *__restrict__ gin) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)K * B) return;
  const int b = (int)(e / K), k = (int)(e - (long long)b * K);
  double g = gout[e] * (scale ? __ldg(scale + k) : 1.0);
  if (op == 1) g *= out[e];   // d exp(v) = exp(v) dv
  atomicAdd(gin + (size_t)b * ld + __ldg(map + k), g);
}
extern "C" cudaError_t bc_rows_from_param(const double *param, long long stride, const int *map, int K, int B, int op, double *rows, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  dim3 grid((K + TK - 1) / TK, (B + TI - 1) / TI);
  rows_from_param_kernel<<<grid, 256, 0, st>>>(param, stride, map, K, B, op, rows);
  return cudaGetLastError();
}
extern "C" cudaError_t bc_param_from_rows(const double *grows, const double *param, long long stride, const int *map, int K, int B, int op, double *gparam, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  const long long tot = (long long)K * B;
  param_from_rows_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(grows, param, stride, map, K, B, op, gparam);
  return cudaGetLastError();
}
extern "C" cudaError_t bc_gather_cols(const double *in, long long ld, const int *map, const double *scale, int K, int B, int op, double *out, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  const long long tot = (long long)K * B;
  gather_cols_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(in, ld, map, scale, K, B, op, out);
  return cudaGetLastError();
}
extern "C" cudaError_t bc_scatter_cols(const double *gout, const double *out, long long ld, const int *map, const double *scale, int K, int B, int op, double *gin, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  const long long tot = (long long)K * B;
  scatter_cols_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(gout, out, ld, map, scale, K, B, op, gin);
  return cudaGetLastError();
}

extern "C" cudaError_t bc_p2e(const double *p, const int *rptr, const int *cols, const double *vals, double *out, int K, int B, int ldo, int roff,
                              const int *smap, const int *dmap, double sign, long long ldp, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  dim3 grid((K + TK - 1) / TK, (B + TI - 1) / TI);
  p2e_kernel<<<grid, 256, 0, st>>>(p, rptr, cols, vals, out, K, B, ldo, roff, smap, dmap, sign, ldp);
  return cudaGetLastError();
}
extern "C" cudaError_t bc_e2p(const double *in, const int *rptr, const int *cols, const double *vals, double *dp, int K, int B, int ldi, int roff,
                              const int *smap, const int *dmap, double sign, int skip, long long ldp, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  dim3 grid((K + TK - 1) / TK, (B + TI - 1) / TI);
  e2p_kernel<<<grid, 256, 0, st>>>(in, rptr, cols, vals, dp, K, B, ldi, roff, smap, dmap, sign, skip, ldp);
  return cudaGetLastError();
}

extern "C" cudaError_t bc_b2e(const double *in, double *out, int K, int B, int ldo, int roff, const int *smap,
                              const int *dmap, double sign, long long ldb, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  dim3 grid((K + TK - 1) / TK, (B + TI - 1) / TI);
  b2e_kernel<<<grid, 256, 0, st>>>(in, out, K, B, ldo, roff, smap, dmap, sign, ldb);
  return cudaGetLastError();
}
extern "C" cudaError_t bc_e2b(const double *in, double *out, int K, int B, int ldi, int roff, const int *smap,
                              const int *dmap, double sign, long long ldb, cudaStream_t st) {
  if (K <= 0 || B <= 0) return cudaSuccess;
  dim3 grid((K + TK - 1) / TK, (B + TI - 1) / TI);
  e2b_kernel<<<grid, 256, 0, st>>>(in, out, K, B, ldi, roff, smap, dmap, sign, ldb);
  return cudaGetLastError();
}
