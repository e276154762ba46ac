// shared.cu -- batch-summed matrix gradient of a batch that shares A and P (bcone_vjp_shared).
//
// With shared matrices the backward kernels do not assemble dA / dP per instance; each writes its instance's
//   r = (r_x [n], r_y [m], r_tau) and pi_y [m]   (layout at put_srec, bc_srec_doubles apart)
// to a per-call scratch, and this reduction forms the batch sums on the structural entries:
//   dA_sum[k] = sum_b  x_b[j] r_y,b[i] - pi_y,b[i] r_x,b[j]                              (k = (i, j) of A)
//   dP_sum[k] = sum_b  g_ij + (i != j) g_ji,   g_ij = (r_tau,b x_b[i] - r_x,b[i]) x_b[j]  (k = (i, j), i <= j, of P)
// i.e. exactly the per-instance terms bwd.cu / bwd_fast.cu / bwd_block.cu would have written, summed over b.
//
// Dense patterns are matrix products over the batch, run on the FP64 tensor cores (dmma884, one warp per 8 x 8 output tile):
//   dense A:  dA_sum = [r_y | -pi_y] [x | r_x]^T, an [m x 2B] . [2B x n] product (instance b contributes the two k-columns
//             (r_y,b, x_b) and (-pi_y,b, r_x,b));
//   dense P:  G = sum_b w_b x_b^T with w_b = r_tau,b x_b - r_x,b, an [n x B] . [B x n] product; dP_sum[(i, j)] = G_ij + G_ji
//             off the diagonal, G_ii on it.
// CSR patterns use a sampled product: one thread per structural entry, summing over its chunk of the batch.
//
// Determinism: the batch is split into fixed chunks (by B alone); stage 1 reduces each chunk into a partial row (the tensor
// core's accumulation order is fixed, the sampled loop runs in instance order), stage 2 sums the partial rows in chunk order.
// No floating-point atomics: two runs give identical bits.
#include <cuda_runtime.h>
#include "common.cuh"

namespace {
constexpr int SR_THREADS = 256;
constexpr int SR_TILE_WARPS = 4;   // warps (8 x 8 output tiles) per CTA of the tensor-core kernels
constexpr int SR_MAX_CHUNKS = 32;
constexpr int SR_MIN_CHUNK = 64;   // instances per chunk at least (short chunks only add partials)

// dense A: warp w of the grid owns output tile (ti, tj) = rows [8 ti, 8 ti + 8) x columns [8 tj, 8 tj + 8) of the m x n gradient
// and reduces instances [b0, b1) of its chunk into part[chunk][i n + j].  Fragments (PTX m8n8k4): lane holds A[fr][fc] and
// B[fc][fr], fr = lane / 4, fc = lane % 4; k-step s covers instances b0 + 2 s (k = 0, 1) and b0 + 2 s + 1 (k = 2, 3).
__global__ void __launch_bounds__(32 * SR_TILE_WARPS) shared_grad_A_dense(int n, int m, const double *__restrict__ rec,
                                                                         const double *__restrict__ x, int B, int chunk,
                                                                         double *__restrict__ part) {
  const int lane = threadIdx.x & 31, tiles_n = (n + 7) >> 3, tile = blockIdx.x * SR_TILE_WARPS + (threadIdx.x >> 5);
  if (tile >= tiles_n * ((m + 7) >> 3)) return;
  const int ti = tile / tiles_n, tj = tile - ti * tiles_n, fr = lane >> 2, fc = lane & 3;
  const long long R = bc_srec_doubles(n, m);
  const int i = 8 * ti + fr, j = 8 * tj + fr, second = fc & 1;   // second: the (-pi_y, r_x) column of an instance
  const bool iok = i < m, jok = j < n;
  const int b0 = blockIdx.y * chunk, b1 = min(B, b0 + chunk);
  // A operand: r_y[i] or -pi_y[i]; B operand: x[j] or r_x[j] -- of instance b0 + 2 s + fc / 2
  const double *ra = rec + (long long)(b0 + (fc >> 1)) * R + n + (second ? m + 1 : 0) + (iok ? i : 0);
  const double *rb = second ? rec + (long long)(b0 + (fc >> 1)) * R + (jok ? j : 0) : x + (size_t)(b0 + (fc >> 1)) * n + (jok ? j : 0);
  const long long sa = 2 * R, sb = second ? 2 * R : 2LL * n;
  double d0 = 0.0, d1 = 0.0;
  for (int b = b0 + (fc >> 1); b - (fc >> 1) < b1; b += 2, ra += sa, rb += sb) {
    const bool ok = b < b1;
    const double av = (ok && iok) ? __ldg(ra) : 0.0, bv = (ok && jok) ? __ldg(rb) : 0.0;
    dmma884(d0, d1, second ? -av : av, bv);
  }
  const int oc = 8 * tj + 2 * fc;   // this lane's accumulators: row i, columns oc, oc + 1
  double *out = part + (size_t)blockIdx.y * ((size_t)m * n) + (size_t)i * n;
  if (iok && oc < n) out[oc] = d0;
  if (iok && oc + 1 < n) out[oc + 1] = d1;
}

// dense P: G = sum_b w_b x_b^T (full n x n) into part[chunk][i n + j]; k-step s covers instances b0 + 4 s + fc.
__global__ void __launch_bounds__(32 * SR_TILE_WARPS) shared_grad_P_dense(int n, int m, const double *__restrict__ rec,
                                                                         const double *__restrict__ x, int B, int chunk,
                                                                         double *__restrict__ part) {
  const int lane = threadIdx.x & 31, tiles = (n + 7) >> 3, tile = blockIdx.x * SR_TILE_WARPS + (threadIdx.x >> 5);
  if (tile >= tiles * tiles) return;
  const int ti = tile / tiles, tj = tile - ti * tiles, fr = lane >> 2, fc = lane & 3;
  const long long R = bc_srec_doubles(n, m);
  const int i = 8 * ti + fr, j = 8 * tj + fr;
  const bool iok = i < n, jok = j < n;
  const int b0 = blockIdx.y * chunk, b1 = min(B, b0 + chunk);
  const double *rr = rec + (long long)(b0 + fc) * R, *xb = x + (size_t)(b0 + fc) * n;
  double d0 = 0.0, d1 = 0.0;
  for (int b = b0 + fc; b - fc < b1; b += 4, rr += 4 * R, xb += 4 * (size_t)n) {
    const bool ok = b < b1;
    double av = 0.0, bv = 0.0;
    if (ok && iok) { const double rt = __ldg(rr + n + m); av = rt * __ldg(xb + i) - __ldg(rr + i); }   // w_b[i]
    if (ok && jok) bv = __ldg(xb + j);
    dmma884(d0, d1, av, bv);
  }
  const int oc = 8 * tj + 2 * fc;
  double *out = part + (size_t)blockIdx.y * ((size_t)n * n) + (size_t)i * n;
  if (iok && oc < n) out[oc] = d0;
  if (iok && oc + 1 < n) out[oc + 1] = d1;
}

// CSR A: one thread per structural entry
__global__ void __launch_bounds__(SR_THREADS) shared_grad_A_csr(const DevStruct S, const double *__restrict__ rec, const double *__restrict__ x,
                                                                int B, int chunk, double *__restrict__ part) {
  const int n = S.n, m = S.m, k = blockIdx.x * SR_THREADS + threadIdx.x;
  if (k >= S.nnzA) return;
  const long long R = bc_srec_doubles(n, m);
  const int b0 = blockIdx.y * chunk, b1 = min(B, b0 + chunk);
  const int i = __ldg(S.A_rowof + k), j = __ldg(S.A_indices + k);
  const double *rb = rec + b0 * R, *xb = x + (size_t)b0 * n;
  double acc = 0.0;
#pragma unroll 4
  for (int b = b0; b < b1; b++, rb += R, xb += n)
    acc += __ldg(xb + j) * __ldg(rb + n + i) - __ldg(rb + n + m + 1 + i) * __ldg(rb + j);
  part[(size_t)blockIdx.y * S.nnzA + k] = acc;
}

// CSR P: one thread per structural entry of the upper triangle
__global__ void __launch_bounds__(SR_THREADS) shared_grad_P_csr(const DevStruct S, const double *__restrict__ rec, const double *__restrict__ x,
                                                                int B, int chunk, double *__restrict__ part) {
  const int n = S.n, m = S.m, k = blockIdx.x * SR_THREADS + threadIdx.x;
  if (k >= S.nnzP) return;
  const long long R = bc_srec_doubles(n, m);
  const int b0 = blockIdx.y * chunk, b1 = min(B, b0 + chunk);
  const int i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);
  const double *rb = rec + b0 * R, *xb = x + (size_t)b0 * n;
  double acc = 0.0;
#pragma unroll 4
  for (int b = b0; b < b1; b++, rb += R, xb += n) {
    const double rt = __ldg(rb + n + m), xi = __ldg(xb + i), xj = __ldg(xb + j);
    const double gij = (rt * xi - __ldg(rb + i)) * xj, gji = (rt * xj - __ldg(rb + j)) * xi;
    acc += (i == j) ? gij : gij + gji;
  }
  part[(size_t)blockIdx.y * S.nnzP + k] = acc;
}

// stage 2, A: dA[k] = sum over chunks in order (dense: the partial row is the m x n tile output, k = i n + j is its index too)
__global__ void __launch_bounds__(SR_THREADS) shared_grad_A_sum(const double *__restrict__ part, int K, int nchunks, double *__restrict__ dA) {
  const int k = blockIdx.x * SR_THREADS + threadIdx.x;
  if (k >= K) return;
  double acc = 0.0;
  for (int c = 0; c < nchunks; c++) acc += part[(size_t)c * K + k];
  dA[k] = acc;
}

// stage 2, P: CSR partials are per slot; dense partials are G (n x n), folded onto the upper triangle here
__global__ void __launch_bounds__(SR_THREADS) shared_grad_P_sum(const DevStruct S, const double *__restrict__ part, int nchunks, int dense,
                                                                double *__restrict__ dP) {
  const int k = blockIdx.x * SR_THREADS + threadIdx.x;
  if (k >= S.nnzP) return;
  double acc = 0.0;
  if (dense) {
    const int n = S.n, i = __ldg(S.P_rowof + k), j = __ldg(S.P_indices + k);
    const size_t nn = (size_t)n * n;
    for (int c = 0; c < nchunks; c++) {
      const double *G = part + (size_t)c * nn;
      acc += (i == j) ? G[(size_t)i * n + i] : G[(size_t)i * n + j] + G[(size_t)j * n + i];
    }
  } else {
    for (int c = 0; c < nchunks; c++) acc += part[(size_t)c * S.nnzP + k];
  }
  dP[k] = acc;
}
}  // namespace

extern "C" int bc_shared_chunks(int B) {
  int c = (B + SR_MIN_CHUNK - 1) / SR_MIN_CHUNK;
  return c < 1 ? 1 : (c > SR_MAX_CHUNKS ? SR_MAX_CHUNKS : c);
}

// doubles of partial sums one call needs: chunks x (nnzA + the P partial row: n^2 for a dense P, nnzP otherwise)
extern "C" size_t bc_shared_part_doubles(const DevStruct *S, int B) {
  const size_t kp = S->nnzP > 0 ? (S->p_dense ? (size_t)S->n * S->n : (size_t)S->nnzP) : 0;
  return (size_t)bc_shared_chunks(B) * ((size_t)S->nnzA + kp);
}

// part: bc_shared_part_doubles(S, B) doubles.  dP = NULL: A only.
extern "C" cudaError_t bc_shared_grad(const DevStruct *S, const double *rec, const double *x, int B, double *dA, double *dP, double *part,
                                      cudaStream_t st) {
  if (B <= 0) return cudaSuccess;
  const int n = S->n, m = S->m, nch = bc_shared_chunks(B), chunk = (B + nch - 1) / nch;
  double *partP = part + (size_t)nch * S->nnzA;
  if (S->nnzA > 0) {
    if (S->dense) {
      const int tiles = ((m + 7) >> 3) * ((n + 7) >> 3);
      shared_grad_A_dense<<<dim3((tiles + SR_TILE_WARPS - 1) / SR_TILE_WARPS, nch), 32 * SR_TILE_WARPS, 0, st>>>(n, m, rec, x, B, chunk, part);
    } else {
      shared_grad_A_csr<<<dim3((S->nnzA + SR_THREADS - 1) / SR_THREADS, nch), SR_THREADS, 0, st>>>(*S, rec, x, B, chunk, part);
    }
    shared_grad_A_sum<<<(S->nnzA + SR_THREADS - 1) / SR_THREADS, SR_THREADS, 0, st>>>(part, S->nnzA, nch, dA);
  }
  if (dP && S->nnzP > 0) {
    if (S->p_dense) {
      const int t = (n + 7) >> 3;
      shared_grad_P_dense<<<dim3((t * t + SR_TILE_WARPS - 1) / SR_TILE_WARPS, nch), 32 * SR_TILE_WARPS, 0, st>>>(n, m, rec, x, B, chunk, partP);
    } else {
      shared_grad_P_csr<<<dim3((S->nnzP + SR_THREADS - 1) / SR_THREADS, nch), SR_THREADS, 0, st>>>(*S, rec, x, B, chunk, partP);
    }
    shared_grad_P_sum<<<(S->nnzP + SR_THREADS - 1) / SR_THREADS, SR_THREADS, 0, st>>>(*S, partP, nch, S->p_dense, dP);
  }
  return cudaGetLastError();
}
