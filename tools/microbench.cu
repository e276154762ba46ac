// Micro-benchmarks of the shared-memory matvec building blocks (cycles per call, one CTA per SM).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench tools/microbench.cu
#include <cstdio>
#include <vector>
#define BC_CHOLPROF 1
#include "../cvxpylayers_b200/csrc/common.cuh"

constexpr int NT = 32;
__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

struct Args { double *A; double *out; unsigned long long *cyc; int m, n, reps; };

template <class F>
__device__ __forceinline__ void timed(unsigned long long *cyc, int slot, int reps, F f) {
  __syncthreads();
  const long long t0 = clock64();
  for (int r = 0; r < reps; r++) f(r);
  __syncthreads();
  const long long t1 = clock64();
  if (threadIdx.x == 0) atomicAdd(cyc + slot, (unsigned long long)(t1 - t0));
}

__global__ void __launch_bounds__(512, 1) mb_kernel(Args a) {
  extern __shared__ __align__(16) double smem[];
  const int m = a.m, n = a.n, T = blockDim.x, t = threadIdx.x, reps = a.reps;
  double *Av = smem;                       // m*n
  double *Li = Av + m * n;                 // n(n+1)/2 (+pad)
  double *x = Li + ((n * (n + 1) / 2 + 1) & ~1);   // n
  double *y = x + n;                       // m
  double *o1 = y + m;                      // m
  double *o2 = o1 + m;                     // n
  double *part = o2 + n;                   // 20*n  (>= 8n, >= 10 m)
  double *red = part + 20 * n;             // 256
  for (int k = t; k < m * n; k += T) Av[k] = a.A[k];
  for (int k = t; k < n * (n + 1) / 2; k += T) Li[k] = 1e-3 * (k % 17);
  for (int k = t; k < n; k += T) { x[k] = 1.0 + 1e-3 * k; o2[k] = 0; }
  for (int k = t; k < m; k += T) { y[k] = 1.0 - 1e-3 * k; o1[k] = 0; }
  __syncthreads();
  const ColPlan plN = make_colplan(n, n);

  // 0: barrier only
  timed(a.cyc, 0, reps, [&](int) { __syncthreads(); });
  // 1: DFMA throughput: 8 chains x 32 per rep
  {
    double c[8]; for (int k = 0; k < 8; k++) c[k] = x[(t + k) % n];
    const double mul = y[t % m];
    timed(a.cyc, 1, reps, [&](int) {
#pragma unroll
      for (int q = 0; q < 32; q++)
#pragma unroll
        for (int k = 0; k < 8; k++) c[k] = fma(c[k], mul, 1e-9);
    });
    double s = 0; for (int k = 0; k < 8; k++) s += c[k];
    if (s == 1.2345) a.out[t] = s;
  }
  // 2: LDS.128 throughput, conflict-free, 64 loads per rep
  {
    double2 acc = make_double2(0, 0);
    const double2 *p = reinterpret_cast<const double2 *>(Av) + t;
    timed(a.cyc, 2, reps, [&](int r) {
#pragma unroll
      for (int q = 0; q < 16; q++) { const double2 v = p[(q * 512 + r) & 8191]; acc.x += v.x; acc.y += v.y; }
    });
    if (acc.x == 1.2345) a.out[t] = acc.y;
  }
  // 3: dense_rows2 + barrier
  timed(a.cyc, 3, reps, [&](int) { dense_rows2(Av, m, n, x, [&](int i, double v) { o1[i] = v; }); __syncthreads(); });
  // 4: dense_cols2 (ends with a barrier)
  timed(a.cyc, 4, reps, [&](int) { dense_cols2(Av, m, n, y, part, [&](int j, double v) { o2[j] = v; }); });
  // 5: packed rows + barrier
  timed(a.cyc, 5, reps, [&](int) { matvec_rows(Li, PackedLowerLayout{}, n, n, x, [&](int i, double v) { o2[i] = v; }); __syncthreads(); });
  // 6: packed cols
  timed(a.cyc, 6, reps, [&](int) { matvec_cols(Li, PackedLowerLayout{}, n, n, x, part, [&](int j, double v) { o2[j] = v; }, plN); });
  // 7: block_reduce<4>
  {
    double d4[4] = {x[t % n], 1, 2, 3};
    timed(a.cyc, 7, reps, [&](int) { block_reduce<4, false>(d4, red); });
    if (d4[0] == 1.2345) a.out[t] = d4[1];
  }
  // 8/9: register-resident 4 x 10 tiles of A (m = 200, n = 100, 500 threads)
  if (m == 200 && n == 100) {
    const int R = t / 10, C = t % 10;
    double *part50 = Li;   // 50 n doubles: the packed factor is not needed any more
    const bool act = t < 500;
    double ar[4][10];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
      for (int c = 0; c < 10; c++) ar[r][c] = act ? Av[(4 * R + r) * n + 10 * C + c] : 0.0;
    // rows: out_i = sum_j A_ij x_j
    timed(a.cyc, 8, reps, [&](int) {
      if (act) {
        double xv[10];
#pragma unroll
        for (int c = 0; c < 10; c += 2) { const double2 v = *reinterpret_cast<const double2 *>(x + 10 * C + c); xv[c] = v.x; xv[c + 1] = v.y; }
#pragma unroll
        for (int r = 0; r < 4; r++) {
          double s0 = 0, s1 = 0;
#pragma unroll
          for (int c = 0; c < 10; c += 2) { s0 = fma(ar[r][c], xv[c], s0); s1 = fma(ar[r][c + 1], xv[c + 1], s1); }
          part[(4 * R + r) * 10 + C] = s0 + s1;
        }
      }
      __syncthreads();
      if (t < m) {
        const double2 *p = reinterpret_cast<const double2 *>(part + t * 10);
        const double2 v0 = p[0], v1 = p[1], v2 = p[2], v3 = p[3], v4 = p[4];
        o1[t] = ((v0.x + v0.y) + (v1.x + v1.y)) + ((v2.x + v2.y) + (v3.x + v3.y)) + (v4.x + v4.y);
      }
      __syncthreads();
    });
    // cols: out_j = sum_i A_ij y_i
    timed(a.cyc, 9, reps, [&](int) {
      if (act) {
        const double2 y01 = *reinterpret_cast<const double2 *>(y + 4 * R), y23 = *reinterpret_cast<const double2 *>(y + 4 * R + 2);
        double q[10];
#pragma unroll
        for (int c = 0; c < 10; c++) q[c] = fma(ar[3][c], y23.y, fma(ar[2][c], y23.x, fma(ar[1][c], y01.y, ar[0][c] * y01.x)));
#pragma unroll
        for (int c = 0; c < 10; c += 2) *reinterpret_cast<double2 *>(part50 + R * n + 10 * C + c) = make_double2(q[c], q[c + 1]);
      }
      __syncthreads();
      if (t < n) {
        double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
#pragma unroll
        for (int Rr = 0; Rr < 50; Rr += 5) {
          s0 += part50[Rr * n + t]; s1 += part50[(Rr + 1) * n + t]; s2 += part50[(Rr + 2) * n + t]; s3 += part50[(Rr + 3) * n + t]; s4 += part50[(Rr + 4) * n + t];
        }
        o2[t] = ((s0 + s1) + (s2 + s3)) + s4;
      }
      __syncthreads();
    });
    // 10: cols with a 4-way split reduce (400 threads, quad shuffle)
    timed(a.cyc, 10, reps, [&](int) {
      if (act) {
        const double2 y01 = *reinterpret_cast<const double2 *>(y + 4 * R), y23 = *reinterpret_cast<const double2 *>(y + 4 * R + 2);
        double q[10];
#pragma unroll
        for (int c = 0; c < 10; c++) q[c] = fma(ar[3][c], y23.y, fma(ar[2][c], y23.x, fma(ar[1][c], y01.y, ar[0][c] * y01.x)));
#pragma unroll
        for (int c = 0; c < 10; c += 2) *reinterpret_cast<double2 *>(part50 + R * n + 10 * C + c) = make_double2(q[c], q[c + 1]);
      }
      __syncthreads();
      {
        const int j = t >> 2, g = t & 3;
        double s0 = 0, s1 = 0;
        if (j < n) {
#pragma unroll
          for (int Rr = 0; Rr < 48; Rr += 8) { s0 += part50[(Rr + g) * n + j]; s1 += part50[(Rr + 4 + g) * n + j]; }
          if (g < 2) s0 += part50[(48 + g) * n + j];
        }
        s0 += s1;
        s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
        s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
        if (g == 0 && j < n) o2[j] = s0;
      }
      __syncthreads();
    });
    double s = 0;
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
      for (int c = 0; c < 10; c++) s += ar[r][c];
    if (s == 1.2345) a.out[t] = s;
  }
  // 11: Ruiz-style A sweep (row max via warp reduce, column max per lane), as in fwd.cu
  {
    const int lane = t & 31, warp = t >> 5, nw = T >> 5;
    timed(a.cyc, 11, reps, [&](int) {
      double er[4], cacc[4] = {0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; er[k] = c < n ? x[c] : 0.0; }
      for (int i = warp; i < m; i += nw) {
        const double d = y[i];
        const double *row = Av + i * n;
        double r = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const int c = lane + 32 * k;
          if (c < n) { const double v = fabs(row[c]) * er[k]; r = fmax(r, v); cacc[k] = fmax(cacc[k], v * d); }
        }
        r = warp_max(r) * d;
        if (lane == 0) o1[i] = r;
      }
      const int slot = warp & 7;
      if (warp < 8) {
#pragma unroll
        for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; if (c < n) part[slot * n + c] = cacc[k]; }
      }
      __syncthreads();
      if (warp >= 8) {
#pragma unroll
        for (int k = 0; k < 4; k++) { const int c = lane + 32 * k; if (c < n) part[slot * n + c] = fmax(part[slot * n + c], cacc[k]); }
      }
      __syncthreads();
      if (t < n) { double r = 0; for (int q = 0; q < 8; q++) r = fmax(r, part[q * n + t]); o2[t] = r; }
      __syncthreads();
    });
  }
  // 12: DMMA m8n8k4 throughput: 8 independent accumulator pairs x 16 per rep
  {
    double acc[8][2];
    for (int k = 0; k < 8; k++) { acc[k][0] = x[(t + k) % n]; acc[k][1] = 0; }
    const double fa = y[t % m], fb = x[t % n];
    timed(a.cyc, 12, reps, [&](int) {
#pragma unroll
      for (int q = 0; q < 16; q++)
#pragma unroll
        for (int k = 0; k < 8; k++) dmma(acc[k][0], acc[k][1], fa, fb);
    });
    double s = 0; for (int k = 0; k < 8; k++) s += acc[k][0] + acc[k][1];
    if (s == 1.2345) a.out[t] = s;
  }
  // 13: K = A' W A (lower, 8x8 tiles, 13 x 13 blocks) with DMMA: warp per 16 x 32 macro tile strip
  {
    const int lane = t & 31, warp = t >> 5, nw = T >> 5;
    const int nb = (n + 7) >> 3;                 // 13
    double *Kout = Li;                           // packed lower n(n+1)/2
    timed(a.cyc, 13, 20, [&](int) {
      // macro tiles: block-row pair JP (rows 16 JP .. 16 JP + 15), block-col quad KQ (cols 32 KQ ..): only those touching the lower triangle
      const int nJP = (nb + 1) >> 1, nKQ = (nb + 3) >> 2;
      int cnt = 0;
      for (int JP = 0; JP < nJP; JP++)
        for (int KQ = 0; KQ < nKQ; KQ++) {
          if (4 * KQ > 2 * JP + 1) continue;     // entirely above the diagonal
          if ((cnt++ % nw) != warp) continue;
          double acc[2][4][2];
#pragma unroll
          for (int u = 0; u < 2; u++)
#pragma unroll
            for (int v = 0; v < 4; v++) acc[u][v][0] = acc[u][v][1] = 0.0;
          const int jr = 16 * JP + (lane >> 2), kc = 32 * KQ + (lane >> 2);
          for (int i = 0; i < m; i += 4) {
            const double *row = Av + (i + (lane & 3)) * n;
            const double w = (i + (lane & 3)) < 50 ? 1000.0 : 1.0;
            double fa[2], fb[4];
#pragma unroll
            for (int u = 0; u < 2; u++) { const int j = jr + 8 * u; fa[u] = j < n ? row[j] * w : 0.0; }
#pragma unroll
            for (int v = 0; v < 4; v++) { const int k = kc + 8 * v; fb[v] = k < n ? row[k] : 0.0; }
#pragma unroll
            for (int u = 0; u < 2; u++)
#pragma unroll
              for (int v = 0; v < 4; v++) dmma(acc[u][v][0], acc[u][v][1], fa[u], fb[v]);
          }
#pragma unroll
          for (int u = 0; u < 2; u++)
#pragma unroll
            for (int v = 0; v < 4; v++) {
              const int j = 16 * JP + 8 * u + (lane >> 2), k = 32 * KQ + 8 * v + 2 * (lane & 3);
              if (j < n && k <= j) Kout[((j * (j + 1)) >> 1) + k] = acc[u][v][0];
              if (j < n && k + 1 <= j) Kout[((j * (j + 1)) >> 1) + k + 1] = acc[u][v][1];
            }
        }
      __syncthreads();
    });
    if (t == 0) a.out[2000] = Kout[(57 * 58 >> 1) + 13];
    __syncthreads();
  }
  // 14: the same K by 2 x 2 register tiles (the current form_K)
  {
    double *Kout = Li;
    timed(a.cyc, 14, 20, [&](int) {
      const int nb2 = n >> 1, ntile = (nb2 * (nb2 + 1)) >> 1;
      for (int e = t; e < ntile; e += T) {
        int J = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
        while (((J + 1) * (J + 2)) >> 1 <= e) J++;
        while ((J * (J + 1)) >> 1 > e) J--;
        const int Kb = e - ((J * (J + 1)) >> 1);
        const double2 *pj = reinterpret_cast<const double2 *>(Av) + J, *pk = reinterpret_cast<const double2 *>(Av) + Kb;
        double z00 = 0, z01 = 0, z10 = 0, z11 = 0, s00 = 0, s01 = 0, s10 = 0, s11 = 0;
        int i = 0;
        for (; i < 50; i++) { const double2 u = pj[i * nb2], v = pk[i * nb2]; z00 = fma(u.x, v.x, z00); z01 = fma(u.x, v.y, z01); z10 = fma(u.y, v.x, z10); z11 = fma(u.y, v.y, z11); }
        for (; i < m; i++) { const double2 u = pj[i * nb2], v = pk[i * nb2]; s00 = fma(u.x, v.x, s00); s01 = fma(u.x, v.y, s01); s10 = fma(u.y, v.x, s10); s11 = fma(u.y, v.y, s11); }
        const int j0 = 2 * J, k0 = 2 * Kb;
        Kout[((j0 * (j0 + 1)) >> 1) + k0] = z00 * 1000.0 + s00;
        if (k0 + 1 <= j0) Kout[((j0 * (j0 + 1)) >> 1) + k0 + 1] = z01 * 1000.0 + s01;
        Kout[(((j0 + 1) * (j0 + 2)) >> 1) + k0] = z10 * 1000.0 + s10;
        Kout[(((j0 + 1) * (j0 + 2)) >> 1) + k0 + 1] = z11 * 1000.0 + s11;
      }
      __syncthreads();
    });
    if (t == 0) a.out[2001] = Kout[(57 * 58 >> 1) + 13];
  }
  // 25: DMMA latency: one dependent chain of 64 per rep (all warps), 26: the same on warp 0 only; 27: DFMA dependent chain of 64
  {
    double c0 = x[t % n], c1 = 0;
    const double fa = 1e-3 * y[t % m], fb = x[t % n];
    timed(a.cyc, 25, reps, [&](int) {
#pragma unroll
      for (int q = 0; q < 64; q++) dmma(c0, c1, fa, fb);
    });
    timed(a.cyc, 26, reps, [&](int) {
      if (t < 32) {
#pragma unroll
        for (int q = 0; q < 64; q++) dmma(c0, c1, fa, fb);
      }
    });
    double f0 = c0;
    timed(a.cyc, 27, reps, [&](int) {
      if (t < 32) {
#pragma unroll
        for (int q = 0; q < 64; q++) f0 = fma(f0, fa, fb);
      }
    });
    if (c0 + c1 + f0 == 1.2345) a.out[t] = c0;
  }
  // 15 (+ sub-phases 17..20): packed Cholesky + inverse of an n x n SPD matrix
  {
    for (int e = t; e < n * (n + 1) / 2; e += T) {
      int j = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
      while ((j + 1) * (j + 2) / 2 <= e) j++;
      while (j * (j + 1) / 2 > e) j--;
      const int k = e - j * (j + 1) / 2;
      Li[e] = (j == k) ? 3.0 + 0.01 * j : 0.5 * sin(0.37 * j + 0.11 * k) / (1.0 + abs(j - k));
    }
    __syncthreads();
    const long long t0 = clock64();
    const bool ok = chol_inv_packed(Li, n, part, a.cyc);
    __syncthreads();
    if (t == 0) { atomicAdd(a.cyc + 15, (unsigned long long)(clock64() - t0)); a.out[2002] = ok ? Li[(57 * 58 >> 1) + 13] : -1.0; }
  }
  if (t < n) a.out[512 + t] = o2[t];
  if (t < m) a.out[1024 + t] = o1[t];
}

int main(int argc, char **argv) {
  const int m = 200, n = argc > 1 ? atoi(argv[1]) : 100, reps = 200;   // n: size of every product and of the Cholesky ledger
  if (n < 2 || n > 128 || (n & 1)) { printf("n must be even, 2..128\n"); return 1; }
  std::vector<double> hA(m * n);
  for (int k = 0; k < m * n; k++) hA[k] = 0.001 * ((k * 7919) % 1000) - 0.5;
  Args a; a.m = m; a.n = n; a.reps = reps;
  cudaMalloc(&a.A, sizeof(double) * m * n); cudaMalloc(&a.out, sizeof(double) * 4096); cudaMalloc(&a.cyc, sizeof(unsigned long long) * NT);
  cudaMemcpy(a.A, hA.data(), sizeof(double) * m * n, cudaMemcpyHostToDevice);
  cudaMemset(a.cyc, 0, sizeof(unsigned long long) * NT);
  const size_t smem = sizeof(double) * (m * n + n * (n + 1) / 2 + 2 + n + m + m + n + 20 * n + 256);
  cudaFuncSetAttribute(mb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int grid = 0;   // one CTA per SM
  cudaDeviceGetAttribute(&grid, cudaDevAttrMultiProcessorCount, 0);
  mb_kernel<<<grid, 512, smem>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(e)); return 1; }
  unsigned long long h[NT]; cudaMemcpy(h, a.cyc, sizeof(h), cudaMemcpyDeviceToHost);
  std::vector<double> ho(4096); cudaMemcpy(ho.data(), a.out, sizeof(double) * 4096, cudaMemcpyDeviceToHost);
  const char *names[NT] = {"barrier", "DFMA x256/thread", "LDS.128 x16/thread", "dense_rows2 + barrier", "dense_cols2", "packed rows + barrier", "packed cols",
                           "block_reduce<4>", "regtile rows", "regtile cols (100x50)", "regtile cols (quad)", "ruiz A sweep", "DMMA x128/thread", "K formation DMMA (x20)", "K formation 2x2 (x20)", ""};
  printf("smem %zu B\n", smem);
  for (int k = 0; k < 15; k++) printf("%-26s %10.1f cycles/call\n", names[k], (double)h[k] / grid / (k >= 13 ? 20 : reps));
  // slots 17..20 of chol_inv_packed, summed over its 8-column steps (thread 0's clock)
  const char *cn[6] = {"chol+inv total", "", "  A: X store|panel|Z", "  barrier 1", "  B: trail+diag|inverse", "  barrier 2"};
  printf("n = %d\n", n);
  for (int k = 15; k < 21; k++)
    if (k != 16) printf("%-26s %10.1f cycles/call\n", cn[k - 15], (double)h[k] / grid);
  printf("DMMA chain x64 (16 warps) %.1f, (1 warp) %.1f, DFMA chain x64 (1 warp) %.1f cycles/call\n", (double)h[25] / grid / reps, (double)h[26] / grid / reps, (double)h[27] / grid / reps);
  printf("chol check Linv[57][13]=%.12g  factor %.1f inverse %.1f\n", ho[2002], (double)h[5] / grid, (double)h[6] / grid);
  printf("check o2[3]=%g o1[5]=%g  K[57][13] dmma=%.12g 2x2=%.12g\n", ho[512 + 3], ho[1024 + 5], ho[2000], ho[2001]);
  return 0;
}
