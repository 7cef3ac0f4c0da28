// Blocked fp64 Cholesky and triangular solves of a dense reduced system (dense_chol.cuh).  Shared by the global bundle
// adjustment and the translation recovery, so that the library holds one definition of each kernel.
#include "dense_chol.cuh"

namespace {
constexpr int NB = CHOL_NB;
}  // namespace

// ---- blocked Cholesky of S (row-major, lower triangle), tile k's three steps ------------------------------------------
__global__ void __launch_bounds__(256) k_chol_diag(double* S, int np, int k, int* flag) {
  __shared__ double T[NB][NB + 1];
  if (*flag) return;
  const int tid = threadIdx.x;
  double* A = S + (int64_t)k * NB * np + (int64_t)k * NB;
  for (int e = tid; e < NB * NB; e += 256) T[e / NB][e % NB] = A[(int64_t)(e / NB) * np + e % NB];
  __syncthreads();
  for (int c = 0; c < NB; ++c) {
    if (tid == 0) {
      const double p = T[c][c];
      if (!(p > 0.0) || !isfinite(p)) *flag = 1;
      T[c][c] = sqrt(p);
    }
    __syncthreads();
    for (int r = c + 1 + tid; r < NB; r += 256) T[r][c] /= T[c][c];
    __syncthreads();
    const int m = NB - 1 - c;
    for (int e = tid; e < m * m; e += 256) {
      const int r = c + 1 + e / m, q = c + 1 + e % m;
      if (q <= r) T[r][q] -= T[r][c] * T[q][c];
    }
    __syncthreads();
  }
  for (int e = tid; e < NB * NB; e += 256)
    if (e % NB <= e / NB) A[(int64_t)(e / NB) * np + e % NB] = T[e / NB][e % NB];
}

// tile row i = k + 1 + blockIdx.x: L_ik = A_ik L_kk^-T, one thread per row
__global__ void __launch_bounds__(NB) k_chol_panel(double* S, int np, int k, const int* flag) {
  extern __shared__ double sm[];
  double(*Lk)[NB + 1] = reinterpret_cast<double(*)[NB + 1]>(sm);
  double(*A)[NB + 1] = reinterpret_cast<double(*)[NB + 1]>(sm + NB * (NB + 1));
  if (*flag) return;
  const int tid = threadIdx.x, i = k + 1 + blockIdx.x;
  const double* Lg = S + (int64_t)k * NB * np + (int64_t)k * NB;
  double* Ag = S + (int64_t)i * NB * np + (int64_t)k * NB;
  for (int e = tid; e < NB * NB; e += NB) {
    Lk[e / NB][e % NB] = Lg[(int64_t)(e / NB) * np + e % NB];
    A[e / NB][e % NB] = Ag[(int64_t)(e / NB) * np + e % NB];
  }
  __syncthreads();
  for (int c = 0; c < NB; ++c) {
    double x = A[tid][c];
    for (int m = 0; m < c; ++m) x -= A[tid][m] * Lk[c][m];
    A[tid][c] = x / Lk[c][c];
  }
  __syncthreads();
  for (int e = tid; e < NB * NB; e += NB) Ag[(int64_t)(e / NB) * np + e % NB] = A[e / NB][e % NB];
}

// trailing update of tile (i, j), k < j <= i: A_ij -= L_ik L_jk^T; 256 threads, 4 x 4 outputs each
__global__ void __launch_bounds__(256) k_chol_update(double* S, int np, int k, const int* flag) {
  extern __shared__ double sm[];
  double(*Li)[NB + 1] = reinterpret_cast<double(*)[NB + 1]>(sm);
  double(*Lj)[NB + 1] = reinterpret_cast<double(*)[NB + 1]>(sm + NB * (NB + 1));
  if (*flag) return;
  const int64_t t = blockIdx.x;
  int a = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((int64_t)(a + 1) * (a + 2) / 2 <= t) ++a;
  while ((int64_t)a * (a + 1) / 2 > t) --a;
  const int i = k + 1 + a, j = k + 1 + (int)(t - (int64_t)a * (a + 1) / 2);
  const int tid = threadIdx.x;
  const double* gi = S + (int64_t)i * NB * np + (int64_t)k * NB;
  const double* gj = S + (int64_t)j * NB * np + (int64_t)k * NB;
  for (int e = tid; e < NB * NB; e += 256) {
    Li[e / NB][e % NB] = gi[(int64_t)(e / NB) * np + e % NB];
    Lj[e / NB][e % NB] = gj[(int64_t)(e / NB) * np + e % NB];
  }
  __syncthreads();
  const int tr = tid / 16, tc = tid % 16;
  double acc[4][4] = {};
#pragma unroll 4
  for (int kk = 0; kk < NB; ++kk) {
    double av[4], bv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) av[u] = Li[tr + 16 * u][kk], bv[u] = Lj[tc + 16 * u][kk];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[u][v] = fma(av[u], bv[v], acc[u][v]);
  }
  double* A = S + (int64_t)i * NB * np + (int64_t)j * NB;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) A[(int64_t)(tr + 16 * u) * np + tc + 16 * v] -= acc[u][v];
}

// L y = b, tile k: every CTA solves tile k's 64 unknowns from b_k (complete after steps 0..k-1); CTA 0 writes y_k, CTA
// q > 0 updates b_{k+q} -= L_{k+q,k} y_k
__global__ void __launch_bounds__(NB) k_trsv_fwd(const double* S, int np, int k, double* b, double* y, const int* flag) {
  __shared__ double v[NB];
  if (*flag) return;
  const int tid = threadIdx.x, i = k + blockIdx.x;
  const double* Lk = S + (int64_t)k * NB * np + (int64_t)k * NB;
  v[tid] = b[k * NB + tid];
  __syncthreads();
  for (int c = 0; c < NB; ++c) {
    if (tid == c) v[c] /= Lk[(int64_t)c * np + c];
    __syncthreads();
    if (tid > c) v[tid] -= Lk[(int64_t)tid * np + c] * v[c];
    __syncthreads();
  }
  if (i == k) {
    y[k * NB + tid] = v[tid];
    return;
  }
  const double* Li = S + (int64_t)(i * NB + tid) * np + (int64_t)k * NB;
  double acc = 0.0;
  for (int c = 0; c < NB; ++c) acc += Li[c] * v[c];
  b[i * NB + tid] -= acc;
}

// L^T x = y, tile k (descending): CTA 0 writes x_k, CTA q > 0 updates y_{k-q} -= L_{k,k-q}^T x_k
__global__ void __launch_bounds__(NB) k_trsv_bwd(const double* S, int np, int k, double* y, double* x, const int* flag) {
  __shared__ double v[NB];
  if (*flag) return;
  const int tid = threadIdx.x, i = k - blockIdx.x;
  const double* Lk = S + (int64_t)k * NB * np + (int64_t)k * NB;
  v[tid] = y[k * NB + tid];
  __syncthreads();
  for (int c = NB - 1; c >= 0; --c) {
    if (tid == c) v[c] /= Lk[(int64_t)c * np + c];
    __syncthreads();
    if (tid < c) v[tid] -= Lk[(int64_t)c * np + tid] * v[c];
    __syncthreads();
  }
  if (i == k) {
    x[k * NB + tid] = v[tid];
    return;
  }
  const double* Lki = S + (int64_t)k * NB * np + (int64_t)i * NB + tid;
  double acc = 0.0;
  for (int c = 0; c < NB; ++c) acc += Lki[(int64_t)c * np] * v[c];
  y[i * NB + tid] -= acc;
}

int dense_chol_solve(b2_context* ctx, double* S, int np, double* b, double* y, double* x, int* flag, cudaStream_t st) {
  const int nt = np / NB;
  const size_t upd_smem = 2 * NB * (NB + 1) * 8;
  B2_CUDA(ctx, cudaFuncSetAttribute(k_chol_update, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)upd_smem));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_chol_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)upd_smem));
  for (int k = 0; k < nt; ++k) {
    B2_LAUNCH(ctx, k_chol_diag, 1, 256, 0, st, S, np, k, flag);
    const int m = nt - 1 - k;
    if (m > 0) {
      B2_LAUNCH(ctx, k_chol_panel, (unsigned)m, NB, upd_smem, st, S, np, k, flag);
      B2_LAUNCH(ctx, k_chol_update, (unsigned)((int64_t)m * (m + 1) / 2), 256, upd_smem, st, S, np, k, flag);
    }
  }
  B2_CHECK_LAUNCH(ctx);
  for (int k = 0; k < nt; ++k) B2_LAUNCH(ctx, k_trsv_fwd, (unsigned)(nt - k), NB, 0, st, S, np, k, b, y, flag);
  for (int k = nt - 1; k >= 0; --k) B2_LAUNCH(ctx, k_trsv_bwd, (unsigned)(k + 1), NB, 0, st, S, np, k, y, x, flag);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}
