// fp32 SIMT "NT" GEMM used by the matcher blocks: C[M,N] = [A1 | A2][M,K1+K2] * B[N,K]^T (+bias) (*scale) (+resid).
// Exact-fp32 path (the parity reference on the device); the wgmma split-precision GEMM replaces it on the hot layers.
#pragma once
#include "common.cuh"

struct GemmArgs {
  const float* A1;
  int lda1;
  int K1;
  const float* A2;  // optional second K segment (torch.cat([x, msg], -1) without materialising the concat)
  int lda2;
  int K2;
  const float* B;  // [N][K1+K2], K contiguous (nn.Linear weight layout)
  int ldb;
  float* C;
  int ldc;
  int M;
  int N;
  const float* bias;   // [N] or null
  const float* resid;  // [M][ldr] or null, added after bias/scale
  int ldr;
  float scale;  // applied to (acc + bias)
  int head_major;  // 1: write C as [N/64][M][64] (attention head layout) instead of row-major
  int relu;        // max(., 0) after bias / scale, before the residual
};

constexpr int GB_M = 64, GB_N = 64, GB_K = 16;

static __global__ void __launch_bounds__(256) k_gemm_nt(GemmArgs g) {
  __shared__ __align__(16) float As[GB_K][GB_M + 4];
  __shared__ __align__(16) float Bs[GB_K][GB_N + 4];
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const int m0 = blockIdx.y * GB_M, n0 = blockIdx.x * GB_N;
  const int lr = t >> 2, lq = t & 3;  // loader: row lr, k quad lq
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int K = g.K1 + g.K2;
  for (int k0 = 0; k0 < K; k0 += GB_K) {
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f), bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + lr < g.M) {
      const float* src = (k0 < g.K1) ? g.A1 + (size_t)(m0 + lr) * g.lda1 + k0 : g.A2 + (size_t)(m0 + lr) * g.lda2 + (k0 - g.K1);
      av = *reinterpret_cast<const float4*>(src + lq * 4);
    }
    if (n0 + lr < g.N) bv = *reinterpret_cast<const float4*>(g.B + (size_t)(n0 + lr) * g.ldb + k0 + lq * 4);
    As[lq * 4 + 0][lr] = av.x;
    As[lq * 4 + 1][lr] = av.y;
    As[lq * 4 + 2][lr] = av.z;
    As[lq * 4 + 3][lr] = av.w;
    Bs[lq * 4 + 0][lr] = bv.x;
    Bs[lq * 4 + 1][lr] = bv.y;
    Bs[lq * 4 + 2][lr] = bv.z;
    Bs[lq * 4 + 3][lr] = bv.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GB_K; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float aa[4] = {a.x, a.y, a.z, a.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      float v = acc[i][j];
      if (g.bias) v += g.bias[n];
      v *= g.scale;
      if (g.relu) v = fmaxf(v, 0.f);
      if (g.resid) v += g.resid[(size_t)m * g.ldr + n];
      if (g.head_major)
        g.C[((size_t)(n >> 6) * g.M + m) * 64 + (n & 63)] = v;
      else
        g.C[(size_t)m * g.ldc + n] = v;
    }
  }
}

static inline int launch_gemm(b2_context* ctx, cudaStream_t st, const GemmArgs& g) {
  if (g.M <= 0 || g.N <= 0) return B2_OK;
  dim3 grid(cdiv(g.N, GB_N), cdiv(g.M, GB_M));
  b2_prof_work(ctx, "k_gemm_nt", 2.0 * g.M * g.N * (g.K1 + g.K2));
  B2_LAUNCH(ctx, k_gemm_nt, grid, 256, 0, st, g);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

static inline GemmArgs gemm_linear(const float* x, int ldx, int K, const float* w, const float* b, float* y, int ldy, int M, int N) {
  GemmArgs g{};
  g.A1 = x, g.lda1 = ldx, g.K1 = K, g.A2 = nullptr, g.lda2 = 0, g.K2 = 0;
  g.B = w, g.ldb = K, g.C = y, g.ldc = ldy, g.M = M, g.N = N;
  g.bias = b, g.resid = nullptr, g.ldr = 0, g.scale = 1.f, g.head_major = 0, g.relu = 0;
  return g;
}

// flash-style fp32 attention: O[Nq][256] (column h*64 + d) = softmax(scale * Q K^T) V per head.
// Q: [H][Nq][64], K, V: [H][Nk][64].  grid = (ceil(Nq/64), H), block = 256, dynamic smem = 64 KB.
constexpr int FA_T = 64;
constexpr size_t FA_SMEM = 4 * FA_T * 64 * sizeof(float);

static __global__ void __launch_bounds__(256) k_flash_attn(const float* __restrict__ Q, const float* __restrict__ Kp,
                                                     const float* __restrict__ V, float* __restrict__ O, int Nq, int Nk,
                                                     float scale) {
  extern __shared__ __align__(16) float fsm[];
  float* Qt = fsm;                  // [64 d][64 rows]
  float* Kt = Qt + 64 * FA_T;       // [64 d][64 keys]
  float* Vs = Kt + 64 * FA_T;       // [64 keys][64 d]
  float* Ps = Vs + 64 * FA_T;       // [64 rows][64 keys]
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int h = blockIdx.y, q0 = blockIdx.x * FA_T;
  const float* Qh = Q + (size_t)h * Nq * 64;
  const float* Kh = Kp + (size_t)h * Nk * 64;
  const float* Vh = V + (size_t)h * Nk * 64;
  for (int i = t; i < FA_T * 16; i += 256) {
    int r = i >> 4, dq = i & 15;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < Nq) v = *reinterpret_cast<const float4*>(Qh + (size_t)(q0 + r) * 64 + dq * 4);
    Qt[(dq * 4 + 0) * FA_T + r] = v.x;
    Qt[(dq * 4 + 1) * FA_T + r] = v.y;
    Qt[(dq * 4 + 2) * FA_T + r] = v.z;
    Qt[(dq * 4 + 3) * FA_T + r] = v.w;
  }
  float m_i[4], l_i[4], o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_i[i] = -INFINITY;
    l_i[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  }
  for (int k0 = 0; k0 < Nk; k0 += FA_T) {
    __syncthreads();  // previous tile fully consumed (also covers the Q load on the first pass)
    for (int i = t; i < FA_T * 16; i += 256) {
      int r = i >> 4, dq = i & 15;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + r < Nk) {
        kv = *reinterpret_cast<const float4*>(Kh + (size_t)(k0 + r) * 64 + dq * 4);
        vv = *reinterpret_cast<const float4*>(Vh + (size_t)(k0 + r) * 64 + dq * 4);
      }
      Kt[(dq * 4 + 0) * FA_T + r] = kv.x;
      Kt[(dq * 4 + 1) * FA_T + r] = kv.y;
      Kt[(dq * 4 + 2) * FA_T + r] = kv.z;
      Kt[(dq * 4 + 3) * FA_T + r] = kv.w;
      *reinterpret_cast<float4*>(&Vs[r * 64 + dq * 4]) = vv;
    }
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int d = 0; d < 64; ++d) {
      float4 a = *reinterpret_cast<const float4*>(&Qt[d * FA_T + ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Kt[d * FA_T + tx * 4]);
      const float aa[4] = {a.x, a.y, a.z, a.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(aa[i], bb[j], s[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = (k0 + tx * 4 + j < Nk) ? s[i][j] * scale : -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      float m_new = fmaxf(m_i[i], mx);
      float corr = expf(m_i[i] - m_new);  // exp(-inf) = 0 on the first tile
      float rs = 0.f;
      float p[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        p[j] = expf(s[i][j] - m_new);
        rs += p[j];
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
      l_i[i] = l_i[i] * corr + rs;
      m_i[i] = m_new;
#pragma unroll
      for (int j = 0; j < 4; ++j) o[i][j] *= corr;
      *reinterpret_cast<float4*>(&Ps[(ty * 4 + i) * FA_T + tx * 4]) = make_float4(p[0], p[1], p[2], p[3]);
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < FA_T; ++kk) {
      float4 vv = *reinterpret_cast<const float4*>(&Vs[kk * 64 + tx * 4]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float p = Ps[(ty * 4 + i) * FA_T + kk];
        o[i][0] = fmaf(p, vv.x, o[i][0]);
        o[i][1] = fmaf(p, vv.y, o[i][1]);
        o[i][2] = fmaf(p, vv.z, o[i][2]);
        o[i][3] = fmaf(p, vv.w, o[i][3]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int r = q0 + ty * 4 + i;
    if (r < Nq) {
      float inv = 1.0f / l_i[i];
      *reinterpret_cast<float4*>(O + (size_t)r * 256 + h * 64 + tx * 4) =
          make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
    }
  }
}

static inline int launch_flash(b2_context* ctx, cudaStream_t st, const float* Q, const float* K, const float* V, float* O,
                               int Nq, int Nk, float scale) {
  if (Nq <= 0) return B2_OK;
  dim3 grid(cdiv(Nq, FA_T), 4);
  b2_prof_work(ctx, "k_flash_attn", 4.0 * 2.0 * 2.0 * (double)Nq * Nk * 64);  // 4 heads x (QK^T + PV) x 2 FLOP/MAC
  B2_LAUNCH(ctx, k_flash_attn, grid, 256, FA_SMEM, st, Q, K, V, O, Nq, Nk, scale);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}
