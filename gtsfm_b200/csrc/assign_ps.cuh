#pragma once
#include "common.cuh"

// Persistent assignment kernel, two instantiations of one schedule:
//   KIND 0  SuperGlue: log_optimal_transport (superglue.py:141-170) + the mutual arg-max passes (:266-270)
//   KIND 1  LightGlue: sigmoid_log_double_softmax (lightglue.py:265-277) row / column log-softmax statistics + the mutual
//           arg-max of filter_matches (:302-318) - ONE statistics sweep, then the arg-max sweep (no dustbins, no iterations)
// Everything in ONE cooperative launch.  CTA b owns a contiguous block of rows of the augmented (M + 1) x (N + 1) matrix (the dustbin row /
// column are analytic: alpha).  Per iteration every score is read ONCE:
//   * rows stream through a 3-deep cp.async ring in shared memory, two rows per step;
//   * u_i = log_mu_i - LSE_j(Z_ij + v_j): an online (max, sum) per thread over its columns (thread t owns columns t, t + 1024,
//     ...), merged by warp shuffles and one shared-memory hop;
//   * with u_i known, the SAME staged row updates the thread's per-column online (max, sum) of Z_ij + u_i, kept in registers
//     across all rows of the CTA; at the end of the row block the partials go to global memory, a grid barrier later the CTAs
//     merge them column-wise (one warp per column) into v_j = log_nu_j - LSE_i(.), second grid barrier, next iteration.
// After the last iteration the same structure yields the row arg-max (per row, block reduction) and the column arg-max
// (per-thread partials merged across CTAs) of Z + u + v - norm over the M x N core.
// Traffic: (M x N x 4 B + 2 x G x (N + 1) x 8 B) per iteration instead of 2-3 full passes in 2 launches; 20 iterations and the
// arg-max are 1 launch instead of 42.
// ------------------------------------------------------------------------------------------------------------------
constexpr int SK_T = 1024;   // threads per CTA
constexpr int SK_NC = 8;     // columns per thread: N + 1 <= 8192
constexpr int SK_R = 2;      // rows per pipeline step
constexpr int SK_NB = 3;     // ring depth

struct SinkArgs {
  const float* Z;
  int M, N;
  float alpha, norm;
  int iters;
  float *u, *v;       // KIND 0: [M + 1], [N + 1] dual variables.  KIND 1: row maxima [M] / column maxima [N]
  float *rlog, *clog; // KIND 1: log of the row / column sums of exp(x - max)
  const float *z0, *z1;   // KIND 1: matchability logits of the rows / columns ...
  float *lsg0, *lsg1;     // ... and where their logsigmoid is tabulated
  float* part;        // [G][2][N + 1] column partials: (max, sum) during the iterations, (best value, row as float bits) at the end
  unsigned* bar;      // grid-barrier counter, zero on entry
  float* best0;       // [M] row maxima of the final scores
  int *arg0, *arg1;   // [M] row arg-max, [N] column arg-max
  int* err_flag;
};

__device__ __forceinline__ void sk_online(float& m, float& s, float x) {  // (m, s) <- merge with one value x
  const float d = x - m;
  const float e = expf(-fabsf(d));
  s = d > 0.f ? fmaf(s, e, 1.f) : s + e;  // m = -inf: d = +inf, e = 0, s = 1
  m = fmaxf(m, x);
}
__device__ __forceinline__ void sk_merge(float& m, float& s, float m2, float s2) {  // merge two (max, sum) pairs
  const float mx = fmaxf(m, m2);
  if (mx == -INFINITY) {
    m = mx, s = 0.f;
    return;
  }
  s = s * expf(m - mx) + s2 * expf(m2 - mx);
  m = mx;
}
__device__ __forceinline__ bool sk_grid_barrier(unsigned* bar, unsigned& target, unsigned G) {
  __shared__ int sk_ok;
  __syncthreads();
  if (threadIdx.x == 0) {
    target += G;
    __threadfence();
    atomicAdd(bar, 1u);
    int ok = 0;
    for (unsigned spin = 0; spin < (1u << 26); ++spin) {
      if (*reinterpret_cast<volatile unsigned*>(bar) >= target) {
        ok = 1;
        break;
      }
    }
    __threadfence();
    sk_ok = ok;
  }
  __syncthreads();
  return sk_ok != 0;
}

__device__ __forceinline__ float sk_logsigmoid(float z) {  // F.logsigmoid: min(z, 0) - log1p(exp(-|z|))
  return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
}

template <int KIND>
__global__ void __launch_bounds__(SK_T, 1) k_assign_ps(const SinkArgs a) {
  constexpr int AUG = KIND == 0 ? 1 : 0;  // SuperGlue augments the score matrix with a dustbin row and column
  extern __shared__ __align__(16) float sk_smem[];
  __shared__ float red_m[SK_R][32], red_s[SK_R][32];
  __shared__ int red_i[SK_R][32];
  __shared__ float u_row[SK_R];
  __shared__ float rowc[SK_R][3];
  const int M = a.M, N = a.N, N1 = a.N + AUG, M1 = a.M + AUG;
  const int pitch = (N + 31) & ~31;  // floats per staged row
  float* colc = sk_smem + (size_t)SK_NB * SK_R * pitch;  // KIND 1: [3][N] column constants of the arg-max sweep (cmax, clog, lsg1)
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const unsigned G = gridDim.x;
  const int rows_per = (M1 + (int)G - 1) / (int)G;
  const int row0 = blockIdx.x * rows_per, row1 = min(M1, row0 + rows_per);  // (augmented) rows [row0, row1)
  const int nsteps = row1 > row0 ? (row1 - row0 + SK_R - 1) / SK_R : 0;
  const int nc = (N1 + SK_T - 1) / SK_T;  // columns this thread may own (<= SK_NC)
  unsigned target = 0;
  bool ok = true;

  auto stage_rows = [&](int step) {  // cp.async the (real) rows of a step into ring slot step % SK_NB
    float* dst = sk_smem + (size_t)(step % SK_NB) * SK_R * pitch;
    for (int r = 0; r < SK_R; ++r) {
      const int i = row0 + step * SK_R + r;
      if (i < M && i < row1) {
        const float* src = a.Z + (size_t)i * N;
        for (int j = t; j < N; j += SK_T) {
          const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst + r * pitch + j);
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(src + j) : "memory");
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  // one sweep over this CTA's rows.  MODE 0: Sinkhorn half-iterations (row LSE -> u, column partial LSE);
  // MODE 1: final scores (row arg-max -> best0 / arg0, column partial arg-max)
  auto sweep = [&](int mode, const float* vreg, float* c0, float* c1) {
    for (int s = 0; s < SK_NB - 1; ++s) {  // always SK_NB - 1 groups in the prologue: the wait below counts groups
      if (s < nsteps) stage_rows(s);
      else asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (int step = 0; step < nsteps; ++step) {
      if (step + SK_NB - 1 < nsteps) stage_rows(step + SK_NB - 1);
      else asm volatile("cp.async.commit_group;" ::: "memory");  // keep the group count uniform
      asm volatile("cp.async.wait_group %0;" ::"n"(SK_NB - 1) : "memory");
      __syncthreads();
      const float* buf = sk_smem + (size_t)(step % SK_NB) * SK_R * pitch;
      if (KIND == 1 && mode == 1 && t < SK_R * 3) {  // (rmax, rlog, lsg0) of this step's rows
        const int rr = t / 3, cc = t - rr * 3, i = row0 + step * SK_R + rr;
        rowc[rr][cc] = i < M ? (cc == 0 ? a.u[i] : (cc == 1 ? a.rlog[i] : a.lsg0[i])) : 0.f;
      }
      if (KIND == 1 && mode == 1) __syncthreads();
      float zr[SK_R][SK_NC];
#pragma unroll
      for (int r = 0; r < SK_R; ++r) {
        const int i = row0 + step * SK_R + r;
        float m = -INFINITY, sacc = 0.f;
        int bi = 0x7fffffff;
#pragma unroll
        for (int k = 0; k < SK_NC; ++k) {
          const int j = t + k * SK_T;
          zr[r][k] = 0.f;
          if (k < nc && j < N1 && i < row1) {
            const float z = (i < M && j < N) ? buf[r * pitch + j] : a.alpha;
            zr[r][k] = z;
            if (mode == 0) {
              sk_online(m, sacc, KIND == 0 ? z + vreg[k] : z);
            } else if (i < M && j < N) {
              float sc;
              if (KIND == 0) sc = ((z + a.u[i]) + vreg[k]) - a.norm;  // (superglue.py:169): Z + u + v - norm
              else sc = (((z - rowc[r][0]) - rowc[r][1]) + ((z - colc[j]) - colc[N + j])) + (rowc[r][2] + colc[2 * N + j]);  // (lightglue.py:269-274)
              if (sc > m) m = sc, bi = j;
            }
          }
        }
        // warp merge
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
          if (mode == 0) {
            const float s2 = __shfl_xor_sync(0xffffffffu, sacc, o);
            sk_merge(m, sacc, m2, s2);
          } else {
            const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
            if (m2 > m || (m2 == m && i2 < bi)) m = m2, bi = i2;
          }
        }
        if (lane == 0) red_m[r][warp] = m, red_s[r][warp] = sacc, red_i[r][warp] = bi;
      }
      __syncthreads();
      if (warp < SK_R) {  // warp r finishes row r
        const int i = row0 + step * SK_R + warp;
        float m = red_m[warp][lane], sacc = red_s[warp][lane];
        int bi = red_i[warp][lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
          if (mode == 0) {
            const float s2 = __shfl_xor_sync(0xffffffffu, sacc, o);
            sk_merge(m, sacc, m2, s2);
          } else {
            const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
            if (m2 > m || (m2 == m && i2 < bi)) m = m2, bi = i2;
          }
        }
        if (lane == 0 && i < row1) {
          if (mode == 0) {
            if (KIND == 0) {
              const float log_mu = i < M ? a.norm : logf((float)N) + a.norm;
              const float ui = log_mu - (m + logf(sacc));
              a.u[i] = ui;
              u_row[warp] = ui;
            } else {  // row statistics of log_softmax(sim, dim 2) and the row's logsigmoid term
              a.u[i] = m, a.rlog[i] = logf(sacc), a.lsg0[i] = sk_logsigmoid(a.z0[i]);
              u_row[warp] = 0.f;
            }
          } else if (i < M) {
            a.best0[i] = m;
            a.arg0[i] = bi == 0x7fffffff ? 0 : bi;  // no score beat -inf (a NaN row): best -inf, as the column merge does
          }
        }
      }
      if (mode == 0) __syncthreads();  // u_row visible
#pragma unroll
      for (int r = 0; r < SK_R; ++r) {
        const int i = row0 + step * SK_R + r;
        if (i >= row1) continue;
        const float ui = KIND == 1 ? 0.f : (mode == 0 ? u_row[r] : a.u[i]);
#pragma unroll
        for (int k = 0; k < SK_NC; ++k) {
          const int j = t + k * SK_T;
          if (k < nc && j < N1) {
            if (mode == 0) {
              sk_online(c0[k], c1[k], zr[r][k] + ui);
            } else if (i < M && j < N) {
              float sc;
              const float z = zr[r][k];
              if (KIND == 0) sc = ((z + ui) + vreg[k]) - a.norm;
              else sc = (((z - rowc[r][0]) - rowc[r][1]) + ((z - colc[j]) - colc[N + j])) + (rowc[r][2] + colc[2 * N + j]);
              if (sc > c0[k]) c0[k] = sc, c1[k] = __int_as_float(i);  // rows ascend: the first maximum is kept
            }
          }
        }
      }
      __syncthreads();  // every thread is done with this ring slot (and with red_* / u_row) before they are reused
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
  };

  float vreg[SK_NC], c0[SK_NC], c1[SK_NC];
  float* mine = a.part + (size_t)blockIdx.x * 2 * N1;
  const int cols_per = (N1 + (int)G - 1) / (int)G;
  const int col0 = blockIdx.x * cols_per, col1 = min(N1, col0 + cols_per);
  const int n_sweeps = KIND == 0 ? a.iters : 1;  // statistics sweeps before the arg-max sweep
  for (int it = 0; it <= n_sweeps; ++it) {
    const int mode = it == n_sweeps ? 1 : 0;
#pragma unroll
    for (int k = 0; k < SK_NC; ++k) {
      const int j = t + k * SK_T;
      vreg[k] = (KIND == 0 && it > 0 && k < nc && j < N1) ? __ldcg(a.v + j) : 0.f;  // v = 0 before the first iteration (superglue.py:145)
      c0[k] = -INFINITY, c1[k] = 0.f;
    }
    if (KIND == 1 && mode == 1) {  // column constants written by other CTAs in the merge below: (cmax, clog, lsg1)
      for (int j = t; j < N; j += SK_T) colc[j] = __ldcg(a.v + j), colc[N + j] = __ldcg(a.clog + j), colc[2 * N + j] = __ldcg(a.lsg1 + j);
      __syncthreads();
    }
    sweep(mode, vreg, c0, c1);
#pragma unroll
    for (int k = 0; k < SK_NC; ++k) {
      const int j = t + k * SK_T;
      if (k < nc && j < N1) mine[j] = c0[k], mine[N1 + j] = c1[k];
    }
    ok = sk_grid_barrier(a.bar, target, G) && ok;
    // column merge across the G row blocks: one warp per column
    for (int j = col0 + warp; j < col1; j += SK_T / 32) {
      float m = -INFINITY, sacc = 0.f;
      int bi = 0x7fffffff;
      for (unsigned g = lane; g < G; g += 32) {
        const float pm = __ldcg(a.part + (size_t)g * 2 * N1 + j), ps = __ldcg(a.part + (size_t)g * 2 * N1 + N1 + j);
        if (mode == 0) {
          sk_merge(m, sacc, pm, ps);
        } else {
          const int pi = __float_as_int(ps);
          if (pm > m || (pm == m && pm != -INFINITY && pi < bi)) m = pm, bi = pi;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
        if (mode == 0) {
          const float s2 = __shfl_xor_sync(0xffffffffu, sacc, o);
          sk_merge(m, sacc, m2, s2);
        } else {
          const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
          if (m2 > m || (m2 == m && i2 < bi)) m = m2, bi = i2;
        }
      }
      if (lane == 0) {
        if (mode == 0) {
          if (KIND == 0) {
            const float log_nu = j < N ? a.norm : logf((float)M) + a.norm;
            a.v[j] = log_nu - (m + logf(sacc));
          } else {  // column statistics of log_softmax(sim^T) and the column's logsigmoid term
            a.v[j] = m, a.clog[j] = logf(sacc), a.lsg1[j] = sk_logsigmoid(a.z1[j]);
          }
        } else if (j < N) {
          a.arg1[j] = bi == 0x7fffffff ? 0 : bi;
        }
      }
    }
    if (mode == 0) ok = sk_grid_barrier(a.bar, target, G) && ok;
  }
  if (!ok && t == 0 && a.err_flag) *a.err_flag = 1;
}


// host: one cooperative launch (all CTAs co-resident: the grid barrier needs it) of either instantiation
template <int KIND>
static int launch_assign_ps(b2_context* ctx, cudaStream_t st, SinkArgs sa, int G, const char* prof_name) {
  const int pitch = (sa.N + 31) & ~31;
  const size_t smem = ((size_t)SK_NB * SK_R * pitch + (KIND == 1 ? (size_t)3 * sa.N : 0)) * sizeof(float);
  B2_CUDA(ctx, cudaFuncSetAttribute(k_assign_ps<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  void* kargs[] = {&sa};
  const bool prof = ctx->prof.match(prof_name);
  if (prof) b2_prof_mark(ctx, st);
  b2_prof_work(ctx, prof_name, (double)((KIND == 0 ? sa.iters : 1) + 1) * sa.M * sa.N * 4.0);  // algorithmic bytes: the matrix once per sweep
  B2_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)k_assign_ps<KIND>, dim3(G), dim3(SK_T), kargs, smem, st));
  if (prof) b2_prof_mark(ctx, st);
  ctx->launches++;
  return B2_OK;
}
// the largest column count the persistent kernel serves (KIND 1 also keeps 3 x N column constants in shared memory)
static inline bool assign_ps_fits(int kind, int N) {
  const int pitch = (N + 31) & ~31;
  const size_t smem = ((size_t)SK_NB * SK_R * pitch + (kind == 1 ? (size_t)3 * N : 0)) * sizeof(float);
  return N + (kind == 0 ? 1 : 0) <= SK_NC * SK_T && smem <= 220 * 1024;
}
