// SuperGlue matcher for sm_90a, as GTSfM drives it (outdoor weights, 20 Sinkhorn iterations, threshold 0.2).
//
// Reference semantics restated (paths relative to the reference repo):
//   thirdparty/SuperGluePretrainedNetwork/models/superglue.py:63-82 (keypoint normalisation + encoder MLP),
//   :85-119 (multi-head attention + propagation MLP), :122-138 (18 alternating self / cross layers), :141-170
//   (log-space Sinkhorn optimal transport), :254-276 (score matrix, mutual arg-max, threshold); wrapper
//   gtsfm/frontend/matcher/superglue_matcher.py:47-115.
//
// Features are kept [N][256] row-major (the reference's (1, 256, N) transposed): every Conv1d(k=1) is the same NT GEMM
// as an nn.Linear and shares the wgmma split-fp16 kernels with LightGlue.  The host loader has already folded the
// eval-mode BatchNorms and permuted the q/k/v projection rows (and the merge columns) from the reference's
// channel = dim * 4 + head interleave (superglue.py:104) to head-major, so attention runs on plain [4][N][64] operands.
// It has also folded each layer's merge into its mlp.0 (weights.fold_message_projection): mlp.0 reads cat[x, ctx]
// straight from the attention output, and the message itself is never formed.
// The (M+1) x (N+1) coupling matrix is never materialised: the dustbin row / column are handled analytically.
#include <stdlib.h>

#include "common.cuh"
#include "linear.cuh"
#include "assign_ps.cuh"

namespace {
constexpr int SG_LAYERS = 18;
constexpr size_t SG_NFLOATS = 12003905;
struct SgLayerW {
  float *wq, *bq, *wk, *bk, *wv, *bv, *w0, *b0, *w3, *b3;  // w0 / b0: mlp.0 with merge folded in
};
}  // namespace

struct SgSide {
  DevBuf x, xs, q, k, v, ctx, h, hs, md, u, vv, best, arg;
  int n = 0;
};

// One array of the match, recorded when b2_set_option("superglue_trace", 1) is set (b2_superglue_trace_get).
struct SgTraceRec {
  int layer = 0, side = 0, n = 0, kind = 0, cols = 0;  // kind 0: x [n][256] after `layer`; 1: md [n][256]; 2: Z [n][cols]
  std::vector<float> v;
};

struct SuperGlueState {
  bool loaded = false, use_tc = true;
  DevBuf wblob, wblob_h, wblob_l, errflag;
  float *kw[5] = {}, *kb[5] = {};
  SgLayerW lw[SG_LAYERS];
  float *wf = nullptr, *bf = nullptr;
  float bin_score = 0.f;
  SgSide side[2];
  DevBuf sim, counters, attn_part, attn_ml, attn_cnt, sk_part, sk_bar;
  std::vector<SgTraceRec> trace;
};

void sg_destroy(b2_context* ctx) {
  delete ctx->sg;
  ctx->sg = nullptr;
}

// ------------------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------------------

// normalize_keypoints (superglue.py:63-70) + KeypointEncoder MLP 3 -> 32 -> 64 -> 128 -> 256 -> 256 (BatchNorm folded,
// ReLU between) + desc (+=) (superglue.py:243-244).  block = 256 threads, 8 keypoints; weights [cout][cin] fp32.
constexpr int KE_KP = 8;
struct KencW {
  const float* w[5];
  const float* b[5];
};
__global__ void __launch_bounds__(256) k_sg_kenc(const float* __restrict__ kp, const float* __restrict__ score,
                                                  const float* __restrict__ desc, int n, float cx, float cy, float scaling,
                                                  KencW W, float* __restrict__ x, __half* __restrict__ xh, __half* __restrict__ xl) {
  __shared__ float act[2][KE_KP][256];
  const int t = threadIdx.x, p0 = blockIdx.x * KE_KP;
  if (t < KE_KP * 3) {
    int k = t / 3, c = t % 3, p = p0 + k;
    float v = 0.f;
    if (p < n) v = c == 0 ? (kp[2 * p] - cx) / scaling : (c == 1 ? (kp[2 * p + 1] - cy) / scaling : score[p]);
    act[0][k][c] = v;
  }
  __syncthreads();
  const int dims[6] = {3, 32, 64, 128, 256, 256};
  int cur = 0;
  for (int l = 0; l < 5; ++l) {
    const int ci = dims[l], co = dims[l + 1];
    if (t < co) {
      float acc[KE_KP];
      const float b = W.b[l][t];
#pragma unroll
      for (int k = 0; k < KE_KP; ++k) acc[k] = b;
      const float* wr = W.w[l] + (size_t)t * ci;
      for (int c = 0; c < ci; ++c) {
        const float w = wr[c];
#pragma unroll
        for (int k = 0; k < KE_KP; ++k) acc[k] = fmaf(act[cur][k][c], w, acc[k]);
      }
#pragma unroll
      for (int k = 0; k < KE_KP; ++k) act[cur ^ 1][k][t] = l < 4 ? fmaxf(acc[k], 0.f) : acc[k];
    }
    __syncthreads();
    cur ^= 1;
  }
  for (int k = 0; k < KE_KP; ++k) {
    int p = p0 + k;
    if (p >= n) break;
    float v = desc[(size_t)p * 256 + t] + act[cur][k][t];
    x[(size_t)p * 256 + t] = v;
    if (xh) {
      __half hh, ll;
      tc::split_h(v, hh, ll);
      xh[(size_t)p * 256 + t] = hh;
      xl[(size_t)p * 256 + t] = ll;
    }
  }
}

// u[i] = log_mu[i] - logsumexp_j(Z[i][j] + v[j]) over the augmented row (superglue.py:146-147): j < N from the score
// matrix, j = N is the dustbin column (alpha); row M is the dustbin row (all alpha).  one warp per row.
__global__ void __launch_bounds__(256) k_sg_rows(const float* __restrict__ Z, int M, int N, const float* __restrict__ v,
                                                  float alpha, float norm, float* __restrict__ u) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i > M) return;
  float mx = -INFINITY;
  if (i < M) {
    const float* row = Z + (size_t)i * N;
    for (int j = lane; j < N; j += 32) mx = fmaxf(mx, row[j] + v[j]);
  } else {
    for (int j = lane; j < N; j += 32) mx = fmaxf(mx, alpha + v[j]);
  }
  if (lane == 0) mx = fmaxf(mx, alpha + v[N]);
  mx = warp_max(mx);
  float s = 0.f;
  if (i < M) {
    const float* row = Z + (size_t)i * N;
    for (int j = lane; j < N; j += 32) s += expf(row[j] + v[j] - mx);
  } else {
    for (int j = lane; j < N; j += 32) s += expf(alpha + v[j] - mx);
  }
  if (lane == 0) s += expf(alpha + v[N] - mx);
  s = warp_sum(s);
  if (lane == 0) {
    const float log_mu = i < M ? norm : logf((float)N) + norm;
    u[i] = log_mu - (mx + logf(s));
  }
}

// v[j] = log_nu[j] - logsumexp_i(Z[i][j] + u[i]) (superglue.py:148): a block owns 32 columns, 8 warps stride the rows
// with an online (max, sum); column N is the dustbin column.
__global__ void __launch_bounds__(256) k_sg_cols(const float* __restrict__ Z, int M, int N, const float* __restrict__ u,
                                                  float alpha, float norm, float* __restrict__ v) {
  __shared__ float sm[8][32], ss[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  float mx = -INFINITY, s = 0.f;
  if (j <= N) {
    for (int i = warp; i <= M; i += 8) {
      const float x = ((i < M && j < N) ? Z[(size_t)i * N + j] : alpha) + u[i];
      if (x > mx) {
        s = s * expf(mx - x) + 1.0f;
        mx = x;
      } else {
        s += expf(x - mx);
      }
    }
  }
  sm[warp][lane] = mx, ss[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && j <= N) {
    float Mx = sm[0][lane];
    for (int w = 1; w < 8; ++w) Mx = fmaxf(Mx, sm[w][lane]);
    float S = 0.f;
    for (int w = 0; w < 8; ++w)
      if (ss[w][lane] > 0.f) S += ss[w][lane] * expf(sm[w][lane] - Mx);
    const float log_nu = j < N ? norm : logf((float)M) + norm;
    v[j] = log_nu - (Mx + logf(S));
  }
}

// scores = ((Z + u) + v) - norm over the M x N core (superglue.py:169,266): row arg-max (first maximum), warp per row
__global__ void __launch_bounds__(256) k_sg_row_argmax(const float* __restrict__ Z, int M, int N, const float* __restrict__ u,
                                                        const float* __restrict__ v, float norm, float* __restrict__ best,
                                                        int* __restrict__ arg) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= M) return;
  const float* row = Z + (size_t)i * N;
  const float ui = u[i];
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < N; j += 32) {
    float sc = ((row[j] + ui) + v[j]) - norm;
    if (sc > bv) bv = sc, bi = j;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
  }
  if (lane == 0) best[i] = bv, arg[i] = bi == 0x7fffffff ? 0 : bi;  // no score beat -inf (a NaN row): k_sg_filter reads a1[arg]
}
__global__ void __launch_bounds__(256) k_sg_col_argmax(const float* __restrict__ Z, int M, int N, const float* __restrict__ u,
                                                        const float* __restrict__ v, float norm, int* __restrict__ arg) {
  __shared__ float sv[8][32];
  __shared__ int si[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  if (j < N) {
    const float vj = v[j];
    for (int i = warp; i < M; i += 8) {
      float sc = ((Z[(size_t)i * N + j] + u[i]) + vj) - norm;
      if (sc > bv) bv = sc, bi = i;
    }
  }
  sv[warp][lane] = bv, si[warp][lane] = bi;
  __syncthreads();
  if (warp == 0 && j < N) {
    for (int w = 1; w < 8; ++w) {
      float ov = sv[w][lane];
      int oi = si[w][lane];
      if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
    }
    arg[j] = bi == 0x7fffffff ? 0 : bi;
  }
}

// mutual arg-max + threshold (superglue.py:266-276) -> (i, matches0[i]) uint32 rows ascending in i
// (superglue_matcher.py:104-113).  single block, ordered compaction.
__global__ void __launch_bounds__(1024) k_sg_filter(const float* __restrict__ best0, const int* __restrict__ a0,
                                                     const int* __restrict__ a1, int m, float th, unsigned* __restrict__ out,
                                                     float* __restrict__ outs, int* __restrict__ count) {
  __shared__ int wtot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < m; base += 1024) {
    int i = base + threadIdx.x;
    bool valid = false;
    float ms = 0.f;
    int j = 0;
    if (i < m) {
      j = a0[i];
      bool mutual = a1[j] == i;
      ms = mutual ? expf(best0[i]) : 0.f;
      valid = mutual && ms > th;
    }
    unsigned vm = __ballot_sync(0xffffffffu, valid);
    if (lane == 0) wtot[warp] = __popc(vm);
    __syncthreads();
    if (warp == 0) {
      int w = wtot[lane], ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int uu = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += uu;
      }
      wtot[lane] = ws - w;
    }
    __syncthreads();
    int pos = carry + wtot[warp] + __popc(vm & ((1u << lane) - 1));
    if (valid) {
      out[2 * (size_t)pos] = (unsigned)i;
      out[2 * (size_t)pos + 1] = (unsigned)j;
      if (outs) outs[pos] = ms;
    }
    __syncthreads();
    if (threadIdx.x == 1023) carry = pos + (valid ? 1 : 0);
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = carry;
}

__global__ void k_sg_fill(float* p, int n, float v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------

extern "C" int b2_superglue_set_weights(b2_context* ctx, const float* blob, size_t n_floats) {
  if (!ctx || !blob) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (n_floats != SG_NFLOATS)
    return b2_fail(ctx, B2_ERR_ARG, "superglue blob must hold 12003905 floats (BatchNorm folded), got " + std::to_string(n_floats));
  cudaSetDevice(ctx->device);
  if (!ctx->sg) ctx->sg = new SuperGlueState();
  SuperGlueState* s = ctx->sg;
  std::vector<size_t> sizes;
  const int kd[6] = {3, 32, 64, 128, 256, 256};
  for (int l = 0; l < 5; ++l) sizes.push_back((size_t)kd[l + 1] * kd[l]), sizes.push_back(kd[l + 1]);
  for (int l = 0; l < SG_LAYERS; ++l) {
    const size_t z[] = {65536, 256, 65536, 256, 65536, 256, 65536, 256, 512 * 512, 512, 256 * 512, 256};
    for (size_t v : z) sizes.push_back(v);
  }
  sizes.push_back(65536), sizes.push_back(256), sizes.push_back(1);
  size_t total = 0, src_total = 0;
  std::vector<size_t> doff;
  for (size_t z : sizes) {
    doff.push_back(total);
    total += (z + 63) / 64 * 64;
    src_total += z;
  }
  if (src_total != SG_NFLOATS) return b2_fail(ctx, B2_ERR_STATE, "internal superglue layout mismatch");
  std::vector<float> host(total, 0.f);
  size_t so = 0;
  for (size_t i = 0; i < sizes.size(); ++i) {
    if (i >= 10 && (i - 10) % 12 == 6 && !folded_projection(blob + so, blob + so + sizes[i], 256))  // attn.merge of a GNN layer
      return b2_fail(ctx, B2_ERR_ARG, "superglue blob: layer " + std::to_string((i - 10) / 12) + "'s attn.merge is not folded into "
                                      "mlp.0 (pack the checkpoint with weights.pack_superglue)");
    memcpy(host.data() + doff[i], blob + so, sizes[i] * sizeof(float));
    so += sizes[i];
  }
  s->bin_score = blob[SG_NFLOATS - 1];
  B2_CUDA(ctx, s->wblob.ensure(total * sizeof(float)));
  B2_CUDA(ctx, s->wblob_h.ensure(total * sizeof(__half)));
  B2_CUDA(ctx, s->wblob_l.ensure(total * sizeof(__half)));
  B2_CUDA(ctx, s->errflag.ensure(16));
  B2_CUDA(ctx, s->counters.ensure(64));
  B2_CUDA(ctx, cudaMemset(s->errflag.p, 0, 16));
  B2_CUDA(ctx, cudaMemcpy(s->wblob.p, host.data(), total * sizeof(float), cudaMemcpyHostToDevice));
  B2_LAUNCH(ctx, k_split_f32, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)0, s->wblob.as<float>(), total,
            s->wblob_h.as<__half>(), s->wblob_l.as<__half>());
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaDeviceSynchronize());
  float* base = s->wblob.as<float>();
  size_t ti = 0;
  auto next = [&]() { return base + doff[ti++]; };
  for (int l = 0; l < 5; ++l) s->kw[l] = next(), s->kb[l] = next();
  for (int l = 0; l < SG_LAYERS; ++l) {
    SgLayerW& w = s->lw[l];
    w.wq = next(), w.bq = next(), w.wk = next(), w.bk = next(), w.wv = next(), w.bv = next(), next(), next();  // merge: the identity
    w.w0 = next(), w.b0 = next(), w.w3 = next(), w.b3 = next();
  }
  s->wf = next(), s->bf = next();
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_attn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FA_SMEM));
  s->use_tc = !b2_force_simt(ctx);
  s->loaded = true;
  return B2_OK;
}

// The assignment step on the score matrix Z [M][N]: log-space Sinkhorn (superglue.py:141-170), mutual arg-max and threshold
// (:266-276) -> the ordered match list.  u [M + 1] and v [N + 1] receive the duals, best0 / arg0 [M] and arg1 [N] the arg-max.
struct SgAssign {
  const float* Z;
  int M, N;
  float alpha;
  int iters;
  float thr;
  float *u, *v, *best0;
  int *arg0, *arg1;
  DevBuf *part, *bar;  // scratch of the persistent kernel
  int* err_flag;
  unsigned* out_matches;
  float* out_scores;
  int* count;
};

// path 0 runs the persistent kernel when it fits (what the matcher does), 1 forces it, 2 forces the multi-launch passes; G
// is the persistent kernel's CTA count.  *ran (when given) receives the path that ran, 1 or 2.
static int sg_assign(b2_context* ctx, cudaStream_t st, const SgAssign& p, int path, int G, int* ran) {
  const float* Z = p.Z;
  const int M = p.M, N = p.N, iters = p.iters;
  const float norm = -logf((float)(M + N));
  float* u = p.u;
  float* v = p.v;
  const bool persistent = path == 0 ? assign_ps_fits(0, N) : path == 1;
  if (persistent && !assign_ps_fits(0, N)) return b2_fail(ctx, B2_ERR_ARG, "the persistent Sinkhorn kernel holds at most 8191 columns");
  if (ran) *ran = persistent ? 1 : 2;
  int rc;
  if (persistent) {
    // persistent cooperative kernel: all iterations + the mutual arg-max passes in one launch, every score read once per iteration
    B2_CUDA(ctx, p.part->ensure((size_t)G * 2 * (N + 1) * sizeof(float)));
    B2_CUDA(ctx, p.bar->ensure(16));
    B2_CUDA(ctx, cudaMemsetAsync(p.bar->p, 0, 16, st));
    if (iters == 0) B2_CUDA(ctx, cudaMemsetAsync(u, 0, (size_t)(M + 1) * sizeof(float), st));
    SinkArgs sa{};
    sa.Z = Z, sa.M = M, sa.N = N, sa.alpha = p.alpha, sa.norm = norm, sa.iters = iters, sa.u = u, sa.v = v;
    sa.part = p.part->as<float>(), sa.bar = p.bar->as<unsigned>(), sa.best0 = p.best0, sa.arg0 = p.arg0;
    sa.arg1 = p.arg1, sa.err_flag = p.err_flag;
    if ((rc = launch_assign_ps<0>(ctx, st, sa, G, "k_sg_sinkhorn"))) return rc;
  } else {
    B2_LAUNCH(ctx, k_sg_fill, cdiv(N + 1, 256), 256, 0, st, v, N + 1, 0.f);
    B2_CHECK_LAUNCH(ctx);
    for (int it = 0; it < iters; ++it) {
      B2_LAUNCH(ctx, k_sg_rows, cdiv(M + 1, 8), 256, 0, st, Z, M, N, v, p.alpha, norm, u);
      B2_CHECK_LAUNCH(ctx);
      B2_LAUNCH(ctx, k_sg_cols, cdiv(N + 1, 32), 256, 0, st, Z, M, N, u, p.alpha, norm, v);
      B2_CHECK_LAUNCH(ctx);
    }
    if (iters == 0) {
      B2_LAUNCH(ctx, k_sg_fill, cdiv(M + 1, 256), 256, 0, st, u, M + 1, 0.f);
      B2_CHECK_LAUNCH(ctx);
    }
    B2_LAUNCH(ctx, k_sg_row_argmax, cdiv(M, 8), 256, 0, st, Z, M, N, u, v, norm, p.best0, p.arg0);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_sg_col_argmax, cdiv(N, 32), 256, 0, st, Z, M, N, u, v, norm, p.arg1);
    B2_CHECK_LAUNCH(ctx);
  }
  B2_LAUNCH(ctx, k_sg_filter, 1, 1024, 0, st, p.best0, p.arg0, p.arg1, M, p.thr, p.out_matches, p.out_scores, p.count);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// Appends the n x cols fp32 array in `d` to the trace (synchronises the stream).  With `planes`, `d` holds split-fp16
// planes instead (hi [n * cols], then lo [n * cols] scaled by 2^11, as the wgmma path writes a linear's plane output): the
// record is hi + lo * 2^-11, the value the next GEMM reads.
static int sg_trace_push(b2_context* ctx, cudaStream_t st, SuperGlueState* s, int layer, int side, int kind, int n, int cols,
                         const DevBuf& d, bool planes) {
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  SgTraceRec r;
  r.layer = layer, r.side = side, r.n = n, r.kind = kind, r.cols = cols;
  const size_t e = (size_t)n * cols;
  r.v.resize(e);
  if (planes) {
    std::vector<__half> h(2 * e);
    B2_CUDA(ctx, cudaMemcpy(h.data(), d.p, h.size() * sizeof(__half), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < e; ++i) r.v[i] = (float)((double)__half2float(h[i]) + (double)__half2float(h[e + i]) / (double)tc::LO_SCALE);
  } else {
    B2_CUDA(ctx, cudaMemcpy(r.v.data(), d.p, e * sizeof(float), cudaMemcpyDeviceToHost));
  }
  s->trace.push_back(std::move(r));
  return B2_OK;
}

static int sg_trace_x(b2_context* ctx, cudaStream_t st, SuperGlueState* s, int layer) {
  for (int i = 0; i < 2; ++i) {
    int rc = sg_trace_push(ctx, st, s, layer, i, 0, s->side[i].n, 256, s->side[i].x, false);
    if (rc) return rc;
  }
  return B2_OK;
}

static int sg_match_impl(b2_context* ctx,const float* kp0, const float* sc0, const float* desc0, int n0, int h0, int w0,
                         const float* kp1, const float* sc1, const float* desc1, int n1, int h1, int w1, int iters, float thr,
                         unsigned* out_matches, float* out_scores, int* out_k, cudaStream_t st) {
  SuperGlueState* s = ctx->sg;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "superglue weights not set");
  s->trace.clear();
  *out_k = 0;
  if (n0 <= 0 || n1 <= 0) return B2_OK;  // superglue.py:233-240
  TcWeights tw{s->wblob.as<float>(), s->wblob_h.as<__half>(), s->wblob_l.as<__half>(), s->errflag.as<int>(), s->use_tc};
  tw.attn_part = &s->attn_part, tw.attn_ml = &s->attn_ml, tw.attn_cnt = &s->attn_cnt;
  tw.sm_count = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  int rc;
  const float* kps[2] = {kp0, kp1};
  const float* scs[2] = {sc0, sc1};
  const float* descs[2] = {desc0, desc1};
  const int ns[2] = {n0, n1}, hs_[2] = {h0, h1}, ws_[2] = {w0, w1};
  KencW kw;
  for (int l = 0; l < 5; ++l) kw.w[l] = s->kw[l], kw.b[l] = s->kb[l];
  for (int i = 0; i < 2; ++i) {
    SgSide& sd = s->side[i];
    const size_t N = (size_t)ns[i];
    sd.n = ns[i];
    DevBuf* b256[] = {&sd.x, &sd.xs, &sd.q, &sd.k, &sd.v, &sd.ctx, &sd.md};
    for (DevBuf* b : b256) B2_CUDA(ctx, b->ensure(N * 256 * 4));
    B2_CUDA(ctx, sd.h.ensure(N * 512 * 4));
    B2_CUDA(ctx, sd.hs.ensure(N * 512 * 4));
    DevBuf* small[] = {&sd.u, &sd.vv, &sd.best, &sd.arg};
    for (DevBuf* b : small) B2_CUDA(ctx, b->ensure((N + 1) * 4));
    const Pl xp = planes_of(sd.xs, N * 256);
    const float fw = (float)ws_[i], fh = (float)hs_[i];
    B2_LAUNCH(ctx, k_sg_kenc, cdiv(ns[i], KE_KP), 256, 0, st, kps[i], scs[i], descs[i], ns[i], fw / 2.0f, fh / 2.0f,
              fmaxf(fw, fh) * 0.7f, kw, sd.x.as<float>(), s->use_tc ? xp.hi : (__half*)nullptr, s->use_tc ? xp.lo : (__half*)nullptr);
    B2_CHECK_LAUNCH(ctx);
  }
  if (ctx->sg_trace && (rc = sg_trace_x(ctx, st, s, -1))) return rc;
  SgSide &a = s->side[0], &b = s->side[1];
  auto PL = [](DevBuf& buf, int n, int width) { return planes_of(buf, (size_t)n * width); };
  for (int l = 0; l < SG_LAYERS; ++l) {
    const SgLayerW& w = s->lw[l];
    const bool cross = (l & 1) != 0;  // superglue.py:199: ['self', 'cross'] * 9
    // q from x; k, v from the source (x itself, or the other image for cross layers): one two-image launch each
    const float* wts[3] = {w.wq, w.wk, w.wv};
    const float* bs[3] = {w.bq, w.bk, w.bv};
    for (int which = 0; which < 3; ++which) {
      LinArgs p[2];
      for (int i = 0; i < 2; ++i) {
        SgSide& sd = s->side[i];
        LinArgs& g = p[i];
        g.a1f = sd.x.as<float>(), g.a1p = PL(sd.xs, sd.n, 256), g.lda1 = 256, g.K1 = 256, g.w = wts[which], g.ldb = 256, g.bias = bs[which];
        DevBuf& dst = which == 0 ? sd.q : (which == 1 ? sd.k : sd.v);
        g.cf = dst.as<float>(), g.cp = PL(dst, sd.n, 256), g.head_major = 1, g.M = sd.n, g.N = 256;
        g.lo_unscaled = tw.use_tc ? 1 : 0;  // attention operands
      }
      if ((rc = run_linear(ctx, st, tw, p, 2))) return rc;
    }
    SgSide &sa = cross ? b : a, &sb = cross ? a : b;  // sources of image 0 / image 1
    const FlashJob fj[2] = {{&a.q, &sa.k, &sa.v, &a.ctx, a.n, sa.n, a.n, sa.n}, {&b.q, &sb.k, &sb.v, &b.ctx, b.n, sb.n, b.n, sb.n}};
    if ((rc = run_flash(ctx, st, tw, fj, 2, 0.125f))) return rc;
    LinArgs f0[2], f3[2];
    for (int i = 0; i < 2; ++i) {
      SgSide& sd = s->side[i];
      LinArgs& f = f0[i];  // mlp.0 (BatchNorm and merge folded) + ReLU on cat([x, ctx]) = mlp.0 on cat([x, message])
      f.a1f = sd.x.as<float>(), f.a1p = PL(sd.xs, sd.n, 256), f.lda1 = 256, f.K1 = 256;
      f.a2f = sd.ctx.as<float>(), f.a2p = PL(sd.ctx, sd.n, 256), f.lda2 = 256, f.K2 = 256;
      f.w = w.w0, f.ldb = 512, f.bias = w.b0, f.relu = 1, f.cf = sd.h.as<float>(), f.ldc = 512, f.cp = PL(sd.hs, sd.n, 512), f.ldch = 512;
      f.M = sd.n, f.N = 512;
      LinArgs& c = f3[i];  // desc + mlp.3(...)  (superglue.py:136-137)
      c.a1f = sd.h.as<float>(), c.a1p = PL(sd.hs, sd.n, 512), c.lda1 = 512, c.K1 = 512, c.w = w.w3, c.ldb = 512, c.bias = w.b3;
      c.resid = sd.x.as<float>(), c.ldr = 256, c.cf = sd.x.as<float>(), c.ldc = 256, c.tc_want_f32 = true;
      c.cp = PL(sd.xs, sd.n, 256), c.ldch = 256, c.M = sd.n, c.N = 256;
    }
    if ((rc = run_linear(ctx, st, tw, f0, 2))) return rc;
    if ((rc = run_linear(ctx, st, tw, f3, 2))) return rc;
    if (ctx->sg_trace && (rc = sg_trace_x(ctx, st, s, l))) return rc;
  }
  // final projection + score matrix / sqrt(256) (superglue.py:251-258)
  {
    LinArgs p[2];
    for (int i = 0; i < 2; ++i) {
      SgSide& sd = s->side[i];
      LinArgs& g = p[i];
      g.a1f = sd.x.as<float>(), g.a1p = PL(sd.xs, sd.n, 256), g.lda1 = 256, g.K1 = 256, g.w = s->wf, g.ldb = 256, g.bias = s->bf;
      g.cf = sd.md.as<float>(), g.ldc = 256, g.cp = PL(sd.md, sd.n, 256), g.ldch = 256, g.M = sd.n, g.N = 256;
    }
    if ((rc = run_linear(ctx, st, tw, p, 2))) return rc;
    for (int i = 0; ctx->sg_trace && i < 2; ++i)
      if ((rc = sg_trace_push(ctx, st, s, SG_LAYERS, i, 1, s->side[i].n, 256, s->side[i].md, s->use_tc))) return rc;
  }
  const int M = a.n, N = b.n;
  B2_CUDA(ctx, s->sim.ensure((size_t)M * N * 4));
  LinArgs gs;
  gs.a1f = a.md.as<float>(), gs.a1p = PL(a.md, a.n, 256), gs.lda1 = 256, gs.K1 = 256;
  gs.bf = b.md.as<float>(), gs.bp = PL(b.md, b.n, 256), gs.ldb = 256, gs.scale = 1.0f / 16.0f;
  gs.cf = s->sim.as<float>(), gs.ldc = N, gs.tc_want_f32 = true, gs.M = M, gs.N = N;
  if ((rc = run_linear(ctx, st, tw, &gs, 1))) return rc;
  if (ctx->sg_trace && (rc = sg_trace_push(ctx, st, s, SG_LAYERS, -1, 2, M, N, s->sim, false))) return rc;
  // log-space Sinkhorn (superglue.py:141-170); u lives in a.u [M+1], v in b.vv [N+1]
  int* counters = s->counters.as<int>();
  const SgAssign sg{s->sim.as<float>(), M, N, s->bin_score, iters, thr, a.u.as<float>(), b.vv.as<float>(), a.best.as<float>(),
                    a.arg.as<int>(), b.arg.as<int>(), &s->sk_part, &s->sk_bar, s->errflag.as<int>(), out_matches, out_scores, counters};
  if ((rc = sg_assign(ctx, st, sg, 0, tw.sm_count, nullptr))) return rc;
  int hres[2] = {0, 0};
  B2_CUDA(ctx, cudaMemcpyAsync(&hres[0], counters, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&hres[1], s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (hres[1]) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  *out_k = hres[0];
  ctx->debug["sg_desc0"] = {a.x.as<float>(), (int64_t)a.n * 256};
  return B2_OK;
}

extern "C" int b2_superglue_match_dev(b2_context* ctx, const float* kp0, const float* score0, const float* desc0, int n0, int h0,
                                      int w0, const float* kp1, const float* score1, const float* desc1, int n1, int h1, int w1,
                                      int sinkhorn_iters, float match_threshold, uint32_t* out_matches, float* out_scores,
                                      int* out_k, void* stream) {
  if (!ctx || !out_k || n0 < 0 || n1 < 0 || sinkhorn_iters < 0) return B2_ERR_ARG;
  if (n0 > 0 && n1 > 0 && (!kp0 || !score0 || !desc0 || !kp1 || !score1 || !desc1 || !out_matches)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return sg_match_impl(ctx, kp0, score0, desc0, n0, h0, w0, kp1, score1, desc1, n1, h1, w1, sinkhorn_iters, match_threshold,
                       out_matches, out_scores, out_k, (cudaStream_t)stream);
}

extern "C" int b2_superglue_match_host(b2_context* ctx, const float* kp0, const float* score0, const float* desc0, int n0, int h0,
                                       int w0, const float* kp1, const float* score1, const float* desc1, int n1, int h1, int w1,
                                       int sinkhorn_iters, float match_threshold, uint32_t* out_matches, float* out_scores,
                                       int* out_k) {
  if (!ctx || !out_k || n0 < 0 || n1 < 0 || sinkhorn_iters < 0) return B2_ERR_ARG;
  *out_k = 0;
  if (n0 == 0 || n1 == 0) return B2_OK;
  if (!kp0 || !score0 || !desc0 || !kp1 || !score1 || !desc1 || !out_matches) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int mk = n0 < n1 ? n0 : n1;
  const float* hp[6] = {kp0, score0, desc0, kp1, score1, desc1};
  const size_t bytes[6] = {(size_t)n0 * 8, (size_t)n0 * 4, (size_t)n0 * 1024, (size_t)n1 * 8, (size_t)n1 * 4, (size_t)n1 * 1024};
  for (int i = 0; i < 6; ++i) {
    B2_CUDA(ctx, ctx->stage_d[i].ensure(bytes[i]));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->stage_d[i].p, hp[i], bytes[i], cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(ctx, ctx->stage_d[6].ensure((size_t)mk * 8));
  B2_CUDA(ctx, ctx->stage_d[7].ensure((size_t)mk * 4));
  int rc = sg_match_impl(ctx, ctx->stage_d[0].as<float>(), ctx->stage_d[1].as<float>(), ctx->stage_d[2].as<float>(), n0, h0, w0,
                         ctx->stage_d[3].as<float>(), ctx->stage_d[4].as<float>(), ctx->stage_d[5].as<float>(), n1, h1, w1,
                         sinkhorn_iters, match_threshold, ctx->stage_d[6].as<unsigned>(), ctx->stage_d[7].as<float>(), out_k, st);
  if (rc) return rc;
  if (*out_k > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(out_matches, ctx->stage_d[6].p, (size_t)*out_k * 8, cudaMemcpyDeviceToHost, st));
    if (out_scores) B2_CUDA(ctx, cudaMemcpyAsync(out_scores, ctx->stage_d[7].p, (size_t)*out_k * 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return B2_OK;
}

// ---- the per-layer trace (b2_set_option "superglue_trace") ------------------------------------------------------------------

extern "C" int b2_superglue_trace_count(b2_context* ctx) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return ctx->sg ? (int)ctx->sg->trace.size() : 0;
}

extern "C" int b2_superglue_trace_get(b2_context* ctx, int i, int* meta, float* out) {
  if (!ctx || !meta) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->sg || i < 0 || i >= (int)ctx->sg->trace.size()) return b2_fail(ctx, B2_ERR_ARG, "no such superglue trace record");
  const SgTraceRec& r = ctx->sg->trace[i];
  const int m[5] = {r.layer, r.side, r.n, r.kind, r.cols};
  memcpy(meta, m, sizeof(m));
  if (out) memcpy(out, r.v.data(), r.v.size() * sizeof(float));
  return B2_OK;
}

// ---- test-only entry point: the assignment step on its own, on a host score matrix ------------------------------------------

extern "C" int b2_debug_superglue_assign_host(b2_context* ctx, int path, int ctas, const float* Z, int M, int N, float alpha, int iters,
                                              float threshold, float* u, float* v, float* best0, int* arg0, int* arg1,
                                              uint32_t* out_matches, float* out_scores, int* out_k, int* out_path) {
  if (!ctx || !Z || !u || !v || !best0 || !arg0 || !arg1 || !out_matches || !out_scores || !out_k || !out_path || M <= 0 || N <= 0 ||
      iters < 0 || path < 0 || path > 2 || ctas < 0 || ctas > ctx->sm_count)
    return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  DevBuf dZ, du, dv, dbest, da0, da1, part, bar, err, out, outs, cnt;
  B2_CUDA(ctx, dZ.ensure((size_t)M * N * 4));
  B2_CUDA(ctx, du.ensure((size_t)(M + 1) * 4));
  B2_CUDA(ctx, dv.ensure((size_t)(N + 1) * 4));
  B2_CUDA(ctx, dbest.ensure((size_t)M * 4));
  B2_CUDA(ctx, da0.ensure((size_t)M * 4));
  B2_CUDA(ctx, da1.ensure((size_t)N * 4));
  B2_CUDA(ctx, err.ensure(16));
  B2_CUDA(ctx, out.ensure((size_t)M * 8));
  B2_CUDA(ctx, outs.ensure((size_t)M * 4));
  B2_CUDA(ctx, cnt.ensure(16));
  B2_CUDA(ctx, cudaMemcpyAsync(dZ.p, Z, (size_t)M * N * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(err.p, 0, 16, st));
  // without iterations the persistent kernel never writes v; the reference's v is then its initial 0
  if (iters == 0) B2_CUDA(ctx, cudaMemsetAsync(dv.p, 0, (size_t)(N + 1) * 4, st));
  const int G = ctas > 0 ? ctas : (ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1);
  const SgAssign p{dZ.as<float>(), M, N, alpha, iters, threshold, du.as<float>(), dv.as<float>(), dbest.as<float>(), da0.as<int>(),
                   da1.as<int>(), &part, &bar, err.as<int>(), out.as<unsigned>(), outs.as<float>(), cnt.as<int>()};
  const int rc = sg_assign(ctx, st, p, path, G, out_path);
  if (rc) return rc;
  int k = 0, e = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&k, cnt.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&e, err.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(u, du.p, (size_t)(M + 1) * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(v, dv.p, (size_t)(N + 1) * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(best0, dbest.p, (size_t)M * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(arg0, da0.p, (size_t)M * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(arg1, da1.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (k > 0) {
    B2_CUDA(ctx, cudaMemcpy(out_matches, out.p, (size_t)k * 8, cudaMemcpyDeviceToHost));
    B2_CUDA(ctx, cudaMemcpy(out_scores, outs.p, (size_t)k * 4, cudaMemcpyDeviceToHost));
  }
  *out_k = k;
  if (e) return b2_fail(ctx, B2_ERR_STATE, "the persistent assignment kernel timed out in its grid barrier (kernel bug)");
  return B2_OK;
}
