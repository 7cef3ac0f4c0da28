// LMedS verifier for sm_90a: a batched restatement of cv2's LMeDSPointSetRegistrator (what the reference's LMEDS verifier,
// gtsfm/frontend/verifier/lmeds.py, calls through cv2.findEssentialMat / findFundamentalMat with method LMEDS).
//
// cv2's LMeDS is deterministic: one cv::RNG stream per call, a fixed iteration count and no early stop, the median of the
// float errors as the score.  So the device reproduces it rather than approximating it (oracle/lmeds_ref.py restates it in
// NumPy and tests/test_lmeds_cpu.py pins that restatement against cv2):
//   k_lm_subsets  one thread per problem draws the problem's whole subset table (serial RNG, F redraws collinear subsets)
//   k_lm_hyp      one thread per subset: every real root of the 5-point problem (E) or of the 7-point cubic (F)
//   k_lm_score    one CTA per (subset, solution) slot: the k float errors, then their (k/2)-th smallest by a radix select
//                 on the bit patterns (8-bit digits, 4 passes) over a shared-memory copy, or recomputed per pass when the
//                 problem is larger than shared memory
//   k_lm_select   one CTA per problem: the lowest median in visiting order, sigma, the inlier mask and its count
//   k_rs_pose     ransac.cu's cheirality vote, unchanged (F: E = K2^T F K1 on calibrated inliers)
// Every stage takes the table of a sub-batch (problem = blockIdx.y); the iteration count is known up front, so a sub-batch
// is 5 launches (6 with the gather) and one synchronisation.
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "ransac_prob.cuh"
// ransac.cu compiles the same header: its non-inline host functions get internal linkage here, so the two objects link.
// Marking them inline in the header instead would change how nvcc weighs inlining the RANSAC kernels' solvers.  The
// header's own includes (<math.h>) are made above, outside the namespace.
namespace {
#include "ransac_math.cuh"
}  // namespace

using namespace rmath;

namespace {
constexpr int LM_MAX_SOL = 10;
constexpr int LM_SCORE_THREADS = 256;
constexpr int LM_SMEM_POINTS = 11264;  // errors kept in shared memory (44 KB, under the 48 KB static + dynamic limit); larger problems recompute them per pass
constexpr int LM_SELECT_THREADS = 1024;
constexpr int LM_MAX_ITERS = 65536;
}  // namespace

struct LmOut {
  double model[9];
  double sigma;
  float min_median, thr;
  int slot, count, drawn, valid;
  double pose[13];
};

struct LmProb {
  const double *x1, *x2;  // [k][2]: calibrated (E) or pixels (F, read rounded to float32)
  int k, mode, niters;
  int* idx;               // [niters][m]
  int* nsol;              // [niters]
  double* models;         // [niters][10][9]
  float* med;             // [niters * 10]
  uint8_t* mask;
  LmOut* out;
};

struct LmedsState {
  DevBuf x1, x2, idx, nsol, models, med, mask, small, tab;
  HostBuf hbuf;
};

void lm_destroy(b2_context* ctx) {
  delete ctx->lm;
  ctx->lm = nullptr;
}

__device__ __forceinline__ double lm_pt(int mode, double v) { return mode == 0 ? v : (double)(float)v; }
__device__ __forceinline__ float lm_err(int mode, const double* M, const double* x1, const double* x2, int i) {
  return mode == 0 ? sampson_sq_cv(M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1])
                   : epiline_sq_cv(M, lm_pt(1, x1[2 * i]), lm_pt(1, x1[2 * i + 1]), lm_pt(1, x2[2 * i]), lm_pt(1, x2[2 * i + 1]));
}

__global__ void k_lm_subsets(const LmProb* __restrict__ tab) {
  const LmProb& p = tab[blockIdx.y];
  if (threadIdx.x == 0) p.out->drawn = lmeds_subsets(p.x1, p.x2, p.k, p.mode, p.niters, p.idx);
}

__global__ void __launch_bounds__(64) k_lm_hyp(const LmProb* __restrict__ tab) {
  const LmProb& p = tab[blockIdx.y];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.niters) return;
  if (s >= p.out->drawn) {
    p.nsol[s] = 0;
    return;
  }
  const int m = p.mode == 0 ? 5 : 7, mode = p.mode;
  double a[7][2], b[7][2];
  for (int i = 0; i < m; ++i) {
    const int j = p.idx[s * m + i];
    a[i][0] = lm_pt(mode, p.x1[2 * j]), a[i][1] = lm_pt(mode, p.x1[2 * j + 1]);
    b[i][0] = lm_pt(mode, p.x2[2 * j]), b[i][1] = lm_pt(mode, p.x2[2 * j + 1]);
  }
  double sol[LM_MAX_SOL][9];
  const int n = mode == 0 ? fivept_solve_all(a, b, sol) : sevenpt_solve(a, b, sol);
  p.nsol[s] = n;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < 9; ++i) p.models[((size_t)s * LM_MAX_SOL + j) * 9 + i] = sol[j][i];
}

// bit pattern whose unsigned order is the int32 order of the float's bits (cv2's nth_element on int*).  A NaN error (0 / 0,
// 0 * inf, inf - inf) is x86's default NaN in cv2, 0xffc00000 as a float: negative as int32, so it ranks below every
// number.  The device's arithmetic returns the positive canonical NaN instead, so it is replaced by x86's first.
__device__ __forceinline__ unsigned lm_key(float e) { return (e != e ? 0xffc00000u : __float_as_uint(e)) ^ 0x80000000u; }

__global__ void __launch_bounds__(LM_SCORE_THREADS) k_lm_score(const LmProb* __restrict__ tab) {
  const LmProb& p = tab[blockIdx.y];
  const int slot = blockIdx.x, s = slot / LM_MAX_SOL, j = slot % LM_MAX_SOL;
  if (s >= p.niters) return;
  if (j >= p.nsol[s]) {
    if (threadIdx.x == 0) p.med[slot] = __int_as_float(0x7fffffff);  // empty slot: NaN, never selected
    return;
  }
  extern __shared__ unsigned keys[];
  __shared__ double M[9];
  __shared__ unsigned hist[256];
  __shared__ unsigned prefix;
  __shared__ int rank;
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  const int k = p.k, mode = p.mode;
  const bool in_smem = k <= LM_SMEM_POINTS;
  if (threadIdx.x < 9) M[threadIdx.x] = p.models[(size_t)slot * 9 + threadIdx.x];
  if (threadIdx.x == 0) prefix = 0u, rank = k / 2;
  __syncthreads();
  if (in_smem)
    for (int i = threadIdx.x; i < k; i += LM_SCORE_THREADS) keys[i] = lm_key(lm_err(mode, M, x1, x2, i));
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const unsigned hi_mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = threadIdx.x; i < 256; i += LM_SCORE_THREADS) hist[i] = 0u;
    __syncthreads();
    const unsigned pre = prefix;
    for (int i = threadIdx.x; i < k; i += LM_SCORE_THREADS) {
      const unsigned key = in_smem ? keys[i] : lm_key(lm_err(mode, M, x1, x2, i));
      if ((key & hi_mask) == pre) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int r = rank;
      unsigned d = 0;
      for (; d < 255u; ++d) {
        if (r < (int)hist[d]) break;
        r -= (int)hist[d];
      }
      prefix = pre | (d << shift);
      rank = r;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) p.med[slot] = __uint_as_float(prefix ^ 0x80000000u);
}

// the lowest median in visiting order (slot order; a later slot must be strictly lower), then sigma and the mask
__global__ void __launch_bounds__(LM_SELECT_THREADS) k_lm_select(const LmProb* __restrict__ tab) {
  const LmProb& p = tab[blockIdx.y];
  const int n_slots = p.niters * LM_MAX_SOL, k = p.k, mode = p.mode;
  __shared__ float sv[LM_SELECT_THREADS];
  __shared__ int si[LM_SELECT_THREADS];
  __shared__ double M[9];
  __shared__ float thr;
  __shared__ int cnt[LM_SELECT_THREADS / 32];
  float bv = 0.f;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n_slots; i += LM_SELECT_THREADS) {
    const float v = p.med[i];
    if (v < __int_as_float(0x7f800000) && (bi == 0x7fffffff || v < bv)) bv = v, bi = i;  // NaN / inf: never (cv2: < DBL_MAX)
  }
  sv[threadIdx.x] = bv, si[threadIdx.x] = bi;
  __syncthreads();
  for (int o = LM_SELECT_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const float ov = sv[threadIdx.x + o];
      const int oi = si[threadIdx.x + o];
      if (oi != 0x7fffffff && (si[threadIdx.x] == 0x7fffffff || ov < sv[threadIdx.x] || (ov == sv[threadIdx.x] && oi < si[threadIdx.x])))
        sv[threadIdx.x] = ov, si[threadIdx.x] = oi;
    }
    __syncthreads();
  }
  LmOut* out = p.out;
  const int best = si[0];
  if (best == 0x7fffffff) {
    for (int i = threadIdx.x; i < k; i += LM_SELECT_THREADS) p.mask[i] = 0;
    if (threadIdx.x == 0) out->slot = -1, out->valid = 0, out->count = 0;
    return;
  }
  if (threadIdx.x < 9) M[threadIdx.x] = p.models[(size_t)best * 9 + threadIdx.x];
  if (threadIdx.x == 0) {
    const int m = mode == 0 ? 5 : 7;
    double sg = 2.5 * 1.4826 * (1 + 5. / (k - m)) * sqrt((double)sv[0]);
    sg = sg > 0.001 ? sg : 0.001;
    thr = (float)(sg * sg);
    out->sigma = sg, out->thr = thr, out->min_median = sv[0], out->slot = best;
  }
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < k; i += LM_SELECT_THREADS) {
    const bool in = lm_err(mode, M, p.x1, p.x2, i) <= thr;
    p.mask[i] = in ? 1 : 0;
    c += in;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) cnt[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < LM_SELECT_THREADS / 32; ++w) t += cnt[w];
    out->count = t;
    out->valid = mode == 0 || t >= 7;  // findEssentialMat returns the model whatever the count; findFundamentalMat needs m
    for (int i = 0; i < 9; ++i) out->model[i] = M[i];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------

struct LmScratch {
  int gvotes[8];
};

static int lm_clamp_iters(int max_iters) { return max_iters <= 0 ? 1000 : max_iters; }
static int lm_min_k(int mode) { return mode == 0 ? 6 : 8; }
static int lm_iters(const b2_ransac_problem& p, const b2_lmeds_params& prm) {
  return lmeds_niters(prm.confidence[p.mode], p.mode == 0 ? 5 : 7, lm_clamp_iters(p.max_iters));
}
constexpr size_t LM_SUBSET_BYTES = 7 * 4 + 4 + LM_MAX_SOL * (72 + 4);  // indices, nsol, models and medians of ten slots
constexpr size_t LM_FIXED_BYTES = sizeof(LmOut) + sizeof(LmScratch) + sizeof(LmProb) + sizeof(RsProb);
static size_t lm_problem_bytes(const b2_ransac_problem& p, const b2_lmeds_params& prm) {
  if (p.k < lm_min_k(p.mode)) return LM_FIXED_BYTES;
  return LM_FIXED_BYTES + (size_t)lm_iters(p, prm) * LM_SUBSET_BYTES + (p.x1 ? 0 : (size_t)p.k * 32) + (p.mask ? 0 : (size_t)p.k);
}
constexpr int LM_MAX_BATCH = 65535;  // problems per sub-batch: the kernels' gridDim.y
static int lm_plan(const b2_ransac_problem* problems, int n, const b2_lmeds_params& prm, size_t budget, int* first) {
  int count = 0, in_sub = 0;
  size_t used = 0;
  for (int i = 0; i < n; ++i) {
    const size_t b = lm_problem_bytes(problems[i], prm);
    if (i == 0 || used + b > budget || in_sub == LM_MAX_BATCH) first[count++] = i, used = 0, in_sub = 0;
    used += b;
    ++in_sub;
  }
  first[count] = n;
  return count;
}

#define LM_SYNC(ctx, st)                     \
  do {                                       \
    B2_CUDA(ctx, cudaStreamSynchronize(st)); \
    (ctx)->rs_syncs++;                       \
  } while (0)

// One sub-batch.  hx1 / hx2 / tr / hmask: the trace entry's single host problem (tests only).
static int lm_run_sub(b2_context* ctx, const b2_ransac_problem* probs, int n, const b2_lmeds_params& prm, b2_ransac_result* res,
                      cudaStream_t st, const double* hx1 = nullptr, const double* hx2 = nullptr, b2_lmeds_trace* tr = nullptr,
                      uint8_t* hmask = nullptr) {
  LmedsState* s = ctx->lm;
  std::vector<int> live;
  for (int i = 0; i < n; ++i) {
    memset(&res[i], 0, sizeof(res[i]));
    res[i].status = 1;
    const b2_ransac_problem& p = probs[i];
    if (p.k >= lm_min_k(p.mode)) live.push_back(i);
    else if (p.k > 0 && p.mask) B2_CUDA(ctx, cudaMemsetAsync(p.mask, 0, (size_t)p.k, st));
  }
  const int L = (int)live.size();
  if (L == 0) return B2_OK;
  size_t n_it = 0, n_x = 0, n_mask = 0;
  int max_k = 0, max_it = 0;
  bool any_gather = false;
  for (int i : live) {
    const int it = lm_iters(probs[i], prm);
    n_it += (size_t)it;
    max_it = it > max_it ? it : max_it;
    max_k = probs[i].k > max_k ? probs[i].k : max_k;
    if (!probs[i].x1) n_x += (size_t)probs[i].k;
    if (!probs[i].mask) n_mask += (size_t)probs[i].k;
  }
  const size_t small_bytes = (size_t)L * (sizeof(LmOut) + sizeof(LmScratch));
  B2_CUDA(ctx, s->x1.ensure(n_x * 16 + 16));
  B2_CUDA(ctx, s->x2.ensure(n_x * 16 + 16));
  B2_CUDA(ctx, s->idx.ensure(n_it * 7 * 4));
  B2_CUDA(ctx, s->nsol.ensure(n_it * 4));
  B2_CUDA(ctx, s->models.ensure(n_it * LM_MAX_SOL * 72));
  B2_CUDA(ctx, s->med.ensure(n_it * LM_MAX_SOL * 4));
  B2_CUDA(ctx, s->mask.ensure(n_mask + 16));
  B2_CUDA(ctx, s->small.ensure(small_bytes));
  B2_CUDA(ctx, s->tab.ensure((size_t)L * (sizeof(LmProb) + sizeof(RsProb))));
  B2_CUDA(ctx, s->hbuf.ensure((size_t)L * (sizeof(LmProb) + sizeof(RsProb) + sizeof(LmOut))));
  LmProb* hl = s->hbuf.as<LmProb>();
  RsProb* hr = reinterpret_cast<RsProb*>(hl + L);
  LmOut* hout = reinterpret_cast<LmOut*>(hr + L);
  LmProb* dl = s->tab.as<LmProb>();
  RsProb* dr = reinterpret_cast<RsProb*>(dl + L);
  LmOut* dout = s->small.as<LmOut>();
  LmScratch* dscr = reinterpret_cast<LmScratch*>(dout + L);
  B2_CUDA(ctx, cudaMemsetAsync(s->small.p, 0, small_bytes, st));
  size_t o_it = 0, o_x = 0, o_mask = 0;
  for (int t = 0; t < L; ++t) {
    const b2_ransac_problem& q = probs[live[t]];
    LmProb& l = hl[t];
    RsProb& r = hr[t];
    memset(&l, 0, sizeof(l));
    memset(&r, 0, sizeof(r));
    r.k = l.k = q.k;
    r.mode = l.mode = q.mode;
    l.niters = lm_iters(q, prm);
    if (q.x1) {
      l.x1 = q.x1, l.x2 = q.x2;
    } else {
      double* x1 = s->x1.as<double>() + 2 * o_x;
      double* x2 = s->x2.as<double>() + 2 * o_x;
      o_x += (size_t)q.k;
      l.x1 = x1, l.x2 = x2;
      if (hx1) {
        B2_CUDA(ctx, cudaMemcpyAsync(x1, hx1, (size_t)q.k * 16, cudaMemcpyHostToDevice, st));
        B2_CUDA(ctx, cudaMemcpyAsync(x2, hx2, (size_t)q.k * 16, cudaMemcpyHostToDevice, st));
      } else {
        r.kp1 = q.kp1, r.kp2 = q.kp2, r.matches = reinterpret_cast<const long long*>(q.matches);
        for (int c = 0; c < 3; ++c) r.g1[c] = q.mode == 0 ? q.cal1[c] : (c == 0), r.g2[c] = q.mode == 0 ? q.cal2[c] : (c == 0);
        any_gather = true;
      }
    }
    r.x1 = const_cast<double*>(l.x1), r.x2 = const_cast<double*>(l.x2);
    l.idx = s->idx.as<int>() + o_it * 7, l.nsol = s->nsol.as<int>() + o_it;
    l.models = s->models.as<double>() + o_it * LM_MAX_SOL * 9, l.med = s->med.as<float>() + o_it * LM_MAX_SOL;
    o_it += (size_t)l.niters;
    if (q.mask) l.mask = q.mask;
    else l.mask = s->mask.as<uint8_t>() + o_mask, o_mask += (size_t)q.k;
    l.out = dout + t;
    // pose: ransac.cu's k_rs_pose on the chosen model (F: pose_cal forms E = K2^T F K1 and calibrates the inliers)
    r.E = dout[t].model, r.pose_mask = l.mask, r.gvotes = dscr[t].gvotes, r.pose = dout[t].pose;
    r.pose_on = 1, r.pose_cal = q.mode == 1;
    for (int c = 0; c < 3; ++c) r.c1[c] = q.cal1[c], r.c2[c] = q.cal2[c];
  }
  B2_CUDA(ctx, cudaMemcpyAsync(dl, hl, (size_t)L * (sizeof(LmProb) + sizeof(RsProb)), cudaMemcpyHostToDevice, st));
  if (any_gather) {
    B2_LAUNCH(ctx, k_rs_gather, dim3(cdiv(max_k, 256), L), 256, 0, st, dr);
    B2_CHECK_LAUNCH(ctx);
  }
  B2_LAUNCH(ctx, k_lm_subsets, dim3(1, L), 32, 0, st, dl);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_lm_hyp, dim3(cdiv(max_it, 64), L), 64, 0, st, dl);
  B2_CHECK_LAUNCH(ctx);
  const size_t smem = (size_t)(max_k < LM_SMEM_POINTS ? max_k : LM_SMEM_POINTS) * 4;
  B2_LAUNCH(ctx, k_lm_score, dim3(max_it * LM_MAX_SOL, L), LM_SCORE_THREADS, smem, st, dl);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_lm_select, dim3(1, L), LM_SELECT_THREADS, 0, st, dl);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_rs_pose, dim3(cdiv(max_k, RS_POSE_THREADS), L), RS_POSE_THREADS, 0, st, dr);
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaMemcpyAsync(hout, dout, (size_t)L * sizeof(LmOut), cudaMemcpyDeviceToHost, st));
  if (tr) {
    const int m = hl[0].mode == 0 ? 5 : 7, it = hl[0].niters;
    const auto d2h = cudaMemcpyDeviceToHost;
    if (tr->idx) B2_CUDA(ctx, cudaMemcpyAsync(tr->idx, hl[0].idx, (size_t)it * m * 4, d2h, st));
    if (tr->nsol) B2_CUDA(ctx, cudaMemcpyAsync(tr->nsol, hl[0].nsol, (size_t)it * 4, d2h, st));
    if (tr->models) B2_CUDA(ctx, cudaMemcpyAsync(tr->models, hl[0].models, (size_t)it * LM_MAX_SOL * 72, d2h, st));
    if (tr->medians) B2_CUDA(ctx, cudaMemcpyAsync(tr->medians, hl[0].med, (size_t)it * LM_MAX_SOL * 4, d2h, st));
    if (hmask) B2_CUDA(ctx, cudaMemcpyAsync(hmask, hl[0].mask, (size_t)hl[0].k, d2h, st));
  }
  LM_SYNC(ctx, st);
  for (int t = 0; t < L; ++t) {
    b2_ransac_result& r = res[live[t]];
    const LmOut& o = hout[t];
    if (tr) {
      tr->niters = hl[0].niters, tr->drawn = o.drawn, tr->slot = o.slot, tr->min_median = o.min_median;
      tr->sigma = o.sigma, tr->thr = o.thr, tr->count = o.count;
    }
    r.num_inliers = o.count;
    if (!o.valid) continue;
    r.status = 0;
    memcpy(r.model, o.model, 9 * 8);
    memcpy(r.R, o.pose, 9 * 8), memcpy(r.t, o.pose + 9, 3 * 8);
  }
  return B2_OK;
}

static int lm_check(b2_context* ctx, const b2_ransac_problem* problems, int n, const b2_lmeds_params* params) {
  if (!params) return b2_fail(ctx, B2_ERR_ARG, "lmeds: params is NULL");
  for (int m = 0; m < 2; ++m)
    if (!(params->confidence[m] > 0.0 && params->confidence[m] < 1.0)) return b2_fail(ctx, B2_ERR_ARG, "lmeds: confidence must be in (0, 1)");
  for (int i = 0; i < n; ++i) {
    const b2_ransac_problem& p = problems[i];
    const std::string at = "lmeds problem " + std::to_string(i) + ": ";
    if (p.k < 0 || (p.mode != 0 && p.mode != 1)) return b2_fail(ctx, B2_ERR_ARG, at + "k < 0 or mode not 0 / 1");
    if (p.max_iters > LM_MAX_ITERS) return b2_fail(ctx, B2_ERR_ARG, at + "max_iters above 65536");
    const bool ready = p.x1 || p.x2;
    if (ready && (!p.x1 || !p.x2)) return b2_fail(ctx, B2_ERR_ARG, at + "x1 and x2 go together");
    if (p.k > 0 && !ready && (!p.kp1 || !p.kp2 || !p.matches)) return b2_fail(ctx, B2_ERR_ARG, at + "no points");
    if ((p.mode == 1 || !ready) && !(p.cal1[0] > 0.0 && p.cal2[0] > 0.0)) return b2_fail(ctx, B2_ERR_ARG, at + "focal length must be > 0");
  }
  return B2_OK;
}

extern "C" size_t b2_lmeds_workspace_bytes(const b2_ransac_problem* problem, const b2_lmeds_params* params) {
  if (!problem || !params || (problem->mode != 0 && problem->mode != 1) || problem->k < 0) return 0;
  return lm_problem_bytes(*problem, *params);
}

extern "C" int b2_lmeds_plan(const b2_ransac_problem* problems, int n, const b2_lmeds_params* params, size_t budget_bytes,
                             int* out_first) {
  if (n < 0 || !out_first || !params || (n > 0 && !problems)) return B2_ERR_ARG;
  for (int i = 0; i < n; ++i)
    if ((problems[i].mode != 0 && problems[i].mode != 1) || problems[i].k < 0) return B2_ERR_ARG;
  return lm_plan(problems, n, *params, budget_bytes, out_first);
}

extern "C" int b2_lmeds_verify_batched_dev(b2_context* ctx, const b2_ransac_problem* problems, int n, const b2_lmeds_params* params,
                                           b2_ransac_result* results, void* stream) {
  if (!ctx || n < 0 || (n > 0 && (!problems || !results))) return B2_ERR_ARG;
  if (int rc = lm_check(ctx, problems, n, params)) return rc;
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->lm) ctx->lm = new LmedsState();
  std::vector<int> first(n + 1);
  const int subs = lm_plan(problems, n, *params, (size_t)ctx->rs_workspace_mb << 20, first.data());
  cudaStream_t st = stream ? (cudaStream_t)stream : cudaStreamLegacy;
  for (int b = 0; b < subs; ++b)
    if (int rc = lm_run_sub(ctx, problems + first[b], first[b + 1] - first[b], *params, results + first[b], st)) return rc;
  return B2_OK;
}

extern "C" int b2_debug_lmeds_trace_host(b2_context* ctx, int mode, const double* x1, const double* x2, int k,
                                         const b2_lmeds_params* params, int max_iters, b2_lmeds_trace* trace,
                                         b2_ransac_result* result, uint8_t* out_mask) {
  if (!ctx || !x1 || !x2 || !trace || !result || k < 0 || (mode != 0 && mode != 1)) return B2_ERR_ARG;
  b2_ransac_problem p;
  memset(&p, 0, sizeof(p));
  p.k = k, p.mode = mode, p.max_iters = max_iters;
  p.cal1[0] = p.cal2[0] = 1.0;
  p.x1 = x1, p.x2 = x2;  // the check only tests them for NULL; the run uploads the host points into the workspace
  if (int rc = lm_check(ctx, &p, 1, params)) return rc;
  p.x1 = p.x2 = nullptr;
  if (k >= lm_min_k(mode) && trace->cap < lm_iters(p, *params)) return b2_fail(ctx, B2_ERR_ARG, "lmeds trace: cap below the iteration count");
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->lm) ctx->lm = new LmedsState();
  trace->niters = trace->drawn = trace->count = 0, trace->slot = -1;
  return lm_run_sub(ctx, &p, 1, *params, result, ctx->stream, x1, x2, trace, out_mask);
}
