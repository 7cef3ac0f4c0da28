// RANSAC verifier for sm_90a: 5-point essential / 8-point fundamental hypotheses, squared-Sampson (E) or
// symmetric-epiline (F) MSAC scoring, least-squares local optimisation, cheirality pose recovery.
//
// Replaces what the reference delegates to OpenCV at gtsfm/frontend/verifier/ransac.py:74-81,103-110 and
// gtsfm/utils/verification.py:83 (cv2.findEssentialMat USAC_ACCURATE / cv2.findFundamentalMat FM_RANSAC /
// cv2.recoverPose).  USAC's sampler and graph-cut local optimisation are not reproducible (SURVEY.md §7 hard part 4):
// parity for this row is the reference tests' own criteria + inlier-set agreement with cv2 on seeded scenes.
//
// Work decomposition: hypotheses are generated one per thread (fp64 minimal solvers from ransac_math.cuh), scored one
// CTA per model over all matches, reduced to the best model by a single CTA, then refined / masked / decomposed by
// single-CTA kernels.  Everything is deterministic for a given seed (fixed-order reductions, counter-based RNG).
#include <string.h>

#include "common.cuh"
#include "ransac_math.cuh"

using namespace rmath;

namespace {
constexpr int RS_MAX_SOL = 10;
constexpr int RS_SCORE_THREADS = 128;
constexpr int RS_LO_THREADS = 512;
constexpr int RS_LO_ITERS = 6;
constexpr int RS_TOP = 8;  // hypotheses handed to the local optimisation (the refined candidate with the lowest MSAC cost wins)
constexpr int RS_BATCH = 16384;  // hypotheses per launch (buffers are sized for it; a trace may ask for fewer)
}  // namespace

struct RansacState {
  DevBuf x1, x2, models, nsol, cost, ninl, best, mask, pose;
  HostBuf hbuf;
};

void rs_destroy(b2_context* ctx) {
  delete ctx->rs;
  ctx->rs = nullptr;
}

// best-model record kept on the device between batches (the header's b2_ransac_candidate, so traces copy it as is)
using RsBest = b2_ransac_candidate;

__device__ __forceinline__ double rs_err(int mode, const double* M, double a, double b, double c, double d) {
  return mode == 0 ? sampson_sq(M, a, b, c, d) : epiline_sq(M, a, b, c, d);
}

// ---- hypothesis generation -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) k_rs_hyp_E(const double* __restrict__ x1, const double* __restrict__ x2, int k,
                                                  unsigned long long seed, int sample0, int n_samples,
                                                  double* __restrict__ models, int* __restrict__ nsol, const int* __restrict__ go) {
  if (go && !*go) return;  // extension stage not needed (decided on the device by k_rs_select)
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_samples) return;
  int idx[5];
  sample_distinct(seed, (unsigned long long)(sample0 + s), k, 5, idx);
  double a[5][2], b[5][2];
  for (int i = 0; i < 5; ++i) {
    a[i][0] = x1[2 * idx[i]], a[i][1] = x1[2 * idx[i] + 1];
    b[i][0] = x2[2 * idx[i]], b[i][1] = x2[2 * idx[i] + 1];
  }
  double sol[RS_MAX_SOL][9];
  int n = fivept_solve(a, b, sol);
  nsol[s] = n;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < 9; ++i) models[((size_t)s * RS_MAX_SOL + j) * 9 + i] = sol[j][i];
}

// normalised 8-point algorithm on one 8-sample (Hartley 1997): one F per sample
__global__ void __launch_bounds__(64) k_rs_hyp_F(const double* __restrict__ x1, const double* __restrict__ x2, int k,
                                                  unsigned long long seed, int sample0, int n_samples,
                                                  double* __restrict__ models, int* __restrict__ nsol) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_samples) return;
  int idx[8];
  sample_distinct(seed, (unsigned long long)(sample0 + s), k, 8, idx);
  double a[8][2], b[8][2];
  for (int i = 0; i < 8; ++i) {
    a[i][0] = x1[2 * idx[i]], a[i][1] = x1[2 * idx[i] + 1];
    b[i][0] = x2[2 * idx[i]], b[i][1] = x2[2 * idx[i] + 1];
  }
  const int n = eightpt_solve(a, b, models + (size_t)s * RS_MAX_SOL * 9);
  nsol[s] = n;
}

// ---- scoring: one CTA per model slot ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(RS_SCORE_THREADS) k_rs_score(const double* __restrict__ models, const int* __restrict__ nsol,
                                                                const double* __restrict__ x1, const double* __restrict__ x2,
                                                                int k, double thr2, int mode, double* __restrict__ cost,
                                                                int* __restrict__ ninl, const int* __restrict__ go) {
  if (go && !*go) return;
  const int slot = blockIdx.x, s = slot / RS_MAX_SOL, j = slot % RS_MAX_SOL;
  if (j >= nsol[s]) {
    if (threadIdx.x == 0) cost[slot] = 1e300, ninl[slot] = 0;
    return;
  }
  __shared__ double M[9];
  __shared__ double wc[RS_SCORE_THREADS / 32];
  __shared__ int wn[RS_SCORE_THREADS / 32];
  if (threadIdx.x < 9) M[threadIdx.x] = models[(size_t)slot * 9 + threadIdx.x];
  __syncthreads();
  double c = 0;
  int n = 0;
  for (int i = threadIdx.x; i < k; i += RS_SCORE_THREADS) {
    double e = rs_err(mode, M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
    bool in = e < thr2;
    c += in ? e : thr2;  // MSAC
    n += in;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xffffffffu, c, o);
    n += __shfl_xor_sync(0xffffffffu, n, o);
  }
  if ((threadIdx.x & 31) == 0) wc[threadIdx.x >> 5] = c, wn[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    double cc = 0;
    int nn = 0;
    for (int w = 0; w < RS_SCORE_THREADS / 32; ++w) cc += wc[w], nn += wn[w];
    cost[slot] = cc;
    ninl[slot] = nn;
  }
}

// ---- selection: the RS_TOP lowest MSAC costs of this batch merged with the running candidate list (ties -> lower slot) ----
// cand[0 .. RS_TOP) is kept sorted by (cost, arrival); each round is one block arg-min over the slots that come after the
// previous winner in (cost, index) order.  A contaminated sample (4 of 5 inliers) usually scores close to the best one and
// converges to the right model under the local optimisation, which is what makes few hypotheses enough at 30 % inliers.
__global__ void __launch_bounds__(1024) k_rs_select(const double* __restrict__ models, const double* __restrict__ cost,
                                                     const int* __restrict__ ninl, int n_slots, RsBest* __restrict__ cand,
                                                     const int* __restrict__ go, int* __restrict__ more, int k, int msize,
                                                     double log_1mc, double done_after) {
  if (go && !*go) return;
  __shared__ double sc[1024];
  __shared__ int si[1024];
  __shared__ RsBest merged[RS_TOP];
  __shared__ double prev_c;
  __shared__ int prev_i;
  // virtual slot index of an existing candidate j: -(RS_TOP - j) < 0, i.e. earlier arrivals win ties against this batch
  if (threadIdx.x == 0) prev_c = -1.0, prev_i = -1000000;
  __syncthreads();
  for (int round = 0; round < RS_TOP; ++round) {
    double bc = 1e300;
    int bi = 0x7fffffff;
    const double pc = prev_c;
    const int pi = prev_i;
    auto after_prev = [&](double c, int i) { return c > pc || (c == pc && i > pi); };
    auto better = [&](double c, int i) { return c < bc || (c == bc && i < bi); };
    for (int i = threadIdx.x; i < n_slots; i += 1024) {
      const double c = cost[i];
      if (c < 1e299 && after_prev(c, i) && better(c, i)) bc = c, bi = i;
    }
    if (threadIdx.x < RS_TOP && cand[threadIdx.x].valid) {
      const double c = cand[threadIdx.x].cost;
      const int i = (int)threadIdx.x - RS_TOP;
      if (after_prev(c, i) && better(c, i)) bc = c, bi = i;
    }
    sc[threadIdx.x] = bc, si[threadIdx.x] = bi;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        const double oc = sc[threadIdx.x + o];
        const int oi = si[threadIdx.x + o];
        if (oc < sc[threadIdx.x] || (oc == sc[threadIdx.x] && oi < si[threadIdx.x])) sc[threadIdx.x] = oc, si[threadIdx.x] = oi;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      RsBest& m = merged[round];
      if (si[0] == 0x7fffffff) {
        m.valid = 0, m.cost = 1e300, m.ninl = 0;
        prev_c = 1e300, prev_i = 0x7fffffff;
      } else {
        if (si[0] < 0) {
          m = cand[si[0] + RS_TOP];
        } else {
          for (int i = 0; i < 9; ++i) m.model[i] = models[(size_t)si[0] * 9 + i];
          m.cost = sc[0], m.ninl = ninl[si[0]], m.valid = 1;
        }
        prev_c = sc[0], prev_i = si[0];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x < RS_TOP) cand[threadIdx.x] = merged[threadIdx.x];
  if (threadIdx.x == 0 && more) {
    // standard RANSAC bound with the support of the best hypothesis so far: are `done_after` samples enough for the requested
    // confidence?  If not, the (already enqueued) extension stage runs; otherwise its kernels return at once.
    int need_more = 1;
    if (merged[0].valid) {
      const double w = (double)merged[0].ninl / (double)k;
      const double pw = pow(w, (double)msize);
      const double need = pw >= 1.0 ? 1.0 : (pw <= 0.0 ? 1e300 : log_1mc / log(1.0 - pw));
      need_more = need > done_after ? 1 : 0;
    }
    *more = need_more;
  }
}

// after the local optimisation: the refined candidate with the lowest cost (ties -> lower rank) becomes the result
__global__ void k_rs_pick(const RsBest* __restrict__ cand, RsBest* __restrict__ best) {
  if (threadIdx.x != 0) return;
  int b = -1;
  for (int j = 0; j < RS_TOP; ++j)
    if (cand[j].valid && (b < 0 || cand[j].cost < cand[b].cost)) b = j;
  if (b >= 0) *best = cand[b];
  else best->valid = 0, best->cost = 1e300, best->ninl = 0;
}

// ---- local optimisation: iterated normalised least-squares refit on the current inliers --------------------------
__device__ double block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0;
  for (int w = 0; w < RS_LO_THREADS / 32; ++w) t += sh[w];
  return t;
}

// Jacobi eigen-decomposition of a symmetric 9 x 9 matrix in SHARED memory by one warp, parallel (round-robin) ordering:
// each of the 9 rounds of a sweep applies FOUR rotations on disjoint index pairs at once - their angles come from lanes
// 0..3, the 4 x 9 two-element column updates of A and V and then the 4 x 9 row updates of A are spread over the lanes.
// Disjoint rotations commute, so a round equals the same four rotations applied one after the other.  A single thread
// walking the run-time indexed matrix in local memory (rmath::jacobi_eig<9>) is much slower.
__device__ void jacobi9_warp(double* A, double* V, int lane) {
  __shared__ double rc[4], rs[4];
  __shared__ int rp[4], rq[4];
  for (int i = lane; i < 81; i += 32) V[i] = (i / 9 == i % 9) ? 1.0 : 0.0;
  __syncwarp();
  for (int sweep = 0; sweep < 40; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = lane; i < 81; i += 32) {
      const double v = A[i] * A[i];
      if (i / 9 == i % 9) diag += v;
      else off += v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) off += __shfl_xor_sync(0xffffffffu, off, o), diag += __shfl_xor_sync(0xffffffffu, diag, o);
    if (0.5 * off <= 1e-26 * (diag + 1e-300)) break;
    for (int r = 0; r < 9; ++r) {  // circle method over 10 players, player 9 is a bye: pairs ((r + i) % 9, (r - i) % 9), i = 1..4
      if (lane < 4) {
        const int a = (r + lane + 1) % 9, b = (r + 9 - lane - 1) % 9;
        const int pp = a < b ? a : b, qq = a < b ? b : a;
        const double apq = A[pp * 9 + qq];
        double c = 1.0, sn = 0.0;
        if (fabs(apq) >= 1e-300) {
          const double theta = (A[qq * 9 + qq] - A[pp * 9 + pp]) / (2.0 * apq);
          const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
        }
        rc[lane] = c, rs[lane] = sn, rp[lane] = pp, rq[lane] = qq;
      }
      __syncwarp();
      for (int it = lane; it < 36; it += 32) {  // columns p, q of A and of V, row k
        const int i = it / 9, k = it - i * 9;
        const double c = rc[i], sn = rs[i];
        const int pp = rp[i], qq = rq[i];
        const double akp = A[k * 9 + pp], akq = A[k * 9 + qq];
        A[k * 9 + pp] = c * akp - sn * akq;
        A[k * 9 + qq] = sn * akp + c * akq;
        const double vkp = V[k * 9 + pp], vkq = V[k * 9 + qq];
        V[k * 9 + pp] = c * vkp - sn * vkq;
        V[k * 9 + qq] = sn * vkp + c * vkq;
      }
      __syncwarp();
      for (int it = lane; it < 36; it += 32) {  // rows p, q of A, column k
        const int i = it / 9, k = it - i * 9;
        const double c = rc[i], sn = rs[i];
        const int pp = rp[i], qq = rq[i];
        const double apk = A[pp * 9 + k], aqk = A[qq * 9 + k];
        A[pp * 9 + k] = c * apk - sn * aqk;
        A[qq * 9 + k] = sn * apk + c * aqk;
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(RS_LO_THREADS) k_rs_refine(const double* __restrict__ x1, const double* __restrict__ x2, int k,
                                                              double thr2, int mode, RsBest* __restrict__ cands) {
  RsBest* best = cands + blockIdx.x;  // one CTA per candidate
  __shared__ double sh[RS_LO_THREADS / 32];
  __shared__ double M[9], cand[9];
  __shared__ double mom[45];
  __shared__ double part[RS_LO_THREADS / 32][45];
  __shared__ double JA[81], JV[81];
  if (!best->valid) return;
  if (threadIdx.x < 9) M[threadIdx.x] = best->model[threadIdx.x];
  __syncthreads();
  double cur_cost = best->cost;
  const int min_pts = 8;
  for (int it = 0; it < RS_LO_ITERS; ++it) {
    // The support set of the first refits is taken with a WIDER threshold (4x, 2x the squared threshold): a hypothesis
    // from a slightly contaminated sample holds only part of the true inliers within thr, and a least-squares refit on
    // that part stays biased; acceptance is always judged by the MSAC cost at the real threshold.
    const double sel2 = thr2 * (it == 0 ? 4.0 : (it == 1 ? 2.0 : 1.0));
    // inlier flags of this thread's points under M, evaluated once per iteration (bit j <-> point threadIdx.x + j * T)
    unsigned long long flags = 0ull;
    double a[5] = {0, 0, 0, 0, 0};
    {
      int j = 0;
      for (int i = threadIdx.x; i < k; i += RS_LO_THREADS, ++j) {
        const double e = rs_err(mode, M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
        if (e < sel2) {
          if (j < 64) flags |= 1ull << j;
          a[0] += x1[2 * i], a[1] += x1[2 * i + 1], a[2] += x2[2 * i], a[3] += x2[2 * i + 1], a[4] += 1.0;
        }
      }
    }
    auto is_in = [&](int i, int j) {  // beyond 64 points per thread (k > 32768) fall back to re-evaluation
      return j < 64 ? ((flags >> j) & 1ull) != 0 : rs_err(mode, M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]) < sel2;
    };
    // centroids and mean distances of the inliers under M (Hartley normalisation)
    double cnt = block_sum(a[4], sh);
    if (cnt < min_pts) break;
    double c1x = block_sum(a[0], sh) / cnt, c1y = block_sum(a[1], sh) / cnt, c2x = block_sum(a[2], sh) / cnt,
           c2y = block_sum(a[3], sh) / cnt;
    double d1 = 0, d2 = 0;
    {
      int j = 0;
      for (int i = threadIdx.x; i < k; i += RS_LO_THREADS, ++j) {
        if (is_in(i, j)) {
          d1 += sqrt((x1[2 * i] - c1x) * (x1[2 * i] - c1x) + (x1[2 * i + 1] - c1y) * (x1[2 * i + 1] - c1y));
          d2 += sqrt((x2[2 * i] - c2x) * (x2[2 * i] - c2x) + (x2[2 * i + 1] - c2y) * (x2[2 * i + 1] - c2y));
        }
      }
    }
    d1 = block_sum(d1, sh), d2 = block_sum(d2, sh);
    if (d1 < 1e-12 || d2 < 1e-12) break;
    const double s1 = 1.4142135623730951 * cnt / d1, s2 = 1.4142135623730951 * cnt / d2;
    // upper triangle of sum q q^T
    double acc[45];
#pragma unroll
    for (int i = 0; i < 45; ++i) acc[i] = 0;
    {
      int j = 0;
      for (int i = threadIdx.x; i < k; i += RS_LO_THREADS, ++j) {
        if (is_in(i, j)) {
          double ax = (x1[2 * i] - c1x) * s1, ay = (x1[2 * i + 1] - c1y) * s1;
          double bx = (x2[2 * i] - c2x) * s2, by = (x2[2 * i + 1] - c2y) * s2;
          double q[9] = {bx * ax, bx * ay, bx, by * ax, by * ay, by, ax, ay, 1.0};
          int t = 0;
#pragma unroll
          for (int r = 0; r < 9; ++r)
#pragma unroll
            for (int c = r; c < 9; ++c) acc[t++] += q[r] * q[c];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 45; ++i) {
      double v = acc[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < 45) {
      double v = 0;
      for (int w = 0; w < RS_LO_THREADS / 32; ++w) v += part[w][threadIdx.x];
      mom[threadIdx.x] = v;
    }
    __syncthreads();
    if (threadIdx.x < 32) {  // warp 0: smallest eigenvector of the moment matrix -> candidate model
      if (threadIdx.x == 0) {
        int t = 0;
        for (int r = 0; r < 9; ++r)
          for (int c = r; c < 9; ++c) JA[r * 9 + c] = JA[c * 9 + r] = mom[t++];
      }
      __syncwarp();
      jacobi9_warp(JA, JV, threadIdx.x);
      __syncwarp();
      if (threadIdx.x == 0) {
        int kk = 0;
        for (int i = 1; i < 9; ++i)
          if (JA[i * 9 + i] < JA[kk * 9 + kk]) kk = i;
        double Fn[9];
        for (int i = 0; i < 9; ++i) Fn[i] = JV[i * 9 + kk];
        double T1[9] = {s1, 0, -s1 * c1x, 0, s1, -s1 * c1y, 0, 0, 1}, T2t[9] = {s2, 0, 0, 0, s2, 0, -s2 * c2x, -s2 * c2y, 1};
        double tmp[9], F[9];
        mat3_mul(T2t, Fn, tmp);
        mat3_mul(tmp, T1, F);
        if (mode == 0) enforce_essential(F);
        else enforce_rank2(F);
        double n = 0;
        for (int i = 0; i < 9; ++i) n += F[i] * F[i];
        n = sqrt(n);
        for (int i = 0; i < 9; ++i) cand[i] = n > 1e-300 ? F[i] / n : 0.0;
      }
    }
    __syncthreads();
    double c = 0, ni = 0;
    for (int i = threadIdx.x; i < k; i += RS_LO_THREADS) {
      double e = rs_err(mode, cand, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
      c += e < thr2 ? e : thr2;
      ni += e < thr2 ? 1.0 : 0.0;
    }
    c = block_sum(c, sh);
    ni = block_sum(ni, sh);
    if (!(c < cur_cost)) {  // no improvement: keep M (the wide-threshold rounds get their narrower successors first)
      if (it >= 2) break;
      continue;
    }
    cur_cost = c;
    __syncthreads();
    if (threadIdx.x < 9) M[threadIdx.x] = cand[threadIdx.x];
    if (threadIdx.x == 0) best->cost = c, best->ninl = (int)ni;
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x < 9) best->model[threadIdx.x] = M[threadIdx.x];
}

__global__ void __launch_bounds__(256) k_rs_mask(const double* __restrict__ x1, const double* __restrict__ x2, int k, double thr2,
                                                  int mode, const RsBest* __restrict__ best, uint8_t* __restrict__ mask,
                                                  int* __restrict__ count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool in = false;
  if (i < k && best->valid) in = rs_err(mode, best->model, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]) < thr2;
  if (i < k) mask[i] = in ? 1 : 0;
  unsigned m = __ballot_sync(0xffffffffu, in);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, __popc(m));
}

// ---- pose recovery (cv2.recoverPose semantics): one correspondence per thread, integer votes, last CTA decides ------
constexpr int RS_POSE_THREADS = 128;
__global__ void __launch_bounds__(RS_POSE_THREADS) k_rs_pose(const double* __restrict__ E, const double* __restrict__ x1,
                                                              const double* __restrict__ x2, const uint8_t* __restrict__ mask, int k,
                                                              int* __restrict__ gvotes /*[4] votes + [1] CTA counter, zero on entry*/,
                                                              double* __restrict__ out /*R[9], t[3], good*/,
                                                              double* __restrict__ cands /*R1[9], R2[9], t[3], winner; tests only*/) {
  __shared__ double R1[9], R2[9], t[3];
  __shared__ int votes[4];
  __shared__ int is_last;
  if (threadIdx.x == 0) {
    decompose_E(E, R1, R2, t);
    votes[0] = votes[1] = votes[2] = votes[3] = 0;
  }
  __syncthreads();
  int v[4] = {0, 0, 0, 0};
  const int i = blockIdx.x * RS_POSE_THREADS + threadIdx.x;
  if (i < k && (!mask || mask[i])) {
    const double tn[3] = {-t[0], -t[1], -t[2]};
    v[0] = cheirality_ok(R1, t, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1], 50.0);
    v[1] = cheirality_ok(R2, t, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1], 50.0);
    v[2] = cheirality_ok(R1, tn, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1], 50.0);
    v[3] = cheirality_ok(R2, tn, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1], 50.0);
  }
  for (int c = 0; c < 4; ++c) {
    int s = v[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(&votes[c], s);  // integer: order independent
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int c = 0; c < 4; ++c)
      if (votes[c]) atomicAdd(&gvotes[c], votes[c]);
    __threadfence();
    is_last = atomicAdd(&gvotes[4], 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    __threadfence();
    int tot[4];
    for (int c = 0; c < 4; ++c) tot[c] = *reinterpret_cast<volatile int*>(&gvotes[c]);
    int b = 0;
    for (int c = 1; c < 4; ++c)
      if (tot[c] > tot[b]) b = c;  // ties -> first, in cv2's order (R1,t), (R2,t), (R1,-t), (R2,-t)
    const double* R = (b & 1) ? R2 : R1;
    double sg = (b & 2) ? -1.0 : 1.0;
    for (int j = 0; j < 9; ++j) out[j] = R[j];
    for (int j = 0; j < 3; ++j) out[9 + j] = sg * t[j];
    out[12] = (double)tot[b];
    if (cands) {
      for (int j = 0; j < 9; ++j) cands[j] = R1[j], cands[9 + j] = R2[j];
      for (int j = 0; j < 3; ++j) cands[18 + j] = t[j];
      cands[21] = (double)b;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------

// gather matched keypoints and calibrate them with a distortion-free pinhole model (utils/features.py:41-51 for
// Cal3Bundler with k1 = k2 = 0): x = (u - u0) / f, in double.  f = 1, u0 = v0 = 0 leaves pixels (F path).
__global__ void __launch_bounds__(256) k_rs_gather(const float* __restrict__ kp1, const float* __restrict__ kp2,
                                                    const long long* __restrict__ matches, int k, double f1, double u1,
                                                    double v1, double f2, double u2, double v2, double* __restrict__ x1,
                                                    double* __restrict__ x2) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  long long a = matches[2 * i], b = matches[2 * i + 1];
  x1[2 * i] = ((double)kp1[2 * a] - u1) / f1;
  x1[2 * i + 1] = ((double)kp1[2 * a + 1] - v1) / f1;
  x2[2 * i] = ((double)kp2[2 * b] - u2) / f2;
  x2[2 * i + 1] = ((double)kp2[2 * b + 1] - v2) / f2;
}

// x1 / x2 come either from host arrays (hx != null: uploaded here) or are already in s->x1 / s->x2 (device path).
// out_mask: host pointer when mask_is_device == 0, device pointer otherwise.  tr (tests only, nullptr in production) sets
// the batch size and receives the intermediate state; it adds copies and synchronisations but no launches.
static int rs_run(b2_context* ctx, const double* hx1, const double* hx2, int k, const b2_ransac_params* prm, int mode,
                  double* out_model, uint8_t* out_mask, int* out_ninl, double* out_R, double* out_t,
                  cudaStream_t st = nullptr, int mask_is_device = 0, b2_ransac_trace* tr = nullptr) {
  if (!ctx->rs) ctx->rs = new RansacState();
  RansacState* s = ctx->rs;
  if (!st) st = ctx->stream;
  const int m = mode == 0 ? 5 : 8;
  if (tr) tr->batches = 0, tr->ext_go = -1, tr->records = 0;
  *out_ninl = 0;
  if (out_mask && !mask_is_device) memset(out_mask, 0, (size_t)k);
  if (out_mask && mask_is_device && k > 0) B2_CUDA(ctx, cudaMemsetAsync(out_mask, 0, (size_t)k, st));
  if (k < m) return 1;
  const int hard_cap = mode == 0 ? 65536 : 262144;
  const int max_iters = prm->max_iters < 1 ? 1 : (prm->max_iters > hard_cap ? hard_cap : prm->max_iters);
  const int batch = tr ? tr->batch : RS_BATCH;
  const double thr2 = prm->threshold * prm->threshold;
  B2_CUDA(ctx, s->x1.ensure((size_t)k * 16));
  B2_CUDA(ctx, s->x2.ensure((size_t)k * 16));
  B2_CUDA(ctx, s->models.ensure((size_t)RS_BATCH * RS_MAX_SOL * 9 * 8));
  B2_CUDA(ctx, s->nsol.ensure((size_t)RS_BATCH * 4));
  B2_CUDA(ctx, s->cost.ensure((size_t)RS_BATCH * RS_MAX_SOL * 8));
  B2_CUDA(ctx, s->ninl.ensure((size_t)RS_BATCH * RS_MAX_SOL * 4));
  B2_CUDA(ctx, s->best.ensure(sizeof(RsBest) * (1 + RS_TOP) + 16));  // [0] result, then the counter, then the RS_TOP candidates
  B2_CUDA(ctx, s->mask.ensure((size_t)k + 16));
  // [0,13) R, t, votes of the winner | [16,25) E (recover_pose) | [32,36) int votes[4] + counter | [36,58) R1, R2, t, winner
  B2_CUDA(ctx, s->pose.ensure(64 * 8));
  B2_CUDA(ctx, s->hbuf.ensure(sizeof(RsBest) + 16 * 8 + 64));
  if (hx1) {
    B2_CUDA(ctx, cudaMemcpyAsync(s->x1.p, hx1, (size_t)k * 16, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->x2.p, hx2, (size_t)k * 16, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(ctx, cudaMemsetAsync(s->best.p, 0, sizeof(RsBest) * (1 + RS_TOP) + 16, st));
  RsBest* dbest = s->best.as<RsBest>();
  int* dcount = reinterpret_cast<int*>(s->best.as<char>() + sizeof(RsBest));
  RsBest* dcand = reinterpret_cast<RsBest*>(s->best.as<char>() + sizeof(RsBest) + 16);
  RsBest* hbest = s->hbuf.as<RsBest>();
  const double *x1 = s->x1.as<double>(), *x2 = s->x2.as<double>();
  // trace record of one k_rs_select launch over n samples (more_written: it wrote the confidence flag)
  auto record = [&](int n, bool more_written) -> int {
    if (tr->records >= tr->max_records) return B2_OK;
    const int r = tr->records++;
    const size_t ns = (size_t)tr->batch;
    const auto d2h = cudaMemcpyDeviceToHost;
    if (tr->nsol) B2_CUDA(ctx, cudaMemcpyAsync(tr->nsol + r * ns, s->nsol.p, (size_t)n * 4, d2h, st));
    if (tr->models)
      B2_CUDA(ctx, cudaMemcpyAsync(tr->models + r * ns * RS_MAX_SOL * 9, s->models.p, (size_t)n * RS_MAX_SOL * 72, d2h, st));
    if (tr->cost) B2_CUDA(ctx, cudaMemcpyAsync(tr->cost + r * ns * RS_MAX_SOL, s->cost.p, (size_t)n * RS_MAX_SOL * 8, d2h, st));
    if (tr->ninl) B2_CUDA(ctx, cudaMemcpyAsync(tr->ninl + r * ns * RS_MAX_SOL, s->ninl.p, (size_t)n * RS_MAX_SOL * 4, d2h, st));
    if (tr->selected) B2_CUDA(ctx, cudaMemcpyAsync(tr->selected + (size_t)r * RS_TOP, dcand, sizeof(RsBest) * RS_TOP, d2h, st));
    if (tr->more) {
      if (more_written) B2_CUDA(ctx, cudaMemcpyAsync(tr->more + r, dcount + 1, 4, d2h, st));
      else tr->more[r] = -1;
    }
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    return B2_OK;
  };
  int done = 0;
  while (done < max_iters) {
    const int n = (max_iters - done) < batch ? (max_iters - done) : batch;
    if (mode == 0)
      B2_LAUNCH(ctx, k_rs_hyp_E, cdiv(n, 64), 64, 0, st, x1, x2, k, (unsigned long long)prm->seed, done, n,
                s->models.as<double>(), s->nsol.as<int>(), (const int*)nullptr);
    else
      B2_LAUNCH(ctx, k_rs_hyp_F, cdiv(n, 64), 64, 0, st, x1, x2, k, (unsigned long long)prm->seed, done, n,
                s->models.as<double>(), s->nsol.as<int>());
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_rs_score, n * RS_MAX_SOL, RS_SCORE_THREADS, 0, st, s->models.as<double>(), s->nsol.as<int>(), x1, x2, k,
              thr2, mode, s->cost.as<double>(), s->ninl.as<int>(), (const int*)nullptr);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_rs_select, 1, 1024, 0, st, s->models.as<double>(), s->cost.as<double>(), s->ninl.as<int>(),
              n * RS_MAX_SOL, dcand, (const int*)nullptr, dcount + 1, k, m, log(1.0 - prm->confidence), (double)(done + n));
    B2_CHECK_LAUNCH(ctx);
    if (tr) {
      ++tr->batches;
      if (int rc = record(n, true)) return rc;
    }
    done += n;
    if (done >= max_iters) break;
    // adaptive termination (standard RANSAC bound) between batches
    B2_CUDA(ctx, cudaMemcpyAsync(hbest, dcand, sizeof(RsBest), cudaMemcpyDeviceToHost, st));  // the best unrefined candidate
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    if (hbest->valid) {
      double w = (double)hbest->ninl / k, pw = pow(w, m);
      double need = pw >= 1.0 ? 1.0 : (pw <= 0 ? 1e300 : log(1.0 - prm->confidence) / log(1.0 - pw));
      if ((double)done >= need) break;
    }
  }
  if (mode == 0 && done >= max_iters && max_iters <= 4096) {
    // Extension stage (E only): cv2's budget of `max_iters` samples leaves a 30 %-inlier pair without a single uncontaminated
    // 5-sample one time in eleven; USAC survives that through its graph-cut local optimisation, a plain RANSAC does not.  The
    // hypothesis kernel is latency-bound, so 4x more samples cost about as much as the first batch; they only run when the
    // confidence bound of the best model so far says `max_iters` were not enough (flag written by k_rs_select on the device).
    const int n2 = 4 * max_iters < batch ? 4 * max_iters : batch;
    const int* go = dcount + 1;
    B2_LAUNCH(ctx, k_rs_hyp_E, cdiv(n2, 64), 64, 0, st, x1, x2, k, (unsigned long long)prm->seed, done, n2, s->models.as<double>(),
              s->nsol.as<int>(), go);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_rs_score, n2 * RS_MAX_SOL, RS_SCORE_THREADS, 0, st, s->models.as<double>(), s->nsol.as<int>(), x1, x2, k, thr2, mode,
              s->cost.as<double>(), s->ninl.as<int>(), go);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_rs_select, 1, 1024, 0, st, s->models.as<double>(), s->cost.as<double>(), s->ninl.as<int>(), n2 * RS_MAX_SOL, dcand, go,
              (int*)nullptr, k, m, 0.0, 0.0);
    B2_CHECK_LAUNCH(ctx);
    if (tr) {  // the extension's buffers are only worth recording when its kernels ran
      B2_CUDA(ctx, cudaMemcpyAsync(&tr->ext_go, go, 4, cudaMemcpyDeviceToHost, st));
      B2_CUDA(ctx, cudaStreamSynchronize(st));
      if (tr->ext_go)
        if (int rc = record(n2, false)) return rc;
    }
  }
  if (tr) B2_CUDA(ctx, cudaMemcpyAsync(tr->prerefine, dcand, sizeof(RsBest) * RS_TOP, cudaMemcpyDeviceToHost, st));
  B2_LAUNCH(ctx, k_rs_refine, RS_TOP, RS_LO_THREADS, 0, st, x1, x2, k, thr2, mode, dcand);
  B2_CHECK_LAUNCH(ctx);
  if (tr) B2_CUDA(ctx, cudaMemcpyAsync(tr->refined, dcand, sizeof(RsBest) * RS_TOP, cudaMemcpyDeviceToHost, st));
  B2_LAUNCH(ctx, k_rs_pick, 1, 32, 0, st, dcand, dbest);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_rs_mask, cdiv(k, 256), 256, 0, st, x1, x2, k, thr2, mode, dbest, s->mask.as<uint8_t>(), dcount);
  B2_CHECK_LAUNCH(ctx);
  const bool want_pose = mode == 0 && out_R && out_t;
  int* gvotes = reinterpret_cast<int*>(s->pose.as<double>() + 32);
  double* pose_cands = tr ? s->pose.as<double>() + 36 : nullptr;
  if (want_pose) {
    B2_CUDA(ctx, cudaMemsetAsync(gvotes, 0, 8 * sizeof(int), st));
    B2_LAUNCH(ctx, k_rs_pose, cdiv(k, RS_POSE_THREADS), RS_POSE_THREADS, 0, st, dbest->model, x1, x2, s->mask.as<uint8_t>(), k, gvotes,
              s->pose.as<double>(), pose_cands);
    B2_CHECK_LAUNCH(ctx);
  }
  if (tr) {
    B2_CUDA(ctx, cudaMemcpyAsync(&tr->pick, dbest, sizeof(RsBest), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(&tr->mask_count, dcount, 4, cudaMemcpyDeviceToHost, st));
    if (want_pose) {
      double c[22];
      B2_CUDA(ctx, cudaMemcpyAsync(tr->votes, gvotes, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
      B2_CUDA(ctx, cudaMemcpyAsync(c, pose_cands, sizeof(c), cudaMemcpyDeviceToHost, st));
      B2_CUDA(ctx, cudaStreamSynchronize(st));
      memcpy(tr->pose_cands, c, 21 * 8);
      tr->winner = (int)c[21];
    }
  }
  char* hb = s->hbuf.as<char>();
  B2_CUDA(ctx, cudaMemcpyAsync(hb, dbest, sizeof(RsBest) + 16, cudaMemcpyDeviceToHost, st));
  if (want_pose) B2_CUDA(ctx, cudaMemcpyAsync(hb + sizeof(RsBest) + 16, s->pose.p, 13 * 8, cudaMemcpyDeviceToHost, st));
  if (out_mask)
    B2_CUDA(ctx, cudaMemcpyAsync(out_mask, s->mask.p, (size_t)k, mask_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (!hbest->valid) {
    if (out_mask && !mask_is_device) memset(out_mask, 0, (size_t)k);
    return 1;
  }
  memcpy(out_model, hbest->model, 9 * 8);
  *out_ninl = *reinterpret_cast<int*>(hb + sizeof(RsBest));
  if (want_pose) {
    const double* p = reinterpret_cast<const double*>(hb + sizeof(RsBest) + 16);
    memcpy(out_R, p, 9 * 8);
    memcpy(out_t, p + 9, 3 * 8);
  }
  return B2_OK;
}

extern "C" int b2_ransac_essential_host(b2_context* ctx, const double* x1, const double* x2, int k,
                                        const b2_ransac_params* params, double* out_model, uint8_t* out_mask,
                                        int* out_num_inliers, double* out_R, double* out_t) {
  if (!ctx || !x1 || !x2 || !params || !out_model || !out_num_inliers || k < 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return rs_run(ctx, x1, x2, k, params, 0, out_model, out_mask, out_num_inliers, out_R, out_t);
}

extern "C" int b2_ransac_fundamental_host(b2_context* ctx, const double* x1, const double* x2, int k,
                                          const b2_ransac_params* params, double* out_model, uint8_t* out_mask,
                                          int* out_num_inliers) {
  if (!ctx || !x1 || !x2 || !params || !out_model || !out_num_inliers || k < 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return rs_run(ctx, x1, x2, k, params, 1, out_model, out_mask, out_num_inliers, nullptr, nullptr);
}

extern "C" int b2_ransac_essential_dev(b2_context* ctx, const float* kp1, const float* kp2, const int64_t* matches, int k,
                                       const double* cal1, const double* cal2, const b2_ransac_params* params,
                                       double* out_model, uint8_t* out_mask_dev, int* out_num_inliers, double* out_R,
                                       double* out_t, void* stream) {
  if (!ctx || !params || !out_model || !out_num_inliers || !cal1 || !cal2 || k < 0) return B2_ERR_ARG;
  if (k > 0 && (!kp1 || !kp2 || !matches)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->rs) ctx->rs = new RansacState();
  RansacState* s = ctx->rs;
  cudaStream_t st = (cudaStream_t)stream;
  if (k > 0) {
    B2_CUDA(ctx, s->x1.ensure((size_t)k * 16));
    B2_CUDA(ctx, s->x2.ensure((size_t)k * 16));
    B2_LAUNCH(ctx, k_rs_gather, cdiv(k, 256), 256, 0, st, kp1, kp2, (const long long*)matches, k, cal1[0], cal1[1], cal1[2],
              cal2[0], cal2[1], cal2[2], s->x1.as<double>(), s->x2.as<double>());
    B2_CHECK_LAUNCH(ctx);
  }
  // rs_run uses the legacy stream when `stream` is NULL; the context stream otherwise stays unused here
  return rs_run(ctx, nullptr, nullptr, k, params, 0, out_model, out_mask_dev, out_num_inliers, out_R, out_t,
                st ? st : cudaStreamLegacy, 1);
}

// out_cands / out_votes / out_winner: tests only (nullptr from b2_recover_pose_host)
static int recover_pose(b2_context* ctx, const double* E, const double* x1, const double* x2, int k, double* out_R, double* out_t,
                        int* out_num_good, double* out_cands, int* out_votes, int* out_winner) {
  if (!ctx || !E || !out_R || !out_t || k < 0 || (k > 0 && (!x1 || !x2))) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->rs) ctx->rs = new RansacState();
  RansacState* s = ctx->rs;
  cudaStream_t st = ctx->stream;
  B2_CUDA(ctx, s->x1.ensure((size_t)(k + 1) * 16));
  B2_CUDA(ctx, s->x2.ensure((size_t)(k + 1) * 16));
  B2_CUDA(ctx, s->pose.ensure(64 * 8));
  B2_CUDA(ctx, s->hbuf.ensure(sizeof(RsBest) + 16 * 8 + 64));
  if (k > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(s->x1.p, x1, (size_t)k * 16, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->x2.p, x2, (size_t)k * 16, cudaMemcpyHostToDevice, st));
  }
  double* dE = s->pose.as<double>() + 16;
  B2_CUDA(ctx, cudaMemcpyAsync(dE, E, 9 * 8, cudaMemcpyHostToDevice, st));
  {
    int* gvotes = reinterpret_cast<int*>(s->pose.as<double>() + 32);
    B2_CUDA(ctx, cudaMemsetAsync(gvotes, 0, 8 * sizeof(int), st));
    B2_LAUNCH(ctx, k_rs_pose, k > 0 ? cdiv(k, RS_POSE_THREADS) : 1, RS_POSE_THREADS, 0, st, dE, s->x1.as<double>(), s->x2.as<double>(),
              (const uint8_t*)nullptr, k, gvotes, s->pose.as<double>(), out_cands ? s->pose.as<double>() + 36 : nullptr);
  }
  B2_CHECK_LAUNCH(ctx);
  double* h = s->hbuf.as<double>();
  B2_CUDA(ctx, cudaMemcpyAsync(h, s->pose.p, 13 * 8, cudaMemcpyDeviceToHost, st));
  if (out_cands) {
    double c[22];
    B2_CUDA(ctx, cudaMemcpyAsync(c, s->pose.as<double>() + 36, sizeof(c), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(out_votes, s->pose.as<double>() + 32, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    memcpy(out_cands, c, 21 * 8);
    *out_winner = (int)c[21];
  }
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(out_R, h, 9 * 8);
  memcpy(out_t, h + 9, 3 * 8);
  if (out_num_good) *out_num_good = (int)h[12];
  return B2_OK;
}

extern "C" int b2_recover_pose_host(b2_context* ctx, const double* E, const double* x1, const double* x2, int k,
                                    double* out_R, double* out_t, int* out_num_good) {
  return recover_pose(ctx, E, x1, x2, k, out_R, out_t, out_num_good, nullptr, nullptr, nullptr);
}

// ---- test-only entry points: the same kernels and host logic, with their intermediate state --------------------------

extern "C" int b2_debug_recover_pose_host(b2_context* ctx, const double* E, const double* x1, const double* x2, int k,
                                          double* out_cands, int* out_votes, int* out_winner, double* out_R, double* out_t,
                                          int* out_num_good) {
  if (!out_cands || !out_votes || !out_winner) return B2_ERR_ARG;
  return recover_pose(ctx, E, x1, x2, k, out_R, out_t, out_num_good, out_cands, out_votes, out_winner);
}

extern "C" int b2_debug_ransac_trace_host(b2_context* ctx, int mode, const double* x1, const double* x2, int k,
                                          const b2_ransac_params* params, b2_ransac_trace* trace, double* out_model,
                                          uint8_t* out_mask, int* out_num_inliers, double* out_R, double* out_t) {
  if (!ctx || !x1 || !x2 || !params || !trace || !out_model || !out_num_inliers || k < 0 || (mode != 0 && mode != 1) ||
      trace->batch < 1 || trace->batch > RS_BATCH || trace->max_records < 0)
    return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return rs_run(ctx, x1, x2, k, params, mode, out_model, out_mask, out_num_inliers, mode == 0 ? out_R : nullptr,
                mode == 0 ? out_t : nullptr, nullptr, 0, trace);
}
