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
//
// Every kernel takes a TABLE of problems (RsProb, device memory) and works on problem blockIdx.y, so one launch of a stage
// covers every live pair of a call; problems never interact, and each runs the arithmetic, reduction order and tie rules
// it would run alone, so a pair's result does not depend on what it is batched with.  The per-pair entry points are the
// same code with a table of one.  Sampling rounds are enqueued for all live problems at once: the host rewrites the round
// fields (first sample, count, flags) of the records that still run and uploads that compacted table; k_rs_select writes one
// "confidence not reached" flag per problem, the E extension stage is gated by it on the device, and where a problem still
// has budget left the host reads the whole flag array once per round and drops the problems that are done.
//
// Workspace: a problem's slices of models / nsol / cost / ninl hold its largest round (844 B per sample: 3.4 MB for an E
// problem at 1000 + 4000 samples, 13.8 MB for an F round of 16 384), plus 32 B per match when the calibrated points are
// made here.  A call is cut into consecutive sub-batches whose slices fit the workspace budget (1 GiB unless
// b2_set_option "ransac_workspace_mb" says otherwise; a problem that alone exceeds it runs alone).
#include <string.h>

#include "common.cuh"
#include "ransac_math.cuh"
#include "ransac_prob.cuh"

using namespace rmath;

namespace {
constexpr int RS_MAX_SOL = 10;
constexpr int RS_SCORE_THREADS = 128;
constexpr int RS_LO_THREADS = 512;
constexpr int RS_LO_ITERS = 6;
constexpr int RS_TOP = 8;  // hypotheses handed to the local optimisation (the refined candidate with the lowest MSAC cost wins)
constexpr int RS_BATCH = 16384;  // hypotheses per launch (buffers are sized for it; a trace may ask for fewer)
}  // namespace

// what a call returns per problem, one D2H copy for the whole sub-batch
struct RsOut {
  RsBest best;
  int count, pad;
  double pose[13];
};
struct RsScratch {
  RsBest cand[RS_TOP];
  double E[9];  // b2_recover_pose_host's input
  double pose_cands[22];
  int gvotes[8];
};

struct RansacState {
  DevBuf x1, x2, models, nsol, cost, ninl, small, mask, tab;
  HostBuf hbuf;
};

void rs_destroy(b2_context* ctx) {
  delete ctx->rs;
  ctx->rs = nullptr;
}

// Copies a problem's record to shared memory, where the register-bound kernels read its fields at the point of use (as they
// would read kernel parameters) instead of holding them in registers from the first line on.
__device__ __forceinline__ void rs_load_prob(RsProb* sp, const RsProb* __restrict__ gp) {
  for (int i = threadIdx.x; i < (int)(sizeof(RsProb) / 8); i += blockDim.x)
    reinterpret_cast<unsigned long long*>(sp)[i] = reinterpret_cast<const unsigned long long*>(gp)[i];
  __syncthreads();
}

__device__ __forceinline__ double rs_err(int mode, const double* M, double a, double b, double c, double d) {
  return mode == 0 ? sampson_sq(M, a, b, c, d) : epiline_sq(M, a, b, c, d);
}

// ---- hypothesis generation -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) k_rs_hyp_E(const RsProb* __restrict__ tab, unsigned long long seed) {
  const RsProb& p = tab[blockIdx.y];
  if (p.go && !*p.go) return;  // extension stage not needed (decided on the device by k_rs_select)
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.n) return;
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  double* __restrict__ models = p.models;
  int idx[5];
  sample_distinct(seed, (unsigned long long)(p.sample0 + s), p.k, 5, idx);
  double a[5][2], b[5][2];
  for (int i = 0; i < 5; ++i) {
    a[i][0] = x1[2 * idx[i]], a[i][1] = x1[2 * idx[i] + 1];
    b[i][0] = x2[2 * idx[i]], b[i][1] = x2[2 * idx[i] + 1];
  }
  double sol[RS_MAX_SOL][9];
  int n = fivept_solve(a, b, sol);
  p.nsol[s] = n;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < 9; ++i) models[((size_t)s * RS_MAX_SOL + j) * 9 + i] = sol[j][i];
}

// normalised 8-point algorithm on one 8-sample (Hartley 1997): one F per sample
__global__ void __launch_bounds__(64) k_rs_hyp_F(const RsProb* __restrict__ tab, unsigned long long seed) {
  const RsProb& p = tab[blockIdx.y];
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.n) return;
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  int idx[8];
  sample_distinct(seed, (unsigned long long)(p.sample0 + s), p.k, 8, idx);
  double a[8][2], b[8][2];
  for (int i = 0; i < 8; ++i) {
    a[i][0] = x1[2 * idx[i]], a[i][1] = x1[2 * idx[i] + 1];
    b[i][0] = x2[2 * idx[i]], b[i][1] = x2[2 * idx[i] + 1];
  }
  const int n = eightpt_solve(a, b, p.models + (size_t)s * RS_MAX_SOL * 9);
  p.nsol[s] = n;
}

// ---- scoring: one CTA per model slot (the grid spans the largest round of the table) ---------------------------------
__global__ void __launch_bounds__(RS_SCORE_THREADS) k_rs_score(const RsProb* __restrict__ tab) {
  const RsProb& p = tab[blockIdx.y];
  if (p.go && !*p.go) return;
  const int slot = blockIdx.x, s = slot / RS_MAX_SOL, j = slot % RS_MAX_SOL;
  if (s >= p.n) return;
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  double* __restrict__ cost = p.cost;
  int* __restrict__ ninl = p.ninl;
  const int k = p.k, mode = p.mode;
  const double thr2 = p.thr2;
  if (j >= p.nsol[s]) {
    if (threadIdx.x == 0) cost[slot] = 1e300, ninl[slot] = 0;
    return;
  }
  __shared__ double M[9];
  __shared__ double wc[RS_SCORE_THREADS / 32];
  __shared__ int wn[RS_SCORE_THREADS / 32];
  if (threadIdx.x < 9) M[threadIdx.x] = p.models[(size_t)slot * 9 + threadIdx.x];
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
__global__ void __launch_bounds__(1024) k_rs_select(const RsProb* __restrict__ tab, double log_1mc) {
  const RsProb& p = tab[blockIdx.y];
  if (p.go && !*p.go) return;
  const double *__restrict__ models = p.models, *__restrict__ cost = p.cost;
  const int* __restrict__ ninl = p.ninl;
  RsBest* __restrict__ cand = p.cand;
  const int n_slots = p.n * RS_MAX_SOL;
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
  if (threadIdx.x == 0 && p.more) {
    // standard RANSAC bound with the support of the best hypothesis so far: are `done_after` samples enough for the requested
    // confidence?  If not, the (already enqueued) extension stage runs, or the host enqueues the problem's next round;
    // otherwise the extension's kernels return at once and the problem is left out of later rounds.
    int need_more = 1;
    if (merged[0].valid) {
      const double w = (double)merged[0].ninl / (double)p.k;
      const double pw = pow(w, p.mode == 0 ? 5.0 : 8.0);
      const double need = pw >= 1.0 ? 1.0 : (pw <= 0.0 ? 1e300 : log_1mc / log(1.0 - pw));
      need_more = need > p.done_after ? 1 : 0;
    }
    *p.more = need_more;
  }
}

// after the local optimisation: the refined candidate with the lowest cost (ties -> lower rank) becomes the result
__global__ void k_rs_pick(const RsProb* __restrict__ tab) {
  if (threadIdx.x != 0) return;
  const RsBest* __restrict__ cand = tab[blockIdx.y].cand;
  RsBest* __restrict__ best = tab[blockIdx.y].best;
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

__global__ void __launch_bounds__(RS_LO_THREADS) k_rs_refine(const RsProb* __restrict__ tab) {
  __shared__ RsProb p;
  rs_load_prob(&p, tab + blockIdx.y);
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  const int k = p.k, mode = p.mode;
  const double thr2 = p.thr2;
  RsBest* best = p.cand + blockIdx.x;  // one CTA per candidate
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

__global__ void __launch_bounds__(256) k_rs_mask(const RsProb* __restrict__ tab) {
  const RsProb& p = tab[blockIdx.y];
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  const RsBest* __restrict__ best = p.best;
  const int k = p.k;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool in = false;
  if (i < k && best->valid) in = rs_err(p.mode, best->model, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]) < p.thr2;
  if (i < k) p.mask[i] = in ? 1 : 0;
  unsigned m = __ballot_sync(0xffffffffu, in);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(p.count, __popc(m));
}

// ---- pose recovery (cv2.recoverPose semantics): one correspondence per thread, integer votes, last CTA decides ------
// The grid spans the largest problem of the table; a CTA past its problem's points casts no vote but is still counted, so
// "last" means the same for every problem.  A fundamental-matrix problem (pose_cal) first forms E = K2^T F K1 and calibrates
// its pixel coordinates with each side's (f, u0, v0), which is gtsfm/utils/verification.py:54-112.
__global__ void __launch_bounds__(RS_POSE_THREADS) k_rs_pose(const RsProb* __restrict__ tab) {
  __shared__ RsProb p;
  rs_load_prob(&p, tab + blockIdx.y);
  if (!p.pose_on) return;
  const double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  const uint8_t* __restrict__ mask = p.pose_mask;
  int* __restrict__ gvotes = p.gvotes;
  double *__restrict__ out = p.pose, *__restrict__ cands = p.pose_cands;
  const int k = p.k;
  __shared__ double R1[9], R2[9], t[3];
  __shared__ int votes[4];
  __shared__ int is_last;
  if (threadIdx.x == 0) {
    if (p.pose_cal) {
      const double K2t[9] = {p.c2[0], 0, 0, 0, p.c2[0], 0, p.c2[1], p.c2[2], 1};
      const double K1[9] = {p.c1[0], 0, p.c1[1], 0, p.c1[0], p.c1[2], 0, 0, 1};
      double F[9], tmp[9], Em[9];
      for (int j = 0; j < 9; ++j) F[j] = p.E[j];
      mat3_mul(K2t, F, tmp);
      mat3_mul(tmp, K1, Em);
      decompose_E(Em, R1, R2, t);
    } else {
      decompose_E(p.E, R1, R2, t);
    }
    votes[0] = votes[1] = votes[2] = votes[3] = 0;
  }
  __syncthreads();
  int v[4] = {0, 0, 0, 0};
  const int i = blockIdx.x * RS_POSE_THREADS + threadIdx.x;
  if (i < k && (!mask || mask[i])) {
    const double tn[3] = {-t[0], -t[1], -t[2]};
    double ax = x1[2 * i], ay = x1[2 * i + 1], bx = x2[2 * i], by = x2[2 * i + 1];
    if (p.pose_cal) {
      ax = (ax - p.c1[1]) / p.c1[0], ay = (ay - p.c1[2]) / p.c1[0];
      bx = (bx - p.c2[1]) / p.c2[0], by = (by - p.c2[2]) / p.c2[0];
    }
    v[0] = cheirality_ok(R1, t, ax, ay, bx, by, 50.0);
    v[1] = cheirality_ok(R2, t, ax, ay, bx, by, 50.0);
    v[2] = cheirality_ok(R1, tn, ax, ay, bx, by, 50.0);
    v[3] = cheirality_ok(R2, tn, ax, ay, bx, by, 50.0);
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
__global__ void __launch_bounds__(256) k_rs_gather(const RsProb* __restrict__ tab) {
  const RsProb& p = tab[blockIdx.y];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (!p.kp1 || i >= p.k) return;
  const float *__restrict__ kp1 = p.kp1, *__restrict__ kp2 = p.kp2;
  double *__restrict__ x1 = p.x1, *__restrict__ x2 = p.x2;
  const double f1 = p.g1[0], u1 = p.g1[1], v1 = p.g1[2], f2 = p.g2[0], u2 = p.g2[1], v2 = p.g2[2];
  long long a = p.matches[2 * i], b = p.matches[2 * i + 1];
  x1[2 * i] = ((double)kp1[2 * a] - u1) / f1;
  x1[2 * i + 1] = ((double)kp1[2 * a + 1] - v1) / f1;
  x2[2 * i] = ((double)kp2[2 * b] - u2) / f2;
  x2[2 * i + 1] = ((double)kp2[2 * b + 1] - v2) / f2;
}

// One problem as the host entry points describe it.  Points come from host arrays (hx: uploaded here), from device arrays
// (dx: used where they are) or from keypoints + match rows (k_rs_gather); the mask goes to a device buffer (dmask), to a
// host one (hmask) or nowhere.
struct RsJob {
  const float *kp1 = nullptr, *kp2 = nullptr;
  const int64_t* matches = nullptr;
  const double *dx1 = nullptr, *dx2 = nullptr, *hx1 = nullptr, *hx2 = nullptr;
  int k = 0, mode = 0, max_iters = 0;
  double threshold = 0;
  double cal1[3] = {1, 0, 0}, cal2[3] = {1, 0, 0};
  uint8_t *dmask = nullptr, *hmask = nullptr;
  bool pose = false;
};

static int rs_clamp_iters(int mode, int max_iters) {
  const int hard_cap = mode == 0 ? 65536 : 262144;
  return max_iters < 1 ? 1 : (max_iters > hard_cap ? hard_cap : max_iters);
}
// samples the largest round of a problem draws: a sampling batch, or the E extension stage
static int rs_round_cap(int mode, int max_iters, int batch) {
  const int mi = rs_clamp_iters(mode, max_iters);
  const int main_n = mi < batch ? mi : batch;
  const int ext_n = (mode == 0 && mi <= 4096) ? (4 * mi < batch ? 4 * mi : batch) : 0;
  return main_n > ext_n ? main_n : ext_n;
}
constexpr size_t RS_SAMPLE_BYTES = RS_MAX_SOL * (72 + 8 + 4) + 4;  // models, cost, ninl of ten slots and nsol
constexpr size_t RS_FIXED_BYTES = sizeof(RsOut) + sizeof(RsScratch) + 4 + 3 * sizeof(RsProb);
// workspace bytes of one problem: its sample slices, its points and mask unless the caller's device arrays are used
static size_t rs_job_bytes(int k, int mode, int max_iters, bool own_x, bool own_mask, int batch = RS_BATCH) {
  if (k < (mode == 0 ? 5 : 8)) return RS_FIXED_BYTES;
  return RS_FIXED_BYTES + (size_t)rs_round_cap(mode, max_iters, batch) * RS_SAMPLE_BYTES + (own_x ? (size_t)k * 32 : 0) +
         (own_mask ? (size_t)k : 0);
}
// Consecutive sub-batches under `budget` bytes: first[i] is the first problem of sub-batch i, first[count] = n.  A
// problem larger than the budget gets a sub-batch of its own.
static int rs_plan(const size_t* bytes, int n, size_t budget, int* first) {
  int count = 0;
  size_t used = 0;
  for (int i = 0; i < n; ++i) {
    if (i == 0 || used + bytes[i] > budget) first[count++] = i, used = 0;
    used += bytes[i];
  }
  first[count] = n;
  return count;
}

#define RS_SYNC(ctx, st)                            \
  do {                                              \
    B2_CUDA(ctx, cudaStreamSynchronize(st));        \
    (ctx)->rs_syncs++;                              \
  } while (0)

// One sub-batch: every stage launched once for all its problems.  tr (tests only, nullptr in production, one problem) sets
// the round size and receives the intermediate state; it adds copies and synchronisations but no launches.
static int rs_run_sub(b2_context* ctx, const RsJob* jobs, int n, double confidence, uint64_t seed, b2_ransac_result* res,
                      cudaStream_t st, b2_ransac_trace* tr) {
  RansacState* s = ctx->rs;
  const int batch = tr ? tr->batch : RS_BATCH;
  if (tr) tr->batches = 0, tr->ext_go = -1, tr->records = 0;
  // live problems, essential ones first (the two hypothesis kernels each take a contiguous part of the table)
  std::vector<int> live;
  for (int mode = 0; mode < 2; ++mode)
    for (int i = 0; i < n; ++i)
      if (jobs[i].mode == mode && jobs[i].k >= (mode == 0 ? 5 : 8)) live.push_back(i);
  for (int i = 0; i < n; ++i) {
    memset(&res[i], 0, sizeof(res[i]));
    res[i].status = 1;
    const RsJob& j = jobs[i];
    if (j.k >= (j.mode == 0 ? 5 : 8) || j.k == 0) continue;
    if (j.hmask) memset(j.hmask, 0, (size_t)j.k);
    if (j.dmask) B2_CUDA(ctx, cudaMemsetAsync(j.dmask, 0, (size_t)j.k, st));
  }
  const int L = (int)live.size();
  if (L == 0) return B2_OK;

  size_t n_smp = 0, n_x = 0, n_mask = 0;
  for (int i : live) {
    const RsJob& j = jobs[i];
    n_smp += (size_t)rs_round_cap(j.mode, j.max_iters, batch);
    if (!j.dx1) n_x += (size_t)j.k;
    if (!j.dmask) n_mask += (size_t)j.k;
  }
  const size_t small_bytes = (size_t)L * (sizeof(RsOut) + sizeof(RsScratch) + 4);
  B2_CUDA(ctx, s->x1.ensure(n_x * 16 + 16));
  B2_CUDA(ctx, s->x2.ensure(n_x * 16 + 16));
  B2_CUDA(ctx, s->models.ensure(n_smp * RS_MAX_SOL * 72));
  B2_CUDA(ctx, s->nsol.ensure(n_smp * 4));
  B2_CUDA(ctx, s->cost.ensure(n_smp * RS_MAX_SOL * 8));
  B2_CUDA(ctx, s->ninl.ensure(n_smp * RS_MAX_SOL * 4));
  B2_CUDA(ctx, s->mask.ensure(n_mask + 16));
  B2_CUDA(ctx, s->small.ensure(small_bytes));
  B2_CUDA(ctx, s->tab.ensure(3 * (size_t)L * sizeof(RsProb)));
  // pinned: three tables (all problems | this round | the extension round), the results, the flags
  B2_CUDA(ctx, s->hbuf.ensure((size_t)L * (3 * sizeof(RsProb) + sizeof(RsOut) + 4)));
  RsProb* htab = s->hbuf.as<RsProb>();
  RsOut* hout = reinterpret_cast<RsOut*>(htab + 3 * (size_t)L);
  int* hflags = reinterpret_cast<int*>(hout + L);
  RsProb* dtab = s->tab.as<RsProb>();
  RsOut* dout = s->small.as<RsOut>();
  RsScratch* dscr = reinterpret_cast<RsScratch*>(dout + L);
  int* dflags = reinterpret_cast<int*>(dscr + L);
  B2_CUDA(ctx, cudaMemsetAsync(s->small.p, 0, small_bytes, st));

  int max_k = 0;
  bool any_gather = false, any_pose = false;
  {
    size_t o_smp = 0, o_x = 0, o_mask = 0;
    for (int t = 0; t < L; ++t) {
      const RsJob& j = jobs[live[t]];
      RsProb& p = htab[t];
      memset(&p, 0, sizeof(p));
      p.k = j.k, p.mode = j.mode, p.thr2 = j.threshold * j.threshold;
      if (j.dx1) {
        p.x1 = const_cast<double*>(j.dx1), p.x2 = const_cast<double*>(j.dx2);
      } else {
        p.x1 = s->x1.as<double>() + 2 * o_x, p.x2 = s->x2.as<double>() + 2 * o_x;
        o_x += (size_t)j.k;
        if (j.hx1) {
          B2_CUDA(ctx, cudaMemcpyAsync(p.x1, j.hx1, (size_t)j.k * 16, cudaMemcpyHostToDevice, st));
          B2_CUDA(ctx, cudaMemcpyAsync(p.x2, j.hx2, (size_t)j.k * 16, cudaMemcpyHostToDevice, st));
        } else {
          p.kp1 = j.kp1, p.kp2 = j.kp2, p.matches = reinterpret_cast<const long long*>(j.matches);
          // a fundamental-matrix problem keeps pixels: f = 1, u0 = v0 = 0
          for (int c = 0; c < 3; ++c) p.g1[c] = j.mode == 0 ? j.cal1[c] : (c == 0), p.g2[c] = j.mode == 0 ? j.cal2[c] : (c == 0);
          any_gather = true;
        }
      }
      p.models = s->models.as<double>() + o_smp * RS_MAX_SOL * 9, p.nsol = s->nsol.as<int>() + o_smp;
      p.cost = s->cost.as<double>() + o_smp * RS_MAX_SOL, p.ninl = s->ninl.as<int>() + o_smp * RS_MAX_SOL;
      o_smp += (size_t)rs_round_cap(j.mode, j.max_iters, batch);
      p.cand = dscr[t].cand, p.best = &dout[t].best, p.count = &dout[t].count;
      if (j.dmask) p.mask = j.dmask;
      else p.mask = s->mask.as<uint8_t>() + o_mask, o_mask += (size_t)j.k;
      p.E = dout[t].best.model, p.pose_mask = p.mask, p.gvotes = dscr[t].gvotes, p.pose = dout[t].pose;
      p.pose_cands = tr ? dscr[t].pose_cands : nullptr;
      p.pose_on = j.pose, p.pose_cal = j.pose && j.mode == 1;
      for (int c = 0; c < 3; ++c) p.c1[c] = j.cal1[c], p.c2[c] = j.cal2[c];
      max_k = j.k > max_k ? j.k : max_k;
      any_pose |= j.pose;
    }
  }
  B2_CUDA(ctx, cudaMemcpyAsync(dtab, htab, (size_t)L * sizeof(RsProb), cudaMemcpyHostToDevice, st));
  if (any_gather) {
    B2_LAUNCH(ctx, k_rs_gather, dim3(cdiv(max_k, 256), L), 256, 0, st, dtab);
    B2_CHECK_LAUNCH(ctx);
  }

  const double log_1mc = log(1.0 - confidence);
  // one sampling round over rows [0, R) of table `slot` (rows are sorted essential first): hypotheses, scores, selection
  auto round = [&](int slot, int R) -> int {
    RsProb* h = htab + (size_t)slot * L;
    RsProb* d = dtab + (size_t)slot * L;
    int nE = 0, maxnE = 0, maxnF = 0;
    for (int r = 0; r < R; ++r) {
      if (h[r].mode == 0) ++nE, maxnE = h[r].n > maxnE ? h[r].n : maxnE;
      else maxnF = h[r].n > maxnF ? h[r].n : maxnF;
    }
    B2_CUDA(ctx, cudaMemcpyAsync(d, h, (size_t)R * sizeof(RsProb), cudaMemcpyHostToDevice, st));
    if (nE) B2_LAUNCH(ctx, k_rs_hyp_E, dim3(cdiv(maxnE, 64), nE), 64, 0, st, d, (unsigned long long)seed);
    if (R - nE) B2_LAUNCH(ctx, k_rs_hyp_F, dim3(cdiv(maxnF, 64), R - nE), 64, 0, st, d + nE, (unsigned long long)seed);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_rs_score, dim3((maxnE > maxnF ? maxnE : maxnF) * RS_MAX_SOL, R), RS_SCORE_THREADS, 0, st, d);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_rs_select, dim3(1, R), 1024, 0, st, d, log_1mc);
    B2_CHECK_LAUNCH(ctx);
    return B2_OK;
  };
  // trace record of one k_rs_select launch over n samples (more_written: it wrote the confidence flag)
  auto record = [&](int ns_run, bool more_written) -> int {
    if (tr->records >= tr->max_records) return B2_OK;
    const int r = tr->records++;
    const size_t ns = (size_t)tr->batch;
    const auto d2h = cudaMemcpyDeviceToHost;
    if (tr->nsol) B2_CUDA(ctx, cudaMemcpyAsync(tr->nsol + r * ns, s->nsol.p, (size_t)ns_run * 4, d2h, st));
    if (tr->models)
      B2_CUDA(ctx, cudaMemcpyAsync(tr->models + r * ns * RS_MAX_SOL * 9, s->models.p, (size_t)ns_run * RS_MAX_SOL * 72, d2h, st));
    if (tr->cost) B2_CUDA(ctx, cudaMemcpyAsync(tr->cost + r * ns * RS_MAX_SOL, s->cost.p, (size_t)ns_run * RS_MAX_SOL * 8, d2h, st));
    if (tr->ninl) B2_CUDA(ctx, cudaMemcpyAsync(tr->ninl + r * ns * RS_MAX_SOL, s->ninl.p, (size_t)ns_run * RS_MAX_SOL * 4, d2h, st));
    if (tr->selected) B2_CUDA(ctx, cudaMemcpyAsync(tr->selected + (size_t)r * RS_TOP, dscr[0].cand, sizeof(RsBest) * RS_TOP, d2h, st));
    if (tr->more) {
      if (more_written) B2_CUDA(ctx, cudaMemcpyAsync(tr->more + r, dflags, 4, d2h, st));
      else tr->more[r] = -1;
    }
    RS_SYNC(ctx, st);
    return B2_OK;
  };

  // Sampling.  `run` holds the table rows that still draw samples; a row leaves it when its budget is spent or its flag says
  // the confidence bound is met.  A problem whose budget ends in a round gets its extension stage (E only: cv2's budget of
  // `max_iters` samples leaves a 30 %-inlier pair without a single uncontaminated 5-sample one time in eleven; USAC survives
  // that through its graph-cut local optimisation, a plain RANSAC does not.  The hypothesis kernel is latency-bound, so 4x more
  // samples cost about as much as the first batch) enqueued right behind that round, gated on the device by the flag the
  // round's k_rs_select wrote, so an E batch at the default budget never waits for the host.
  std::vector<int> run(L), done(L, 0), iters(L);
  for (int t = 0; t < L; ++t) run[t] = t, iters[t] = rs_clamp_iters(jobs[live[t]].mode, jobs[live[t]].max_iters);
  while (!run.empty()) {
    RsProb* h = htab + L;
    for (size_t r = 0; r < run.size(); ++r) {
      const int t = run[r];
      h[r] = htab[t];
      h[r].sample0 = done[t];
      h[r].n = iters[t] - done[t] < batch ? iters[t] - done[t] : batch;
      h[r].go = nullptr, h[r].more = dflags + t, h[r].done_after = (double)(done[t] + h[r].n);
    }
    if (int rc = round(1, (int)run.size())) return rc;
    if (tr) {
      ++tr->batches;
      if (int rc = record(h[0].n, true)) return rc;
    }
    std::vector<int> next;
    RsProb* hx = htab + 2 * (size_t)L;
    int n_ext = 0;
    for (size_t r = 0; r < run.size(); ++r) {
      const int t = run[r];
      done[t] += h[r].n;
      if (done[t] < iters[t]) {
        next.push_back(t);
      } else if (h[r].mode == 0 && iters[t] <= 4096) {
        RsProb& e = hx[n_ext++] = htab[t];
        e.sample0 = done[t];
        e.n = 4 * iters[t] < batch ? 4 * iters[t] : batch;
        e.go = dflags + t, e.more = nullptr, e.done_after = 0.0;
      }
    }
    if (n_ext) {
      if (int rc = round(2, n_ext)) return rc;
      if (tr) {  // the extension's buffers are only worth recording when its kernels ran
        B2_CUDA(ctx, cudaMemcpyAsync(&tr->ext_go, dflags, 4, cudaMemcpyDeviceToHost, st));
        RS_SYNC(ctx, st);
        if (tr->ext_go)
          if (int rc = record(hx[0].n, false)) return rc;
      }
    }
    run.clear();
    if (!next.empty()) {  // adaptive termination (standard RANSAC bound) between rounds: one read for the whole sub-batch
      B2_CUDA(ctx, cudaMemcpyAsync(hflags, dflags, (size_t)L * 4, cudaMemcpyDeviceToHost, st));
      RS_SYNC(ctx, st);
      for (int t : next)
        if (hflags[t]) run.push_back(t);
    }
  }

  if (tr) B2_CUDA(ctx, cudaMemcpyAsync(tr->prerefine, dscr[0].cand, sizeof(RsBest) * RS_TOP, cudaMemcpyDeviceToHost, st));
  B2_LAUNCH(ctx, k_rs_refine, dim3(RS_TOP, L), RS_LO_THREADS, 0, st, dtab);
  B2_CHECK_LAUNCH(ctx);
  if (tr) B2_CUDA(ctx, cudaMemcpyAsync(tr->refined, dscr[0].cand, sizeof(RsBest) * RS_TOP, cudaMemcpyDeviceToHost, st));
  B2_LAUNCH(ctx, k_rs_pick, dim3(1, L), 32, 0, st, dtab);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_rs_mask, dim3(cdiv(max_k, 256), L), 256, 0, st, dtab);
  B2_CHECK_LAUNCH(ctx);
  if (any_pose) {
    B2_LAUNCH(ctx, k_rs_pose, dim3(cdiv(max_k, RS_POSE_THREADS), L), RS_POSE_THREADS, 0, st, dtab);
    B2_CHECK_LAUNCH(ctx);
  }
  if (tr) {
    B2_CUDA(ctx, cudaMemcpyAsync(&tr->pick, &dout[0].best, sizeof(RsBest), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(&tr->mask_count, &dout[0].count, 4, cudaMemcpyDeviceToHost, st));
    if (any_pose) {
      double c[22];
      B2_CUDA(ctx, cudaMemcpyAsync(tr->votes, dscr[0].gvotes, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
      B2_CUDA(ctx, cudaMemcpyAsync(c, dscr[0].pose_cands, sizeof(c), cudaMemcpyDeviceToHost, st));
      RS_SYNC(ctx, st);
      memcpy(tr->pose_cands, c, 21 * 8);
      tr->winner = (int)c[21];
    }
  }
  B2_CUDA(ctx, cudaMemcpyAsync(hout, dout, (size_t)L * sizeof(RsOut), cudaMemcpyDeviceToHost, st));
  for (int t = 0; t < L; ++t)
    if (jobs[live[t]].hmask)
      B2_CUDA(ctx, cudaMemcpyAsync(jobs[live[t]].hmask, htab[t].mask, (size_t)jobs[live[t]].k, cudaMemcpyDeviceToHost, st));
  RS_SYNC(ctx, st);
  for (int t = 0; t < L; ++t) {
    const RsJob& j = jobs[live[t]];
    b2_ransac_result& r = res[live[t]];
    if (!hout[t].best.valid) continue;  // status 1; k_rs_mask wrote zeros
    r.status = 0;
    r.num_inliers = hout[t].count;
    memcpy(r.model, hout[t].best.model, 9 * 8);
    if (j.pose) memcpy(r.R, hout[t].pose, 9 * 8), memcpy(r.t, hout[t].pose + 9, 3 * 8);
  }
  return B2_OK;
}

// the caller holds ctx->mu and has selected the device
static int rs_run(b2_context* ctx, const RsJob* jobs, int n, double confidence, uint64_t seed, b2_ransac_result* res,
                  cudaStream_t st, b2_ransac_trace* tr = nullptr) {
  if (!ctx->rs) ctx->rs = new RansacState();
  std::vector<size_t> bytes(n);
  for (int i = 0; i < n; ++i)
    bytes[i] = rs_job_bytes(jobs[i].k, jobs[i].mode, jobs[i].max_iters, !jobs[i].dx1, !jobs[i].dmask, tr ? tr->batch : RS_BATCH);
  std::vector<int> first(n + 1);
  const int subs = rs_plan(bytes.data(), n, (size_t)ctx->rs_workspace_mb << 20, first.data());
  for (int b = 0; b < subs; ++b)
    if (int rc = rs_run_sub(ctx, jobs + first[b], first[b + 1] - first[b], confidence, seed, res + first[b], st, tr)) return rc;
  return B2_OK;
}

// the per-pair entry points: a table of one problem
static int rs_run_one(b2_context* ctx, const RsJob& job, const b2_ransac_params* prm, double* out_model, int* out_ninl,
                      double* out_R, double* out_t, cudaStream_t st, b2_ransac_trace* tr = nullptr) {
  b2_ransac_result r;
  *out_ninl = 0;
  if (int rc = rs_run(ctx, &job, 1, prm->confidence, prm->seed, &r, st, tr)) return rc;
  if (r.status) return 1;
  memcpy(out_model, r.model, 9 * 8);
  *out_ninl = r.num_inliers;
  if (job.pose) memcpy(out_R, r.R, 9 * 8), memcpy(out_t, r.t, 3 * 8);
  return B2_OK;
}

static RsJob rs_host_job(int mode, const double* x1, const double* x2, int k, const b2_ransac_params* prm, uint8_t* out_mask,
                         bool pose) {
  RsJob j;
  j.hx1 = x1, j.hx2 = x2, j.k = k, j.mode = mode, j.max_iters = prm->max_iters, j.threshold = prm->threshold;
  j.hmask = out_mask, j.pose = pose;
  return j;
}

extern "C" int b2_ransac_essential_host(b2_context* ctx, const double* x1, const double* x2, int k,
                                        const b2_ransac_params* params, double* out_model, uint8_t* out_mask,
                                        int* out_num_inliers, double* out_R, double* out_t) {
  if (!ctx || !x1 || !x2 || !params || !out_model || !out_num_inliers || k < 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return rs_run_one(ctx, rs_host_job(0, x1, x2, k, params, out_mask, out_R && out_t), params, out_model, out_num_inliers, out_R,
                    out_t, ctx->stream);
}

extern "C" int b2_ransac_fundamental_host(b2_context* ctx, const double* x1, const double* x2, int k,
                                          const b2_ransac_params* params, double* out_model, uint8_t* out_mask,
                                          int* out_num_inliers) {
  if (!ctx || !x1 || !x2 || !params || !out_model || !out_num_inliers || k < 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return rs_run_one(ctx, rs_host_job(1, x1, x2, k, params, out_mask, false), params, out_model, out_num_inliers, nullptr,
                    nullptr, ctx->stream);
}

extern "C" int b2_ransac_essential_dev(b2_context* ctx, const float* kp1, const float* kp2, const int64_t* matches, int k,
                                       const double* cal1, const double* cal2, const b2_ransac_params* params,
                                       double* out_model, uint8_t* out_mask_dev, int* out_num_inliers, double* out_R,
                                       double* out_t, void* stream) {
  if (!ctx || !params || !out_model || !out_num_inliers || !cal1 || !cal2 || k < 0) return B2_ERR_ARG;
  if (k > 0 && (!kp1 || !kp2 || !matches)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  RsJob j;
  j.kp1 = kp1, j.kp2 = kp2, j.matches = matches, j.k = k, j.mode = 0, j.max_iters = params->max_iters;
  j.threshold = params->threshold, j.dmask = out_mask_dev, j.pose = out_R && out_t;
  memcpy(j.cal1, cal1, sizeof(j.cal1)), memcpy(j.cal2, cal2, sizeof(j.cal2));
  // the legacy stream when `stream` is NULL; the context stream stays unused here
  return rs_run_one(ctx, j, params, out_model, out_num_inliers, out_R, out_t, stream ? (cudaStream_t)stream : cudaStreamLegacy);
}

static size_t rs_problem_bytes(const b2_ransac_problem& p) { return rs_job_bytes(p.k, p.mode, p.max_iters, !p.x1, !p.mask); }

extern "C" size_t b2_ransac_workspace_bytes(const b2_ransac_problem* problem) {
  return problem && (problem->mode == 0 || problem->mode == 1) && problem->k >= 0 ? rs_problem_bytes(*problem) : 0;
}

extern "C" int b2_ransac_plan(const b2_ransac_problem* problems, int n, size_t budget_bytes, int* out_first) {
  if (n < 0 || !out_first || (n > 0 && !problems)) return B2_ERR_ARG;
  std::vector<size_t> bytes(n);
  for (int i = 0; i < n; ++i) {
    if ((problems[i].mode != 0 && problems[i].mode != 1) || problems[i].k < 0) return B2_ERR_ARG;
    bytes[i] = rs_problem_bytes(problems[i]);
  }
  return rs_plan(bytes.data(), n, budget_bytes, out_first);
}

extern "C" int b2_ransac_verify_batched_dev(b2_context* ctx, const b2_ransac_problem* problems, int n,
                                            const b2_ransac_params* params, b2_ransac_result* results, void* stream) {
  if (!ctx || !params || n < 0 || (n > 0 && (!problems || !results))) return B2_ERR_ARG;
  if (!(params->confidence > 0.0 && params->confidence < 1.0)) return b2_fail(ctx, B2_ERR_ARG, "ransac: confidence must be in (0, 1)");
  std::vector<RsJob> jobs(n);
  for (int i = 0; i < n; ++i) {
    const b2_ransac_problem& p = problems[i];
    const std::string at = "ransac problem " + std::to_string(i) + ": ";
    if (p.k < 0 || (p.mode != 0 && p.mode != 1)) return b2_fail(ctx, B2_ERR_ARG, at + "k < 0 or mode not 0 / 1");
    if (!(p.threshold >= 0.0)) return b2_fail(ctx, B2_ERR_ARG, at + "threshold must be >= 0");
    const bool ready = p.x1 || p.x2;
    if (ready && (!p.x1 || !p.x2)) return b2_fail(ctx, B2_ERR_ARG, at + "x1 and x2 go together");
    if (p.k > 0 && !ready && (!p.kp1 || !p.kp2 || !p.matches)) return b2_fail(ctx, B2_ERR_ARG, at + "no points");
    // the focal lengths divide: E problems calibrate the keypoints with them, F problems their inliers for the pose
    if ((p.mode == 1 || !ready) && !(p.cal1[0] > 0.0 && p.cal2[0] > 0.0)) return b2_fail(ctx, B2_ERR_ARG, at + "focal length must be > 0");
    RsJob& j = jobs[i];
    j.kp1 = p.kp1, j.kp2 = p.kp2, j.matches = p.matches, j.dx1 = p.x1, j.dx2 = p.x2;
    j.k = p.k, j.mode = p.mode, j.max_iters = p.max_iters, j.threshold = p.threshold, j.dmask = p.mask, j.pose = true;
    memcpy(j.cal1, p.cal1, sizeof(j.cal1)), memcpy(j.cal2, p.cal2, sizeof(j.cal2));
  }
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return rs_run(ctx, jobs.data(), n, params->confidence, params->seed, results, stream ? (cudaStream_t)stream : cudaStreamLegacy);
}

extern "C" uint64_t b2_ransac_sync_count(const b2_context* ctx) { return ctx ? ctx->rs_syncs : 0; }

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
  B2_CUDA(ctx, s->small.ensure(sizeof(RsOut) + sizeof(RsScratch)));
  B2_CUDA(ctx, s->tab.ensure(sizeof(RsProb)));
  B2_CUDA(ctx, s->hbuf.ensure(sizeof(RsProb) + sizeof(RsOut)));
  if (k > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(s->x1.p, x1, (size_t)k * 16, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->x2.p, x2, (size_t)k * 16, cudaMemcpyHostToDevice, st));
  }
  RsOut* dout = s->small.as<RsOut>();
  RsScratch* dscr = reinterpret_cast<RsScratch*>(dout + 1);
  B2_CUDA(ctx, cudaMemsetAsync(dscr->gvotes, 0, sizeof(dscr->gvotes), st));
  B2_CUDA(ctx, cudaMemcpyAsync(dscr->E, E, 9 * 8, cudaMemcpyHostToDevice, st));
  RsProb* hp = s->hbuf.as<RsProb>();
  memset(hp, 0, sizeof(*hp));
  hp->x1 = s->x1.as<double>(), hp->x2 = s->x2.as<double>(), hp->k = k, hp->E = dscr->E, hp->gvotes = dscr->gvotes;
  hp->pose = dout->pose, hp->pose_cands = out_cands ? dscr->pose_cands : nullptr, hp->pose_on = 1;
  B2_CUDA(ctx, cudaMemcpyAsync(s->tab.p, hp, sizeof(RsProb), cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, k_rs_pose, k > 0 ? cdiv(k, RS_POSE_THREADS) : 1, RS_POSE_THREADS, 0, st, s->tab.as<RsProb>());
  B2_CHECK_LAUNCH(ctx);
  double* h = reinterpret_cast<double*>(hp + 1);
  B2_CUDA(ctx, cudaMemcpyAsync(h, dout->pose, 13 * 8, cudaMemcpyDeviceToHost, st));
  if (out_cands) {
    double c[22];
    B2_CUDA(ctx, cudaMemcpyAsync(c, dscr->pose_cands, sizeof(c), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(out_votes, dscr->gvotes, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
    RS_SYNC(ctx, st);
    memcpy(out_cands, c, 21 * 8);
    *out_winner = (int)c[21];
  }
  RS_SYNC(ctx, st);
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
  return rs_run_one(ctx, rs_host_job(mode, x1, x2, k, params, out_mask, mode == 0 && out_R && out_t), params, out_model,
                    out_num_inliers, out_R, out_t, ctx->stream, trace);
}
