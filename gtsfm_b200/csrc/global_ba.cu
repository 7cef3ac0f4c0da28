// Global bundle adjustment for sm_90a: gtsam's Levenberg-Marquardt on the graph BundleAdjustmentOptimizer builds
// (gtsfm/bundle/bundle_adjustment.py:148-410) over every camera, calibration and point, fp64 throughout.
// oracle/global_ba_ref.py states the same maths in NumPy.  One LM trial is:
//   k_gba_lin      one thread per measurement: whitened, Huber-reweighted residual and Jacobians (twoview_math.cuh's
//                  projection), stored as sqrt(w) J; once per linearisation point, not per trial
//   k_gba_point    one thread per track: the damped 3 x 3 point block, its Cholesky factor L, z = L^-1 g_p and
//                  W_m = L^-1 H_pc for each measurement
//   k_gba_blocks   one CTA per covisible camera pair (a >= b): the 9 x 9 block of the reduced camera system, summed over the
//                  pair's (track, measurement) list in its fixed sorted order
//   k_gba_karcher  beta I6 on the pose part of every block (the Karcher mean factor's linearisation)
//   k_gba_diag     priors and damping on the diagonal; k_gba_rhs the reduced right-hand side
//   dense_chol_solve  blocked right-looking Cholesky of the dense reduced system (64 x 64 tiles) and its two solves
//                  (dense_chol.cu, shared with the translation recovery)
//   k_gba_cams     one thread per camera: the retracted candidate and its priors' share of the decrease
//   k_gba_points   one thread per track: back-substitution, the candidate point, the track's linearised decrease and cost
//   k_gba_reduce   one CTA: the fixed-order sums, plus the Karcher term of the linearised decrease
// The host reads the reduced scalars back once per trial and applies twoview_math.cuh's lm_trial / lm_continue.
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "common.cuh"
#include "dense_chol.cuh"
#include "twoview_math.cuh"
#include "../../include/gtsfm_b200.h"

using namespace tvmath;

namespace {
constexpr int NB = CHOL_NB;        // Cholesky tile
constexpr int GB_THREADS = 128;
constexpr int RED_THREADS = 256;
constexpr int MEAS_DOUBLES = 18 + 6 + 2 + 27;  // per measurement: sqrt(w) Jc [2][9], sqrt(w) Jp [2][3], sqrt(w) r [2], W [3][9]

struct Gb {
  int C, np, gauge;
  int64_t N, M;
  double inv_sigma, huber_k, beta, pose_inv, cal_inv[3];
  const int64_t* toff;    // [N + 1]
  const int* mcam;        // [M]
  const double* uv;       // [M][2]
  const int* coff;        // [C + 1] measurements by camera
  const int* cmeas;       // [M] measurement ids, camera by camera, ascending
  const int2* pairs;      // (ma, mb) sorted by (cam(ma), cam(mb), track)
  const int64_t* poff;    // [nblk + 1]
  const int2* blk;        // [nblk] (a, b)
  const Cam* cam0;        // input cameras
  Cam *cur, *cand;
  double *pts, *ptsn;
  double* mq;             // [M][MEAS_DOUBLES]
  double *L, *z;          // [N][9], [N][3]
  double *S, *b, *y, *dc; // [np][np], [np] x 3
  double *tlin, *told, *tcost, *clin, *cold, *ccost;
  double* scal;           // [4]: lin, old, cost, flag
  int* flag;
};

__device__ __forceinline__ double robust_loss(const Gb& g, double e) { return g.huber_k > 0.0 ? huber_loss(e, g.huber_k) : 0.5 * e * e; }

// PriorFactorPose3(x, prior): whitened error -Local(x, prior) = -Logmap(x^-1 prior) / sigma (Jacobian I / sigma)
__device__ __forceinline__ void pose_prior_err(const Gb& g, const Cam& x, const Cam& p, double* e) {
  double R[9], t[3], d[3] = {p.t[0] - x.t[0], p.t[1] - x.t[1], p.t[2] - x.t[2]};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = x.R[i] * p.R[j] + x.R[3 + i] * p.R[3 + j] + x.R[6 + i] * p.R[6 + j];
    t[i] = x.R[i] * d[0] + x.R[3 + i] * d[1] + x.R[6 + i] * d[2];
  }
  se3_log(R, t, e);
  for (int i = 0; i < 6; ++i) e[i] = -e[i] * g.pose_inv;
}

// the cost of one track at (cams, X): sum of the robust losses of its measurements (0 behind a camera)
__device__ double track_cost(const Gb& g, const Cam* cams, const double* X, int64_t j) {
  double c = 0.0;
  for (int64_t m = g.toff[j]; m < g.toff[j + 1]; ++m) {
    const Cam& k = cams[g.mcam[m]];
    double pr[2];
    if (!(project(k.R, k.t, k.cal, X, pr, nullptr, nullptr) > 0.0)) continue;
    const double a = (pr[0] - g.uv[2 * m]) * g.inv_sigma, b = (pr[1] - g.uv[2 * m + 1]) * g.inv_sigma;
    c += robust_loss(g, sqrt(a * a + b * b));
  }
  return c;
}

// the priors' cost of camera a at `cams`
__device__ double cam_cost(const Gb& g, const Cam* cams, int a) {
  double c = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double e = (cams[a].cal[i] - g.cam0[a].cal[i]) * g.cal_inv[i];
    c += 0.5 * e * e;
  }
  if (g.gauge == B2_BA_FIRST_POSE_PRIOR && a == 0) {
    double e[6];
    pose_prior_err(g, cams[0], g.cam0[0], e);
    for (int i = 0; i < 6; ++i) c += 0.5 * e[i] * e[i];
  }
  return c;
}

}  // namespace

__global__ void __launch_bounds__(GB_THREADS) k_gba_lin(Gb g) {
  const int64_t m = blockIdx.x * (int64_t)GB_THREADS + threadIdx.x;
  if (m >= g.M) return;
  int64_t j = 0;
  {  // the track of m: binary search in toff
    int64_t lo = 0, hi = g.N;
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) / 2;
      if (g.toff[mid] <= m) lo = mid;
      else hi = mid;
    }
    j = lo;
  }
  const Cam& k = g.cur[g.mcam[m]];
  double pr[2], Jc[18], Jp[6];
  double* q = g.mq + m * MEAS_DOUBLES;
  const double z = project(k.R, k.t, k.cal, g.pts + 3 * j, pr, Jc, Jp);
  if (!(z > 0.0)) {  // GeneralSFMFactor2's cheirality branch: zero residual, zero Jacobians
    for (int i = 0; i < 26; ++i) q[i] = 0.0;
    return;
  }
  const double r0 = (pr[0] - g.uv[2 * m]) * g.inv_sigma, r1 = (pr[1] - g.uv[2 * m + 1]) * g.inv_sigma;
  const double w = g.huber_k > 0.0 ? huber_weight(sqrt(r0 * r0 + r1 * r1), g.huber_k) : 1.0;
  const double s = sqrt(w) * g.inv_sigma;
  for (int i = 0; i < 18; ++i) q[i] = s * Jc[i];
  for (int i = 0; i < 6; ++i) q[18 + i] = s * Jp[i];
  q[24] = sqrt(w) * r0, q[25] = sqrt(w) * r1;
}

__global__ void __launch_bounds__(GB_THREADS) k_gba_point(Gb g, double lam) {
  const int64_t j = blockIdx.x * (int64_t)GB_THREADS + threadIdx.x;
  if (j >= g.N) return;
  double H[9] = {0}, gp[3] = {0};
  for (int64_t m = g.toff[j]; m < g.toff[j + 1]; ++m) {
    const double* q = g.mq + m * MEAS_DOUBLES;
    for (int k = 0; k < 2; ++k)
      for (int i = 0; i < 3; ++i) {
        for (int c = 0; c < 3; ++c) H[i * 3 + c] += q[18 + 3 * k + i] * q[18 + 3 * k + c];
        gp[i] += q[18 + 3 * k + i] * q[24 + k];
      }
  }
  for (int i = 0; i < 3; ++i) H[i * 4] += lam;
  if (!chol(H, 3, 3)) *g.flag = 1;
  chol_fwd(H, 3, 3, gp);
  for (int i = 0; i < 9; ++i) g.L[9 * j + i] = H[i];
  for (int i = 0; i < 3; ++i) g.z[3 * j + i] = gp[i];
  for (int64_t m = g.toff[j]; m < g.toff[j + 1]; ++m) {
    double* q = g.mq + m * MEAS_DOUBLES;
    for (int c = 0; c < 9; ++c) {  // column c of W = L^-1 (Jp^T Jc)
      double h[3];
      for (int i = 0; i < 3; ++i) h[i] = q[18 + i] * q[c] + q[21 + i] * q[9 + c];
      chol_fwd(H, 3, 3, h);
      for (int i = 0; i < 3; ++i) q[26 + 9 * i + c] = h[i];
    }
  }
}

// one CTA per covisible block (a, b), a >= b: S_ab = sum over the block's list of [ma == mb] Jc^T Jc - W_ma^T W_mb
__global__ void __launch_bounds__(GB_THREADS) k_gba_blocks(Gb g) {
  if (*g.flag) return;
  const int e = threadIdx.x;
  if (e >= 81) return;
  const int r = e / 9, c = e % 9;
  const int2 ab = g.blk[blockIdx.x];
  double acc = 0.0;
  for (int64_t p = g.poff[blockIdx.x]; p < g.poff[blockIdx.x + 1]; ++p) {
    const int2 mm = g.pairs[p];
    const double* qa = g.mq + (int64_t)mm.x * MEAS_DOUBLES;
    const double* qb = g.mq + (int64_t)mm.y * MEAS_DOUBLES;
    double v = 0.0;
    if (mm.x == mm.y) v = qa[r] * qa[c] + qa[9 + r] * qa[9 + c];
    v -= qa[26 + r] * qb[26 + c] + qa[35 + r] * qb[35 + c] + qa[44 + r] * qb[44 + c];
    acc += v;
  }
  g.S[(int64_t)(9 * ab.x + r) * g.np + 9 * ab.y + c] = acc;
}

// the Karcher mean factor: beta I6 on the pose part of every block (a, b), a >= b
__global__ void k_gba_karcher(Gb g) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t nb = (int64_t)g.C * (g.C + 1) / 2;
  if (*g.flag || t >= nb * 6) return;
  const int64_t blk = t / 6;
  const int i = (int)(t % 6);
  int a = (int)((sqrt(8.0 * blk + 1.0) - 1.0) * 0.5);
  while ((int64_t)(a + 1) * (a + 2) / 2 <= blk) ++a;
  while ((int64_t)a * (a + 1) / 2 > blk) --a;
  const int b = (int)(blk - (int64_t)a * (a + 1) / 2);
  g.S[(int64_t)(9 * a + i) * g.np + 9 * b + i] += g.beta;
}

// the diagonal: calibration priors, the first-pose prior, the damping lam; identity on the padding
__global__ void k_gba_diag(Gb g, double lam) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (*g.flag || u >= g.np) return;
  double* d = g.S + (int64_t)u * g.np + u;
  if (u >= 9 * g.C) {
    *d = 1.0;
    return;
  }
  const int i = u % 9;
  if (i >= 6) *d += g.cal_inv[i - 6] * g.cal_inv[i - 6];
  else if (g.gauge == B2_BA_FIRST_POSE_PRIOR && u < 6) *d += g.pose_inv * g.pose_inv;
  *d += lam;
}

// the reduced right-hand side b = g_c - W^T z over each camera's measurements in order, plus the priors' gradients
__global__ void k_gba_rhs(Gb g) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (*g.flag || u >= g.np) return;
  if (u >= 9 * g.C) {
    g.b[u] = 0.0;
    return;
  }
  const int a = u / 9, i = u % 9;
  double acc = 0.0;
  for (int k = g.coff[a]; k < g.coff[a + 1]; ++k) {
    const int m = g.cmeas[k];
    const double* q = g.mq + (int64_t)m * MEAS_DOUBLES;
    int64_t lo = 0, hi = g.N;  // the track of m
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) / 2;
      if (g.toff[mid] <= m) lo = mid;
      else hi = mid;
    }
    const double* zj = g.z + 3 * lo;
    acc += q[i] * q[24] + q[9 + i] * q[25];
    acc -= q[26 + i] * zj[0] + q[35 + i] * zj[1] + q[44 + i] * zj[2];
  }
  if (i >= 6) {
    acc += (g.cur[a].cal[i - 6] - g.cam0[a].cal[i - 6]) * g.cal_inv[i - 6] * g.cal_inv[i - 6];
  } else if (g.gauge == B2_BA_FIRST_POSE_PRIOR && a == 0) {
    double e[6];
    pose_prior_err(g, g.cur[0], g.cam0[0], e);
    acc += e[i] * g.pose_inv;
  }
  g.b[u] = -acc;  // the solve's right-hand side
}

// one thread per camera: the candidate camera and its priors' linearised decrease, old linearised cost and candidate cost
__global__ void k_gba_cams(Gb g) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= g.C) return;
  const double* d = g.dc + 9 * a;
  Cam c = g.cur[a];
  retract_pose(c.R, c.t, d);
  for (int i = 0; i < 3; ++i) c.cal[i] += d[6 + i];
  g.cand[a] = c;
  double lin = 0.0, old = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double e = (g.cur[a].cal[i] - g.cam0[a].cal[i]) * g.cal_inv[i], jd = d[6 + i] * g.cal_inv[i];
    lin -= e * jd + 0.5 * jd * jd, old += 0.5 * e * e;
  }
  if (g.gauge == B2_BA_FIRST_POSE_PRIOR && a == 0) {
    double e[6];
    pose_prior_err(g, g.cur[0], g.cam0[0], e);
    for (int i = 0; i < 6; ++i) {
      const double jd = d[i] * g.pose_inv;
      lin -= e[i] * jd + 0.5 * jd * jd, old += 0.5 * e[i] * e[i];
    }
  }
  g.clin[a] = lin, g.cold[a] = old;
  g.ccost[a] = cam_cost(g, g.cand, a);
}

// one thread per track: dp = -L^-T (z + sum_m W_m dc_cam(m)), the candidate point, the track's share of the linearised
// decrease (sum_m -(r . Jd + |Jd|^2 / 2) over the whitened, reweighted rows) and of the old linearised cost, and its cost at
// the candidate
__global__ void __launch_bounds__(GB_THREADS) k_gba_points(Gb g) {
  const int64_t j = blockIdx.x * (int64_t)GB_THREADS + threadIdx.x;
  if (j >= g.N) return;
  double yv[3] = {g.z[3 * j], g.z[3 * j + 1], g.z[3 * j + 2]};
  for (int64_t m = g.toff[j]; m < g.toff[j + 1]; ++m) {
    const double* q = g.mq + m * MEAS_DOUBLES;
    const double* d = g.dc + 9 * g.mcam[m];
    for (int i = 0; i < 3; ++i) {
      double s = 0.0;
      for (int c = 0; c < 9; ++c) s += q[26 + 9 * i + c] * d[c];
      yv[i] += s;
    }
  }
  const double* L = g.L + 9 * j;
  for (int i = 2; i >= 0; --i) {  // L^T dp' = y, dp = -dp'
    double s = yv[i];
    for (int m = i + 1; m < 3; ++m) s -= L[m * 3 + i] * yv[m];
    yv[i] = s / L[i * 3 + i];
  }
  const double dp[3] = {-yv[0], -yv[1], -yv[2]};
  double Xn[3];
  for (int i = 0; i < 3; ++i) Xn[i] = g.pts[3 * j + i] + dp[i], g.ptsn[3 * j + i] = Xn[i];
  double lin = 0.0, old = 0.0;
  for (int64_t m = g.toff[j]; m < g.toff[j + 1]; ++m) {
    const double* q = g.mq + m * MEAS_DOUBLES;
    const double* d = g.dc + 9 * g.mcam[m];
    for (int k = 0; k < 2; ++k) {
      double jd = q[18 + 3 * k] * dp[0] + q[19 + 3 * k] * dp[1] + q[20 + 3 * k] * dp[2];
      for (int c = 0; c < 9; ++c) jd += q[9 * k + c] * d[c];
      const double r = q[24 + k];
      lin -= r * jd + 0.5 * jd * jd, old += 0.5 * r * r;
    }
  }
  g.tlin[j] = lin, g.told[j] = old;
  g.tcost[j] = track_cost(g, g.cand, Xn, j);
}

// the cost of the current state, per track and per camera (the LM's initial error)
__global__ void __launch_bounds__(GB_THREADS) k_gba_cost(Gb g) {
  const int64_t j = blockIdx.x * (int64_t)GB_THREADS + threadIdx.x;
  if (j < g.N) g.tcost[j] = track_cost(g, g.cur, g.pts + 3 * j, j);
  if (j < g.C) g.ccost[j] = cam_cost(g, g.cur, (int)j);
}

__device__ double block_sum_fixed(double v, double* red) {
  const int tid = threadIdx.x;
  red[tid] = v;
  __syncthreads();
  for (int s = RED_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// fixed-order sums: scal = {lin, old, cost at the candidate (or the current state: cost_only), failed}
__global__ void __launch_bounds__(RED_THREADS) k_gba_reduce(Gb g, int cost_only) {
  __shared__ double red[RED_THREADS];
  const int tid = threadIdx.x;
  double l = 0.0, o = 0.0, c = 0.0;
  const bool go = cost_only || !*g.flag;
  if (go) {
    for (int64_t j = tid; j < g.N; j += RED_THREADS) {
      c += g.tcost[j];
      if (!cost_only) l += g.tlin[j], o += g.told[j];
    }
    for (int a = tid; a < g.C; a += RED_THREADS) {
      c += g.ccost[a];
      if (!cost_only) l += g.clin[a], o += g.cold[a];
    }
  }
  l = block_sum_fixed(l, red);
  o = block_sum_fixed(o, red);
  c = block_sum_fixed(c, red);
  if (tid == 0) {
    if (go && !cost_only && g.gauge == B2_BA_KARCHER) {  // the Karcher factor: 0 at dx = 0, 0.5 beta |sum_i d_i|^2 after
      double s[6] = {0, 0, 0, 0, 0, 0};
      for (int a = 0; a < g.C; ++a)
        for (int i = 0; i < 6; ++i) s[i] += g.dc[9 * a + i];
      double n2 = 0.0;
      for (int i = 0; i < 6; ++i) n2 += s[i] * s[i];
      l -= 0.5 * g.beta * n2;
    }
    g.scal[0] = l, g.scal[1] = o, g.scal[2] = c, g.scal[3] = cost_only ? 0.0 : (double)*g.flag;
  }
}

__global__ void __launch_bounds__(GB_THREADS) k_gba_reproj(Gb g, double* err) {
  const int64_t m = blockIdx.x * (int64_t)GB_THREADS + threadIdx.x;
  if (m >= g.M) return;
  int64_t lo = 0, hi = g.N;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) / 2;
    if (g.toff[mid] <= m) lo = mid;
    else hi = mid;
  }
  const Cam& k = g.cur[g.mcam[m]];
  double pr[2];
  const double z = project(k.R, k.t, k.cal, g.pts + 3 * lo, pr, nullptr, nullptr);
  const double a = pr[0] - g.uv[2 * m], b = pr[1] - g.uv[2 * m + 1];
  err[m] = z > 0.0 ? sqrt(a * a + b * b) : __longlong_as_double(0x7ff8000000000000LL);
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct GlobalBaState {
  DevBuf ws;
};

void gb_destroy(b2_context* ctx) {
  delete ctx->gb;
  ctx->gb = nullptr;
}

namespace {
struct Layout {
  size_t off[32];
  size_t total;
};

int padded(int C) { return (9 * C + NB - 1) / NB * NB; }

// byte offsets of every device array of a call (16-byte aligned)
Layout layout(int C, int64_t N, int64_t M, int64_t P, int64_t nblk) {
  const int np = padded(C);
  const size_t sizes[] = {
      (size_t)np * np * 8,              // 0 S
      (size_t)np * 8, (size_t)np * 8, (size_t)np * 8,  // 1-3 b, y, dc
      (size_t)M * MEAS_DOUBLES * 8,     // 4 mq
      (size_t)N * 72, (size_t)N * 24,   // 5-6 L, z
      (size_t)N * 24, (size_t)N * 24,   // 7-8 pts, ptsn
      (size_t)N * 24,                   // 9 tlin, told, tcost
      (size_t)C * 24,                   // 10 clin, cold, ccost
      (size_t)C * sizeof(Cam) * 3,      // 11 cam0, cur, cand
      (size_t)(N + 1) * 8,              // 12 toff
      (size_t)M * 4, (size_t)M * 16,    // 13-14 mcam, uv
      (size_t)(C + 1) * 4, (size_t)M * 4,  // 15-16 coff, cmeas
      (size_t)P * 8, (size_t)(nblk + 1) * 8, (size_t)nblk * 8,  // 17-19 pairs, poff, blk
      64,                               // 20 scal + flag
      (size_t)M * 8,                    // 21 reprojection errors
  };
  Layout l{};
  size_t o = 0;
  for (size_t i = 0; i < sizeof(sizes) / sizeof(sizes[0]); ++i) l.off[i] = o, o += (sizes[i] + 255) / 256 * 256;
  l.total = o;
  return l;
}

int64_t pair_count(int64_t N, const int64_t* toff) {
  int64_t p = 0;
  for (int64_t j = 0; j < N; ++j) {
    const int64_t k = toff[j + 1] - toff[j];
    p += k * (k + 1) / 2;
  }
  return p;
}

bool finite_all(const double* v, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}
}  // namespace

extern "C" size_t b2_bundle_adjust_workspace_bytes(int C, int64_t N, const int64_t* track_off) {
  if (C < 1 || N < 1 || !track_off || track_off[0] != 0) return 0;
  for (int64_t j = 0; j < N; ++j)
    if (track_off[j + 1] <= track_off[j]) return 0;
  const int64_t M = track_off[N];
  // every block the pair list can name, bounded by C (C + 1) / 2 and by the pairs themselves
  const int64_t P = pair_count(N, track_off);
  return layout(C, N, M, P, std::min<int64_t>(P, (int64_t)C * (C + 1) / 2)).total;
}

extern "C" int b2_bundle_adjust_host(b2_context* ctx, int C, const double* cams, int64_t N, const double* points,
                                     const int64_t* track_off, const int32_t* meas_cam, const double* meas_uv,
                                     const b2_ba_params* prm, double* cams_out, double* points_out, double* reproj_err,
                                     b2_ba_result* result, double* trace, int32_t* trial_out, int trial_cap, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (!prm) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: params is NULL");
  if (C < 1 || N < 1) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: needs at least one camera and one track");
  if (C > 1000000 || !cams || !points || !track_off || !meas_cam || !meas_uv || !cams_out || !points_out || !reproj_err || !result)
    return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: a required array is NULL");
  if (trial_cap < 0 || (trial_cap > 0 && !trial_out)) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: bad trial_out / trial_cap");
  if (!(prm->noise_sigma > 0.0) || !std::isfinite(prm->noise_sigma) || !(prm->huber_k >= 0.0) || !std::isfinite(prm->huber_k) ||
      (prm->gauge != B2_BA_KARCHER && prm->gauge != B2_BA_FIRST_POSE_PRIOR) || prm->max_iters < 0 || prm->max_iters > 100000 ||
      !(prm->karcher_beta >= 0.0) || !std::isfinite(prm->karcher_beta) ||
      (prm->gauge == B2_BA_FIRST_POSE_PRIOR && !(prm->pose_prior_sigma > 0.0)) || !(prm->cal_prior_sigma[0] > 0.0) ||
      !(prm->cal_prior_sigma[1] > 0.0) || !(prm->cal_prior_sigma[2] > 0.0))
    return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: bad params");
  if (track_off[0] != 0) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: track_off[0] must be 0");
  for (int64_t j = 0; j < N; ++j)
    if (track_off[j + 1] <= track_off[j]) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: track " + std::to_string(j) + " has no measurement");
  const int64_t M = track_off[N];
  if (M >= (int64_t)1 << 31) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: more than 2^31 - 1 measurements");
  if (!finite_all(cams, (int64_t)C * 17) || !finite_all(points, 3 * N) || !finite_all(meas_uv, 2 * M))
    return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: non-finite input");
  for (int a = 0; a < C; ++a)
    if (!(cams[17 * a + 12] > 0.0)) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: camera " + std::to_string(a) + " has f <= 0");
  std::vector<int> seen(C, -1);
  for (int64_t j = 0; j < N; ++j)
    for (int64_t m = track_off[j]; m < track_off[j + 1]; ++m) {
      const int a = meas_cam[m];
      if (a < 0 || a >= C) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: camera index out of range");
      if (seen[a] == (int)j) return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: track " + std::to_string(j) + " has two measurements in one camera");
      seen[a] = (int)j;
    }
  // the covisibility structure, fixed for the call: pairs (ma, mb), cam(ma) >= cam(mb), by block (a, b) then track
  const int64_t P = pair_count(N, track_off);
  const int64_t nb_all = (int64_t)C * (C + 1) / 2;
  const size_t budget = (size_t)ctx->ba_workspace_mb << 20;
  if (layout(C, N, M, P, std::min(P, nb_all)).total > budget)
    return b2_fail(ctx, B2_ERR_ARG, "bundle_adjust: the problem needs more than ba_workspace_mb of device workspace");
  std::vector<int64_t> cnt(nb_all + 1, 0);
  auto bkey = [](int a, int b) { return (int64_t)a * (a + 1) / 2 + b; };
  for (int64_t j = 0; j < N; ++j)
    for (int64_t x = track_off[j]; x < track_off[j + 1]; ++x)
      for (int64_t w = track_off[j]; w < track_off[j + 1]; ++w)
        if (meas_cam[x] > meas_cam[w] || x == w) ++cnt[bkey(meas_cam[x], meas_cam[w]) + 1];
  std::vector<int64_t> poff;
  std::vector<int2> blk;
  std::vector<int64_t> slot(nb_all, -1);
  poff.push_back(0);
  for (int a = 0; a < C; ++a)
    for (int b = 0; b <= a; ++b) {
      const int64_t k = bkey(a, b);
      if (!cnt[k + 1]) continue;
      slot[k] = poff.back();
      blk.push_back(make_int2(a, b));
      poff.push_back(poff.back() + cnt[k + 1]);
    }
  const int64_t nblk = (int64_t)blk.size();
  std::vector<int2> pairs(P);
  for (int64_t j = 0; j < N; ++j)
    for (int64_t x = track_off[j]; x < track_off[j + 1]; ++x)
      for (int64_t w = track_off[j]; w < track_off[j + 1]; ++w)
        if (meas_cam[x] > meas_cam[w] || x == w) pairs[slot[bkey(meas_cam[x], meas_cam[w])]++] = make_int2((int)x, (int)w);
  std::vector<int> coff(C + 1, 0), cmeas(M);
  for (int64_t m = 0; m < M; ++m) ++coff[meas_cam[m] + 1];
  for (int a = 0; a < C; ++a) coff[a + 1] += coff[a];
  {
    std::vector<int> fill(coff.begin(), coff.end() - 1);
    for (int64_t m = 0; m < M; ++m) cmeas[fill[meas_cam[m]]++] = (int)m;
  }

  const Layout l = layout(C, N, M, P, nblk);
  const int np = padded(C);
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  if (!ctx->gb) ctx->gb = new GlobalBaState();
  GlobalBaState* s = ctx->gb;
  B2_CUDA(ctx, s->ws.ensure(l.total));
  char* base = s->ws.as<char>();
  auto at = [&](int i) { return base + l.off[i]; };
  Gb g{};
  g.C = C, g.np = np, g.gauge = prm->gauge, g.N = N, g.M = M;
  g.inv_sigma = 1.0 / prm->noise_sigma, g.huber_k = prm->huber_k, g.beta = prm->karcher_beta;
  g.pose_inv = prm->gauge == B2_BA_FIRST_POSE_PRIOR ? 1.0 / prm->pose_prior_sigma : 0.0;
  for (int i = 0; i < 3; ++i) g.cal_inv[i] = 1.0 / prm->cal_prior_sigma[i];
  g.S = (double*)at(0), g.b = (double*)at(1), g.y = (double*)at(2), g.dc = (double*)at(3);
  g.mq = (double*)at(4), g.L = (double*)at(5), g.z = (double*)at(6);
  g.pts = (double*)at(7), g.ptsn = (double*)at(8);
  g.tlin = (double*)at(9), g.told = g.tlin + N, g.tcost = g.tlin + 2 * N;
  g.clin = (double*)at(10), g.cold = g.clin + C, g.ccost = g.clin + 2 * C;
  Cam* cam0 = (Cam*)at(11);
  g.cam0 = cam0, g.cur = cam0 + C, g.cand = cam0 + 2 * C;
  g.toff = (const int64_t*)at(12), g.mcam = (const int*)at(13), g.uv = (const double*)at(14);
  g.coff = (const int*)at(15), g.cmeas = (const int*)at(16);
  g.pairs = (const int2*)at(17), g.poff = (const int64_t*)at(18), g.blk = (const int2*)at(19);
  g.scal = (double*)at(20), g.flag = (int*)(g.scal + 4);
  double* d_err = (double*)at(21);
  static_assert(sizeof(Cam) == 17 * 8, "Cam is the 17-double camera row");
  B2_CUDA(ctx, cudaMemcpyAsync(cam0, cams, (size_t)C * sizeof(Cam), cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(g.cur, cams, (size_t)C * sizeof(Cam), cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(g.pts, points, (size_t)N * 24, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.toff, track_off, (size_t)(N + 1) * 8, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.mcam, meas_cam, (size_t)M * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.uv, meas_uv, (size_t)M * 16, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.coff, coff.data(), (size_t)(C + 1) * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.cmeas, cmeas.data(), (size_t)M * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.pairs, pairs.data(), (size_t)P * 8, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.poff, poff.data(), (size_t)(nblk + 1) * 8, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)g.blk, blk.data(), (size_t)nblk * 8, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(g.scal, 0, 64, st));
  ctx->h2d_bytes += (uint64_t)(2 * C * sizeof(Cam) + N * 32 + 8 + M * 24 + P * 8 + (nblk + 1) * 16 + (C + 1) * 4 + M * 4);

  const unsigned gm = (unsigned)((M + GB_THREADS - 1) / GB_THREADS), gn = (unsigned)((N + GB_THREADS - 1) / GB_THREADS);
  const unsigned gnc = (unsigned)((std::max<int64_t>(N, C) + GB_THREADS - 1) / GB_THREADS);
  double hs[4];
  auto read_scal = [&]() -> int {
    B2_CUDA(ctx, cudaMemcpyAsync(hs, g.scal, 32, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    return B2_OK;
  };

  // the initial error
  B2_LAUNCH(ctx, k_gba_cost, gnc, GB_THREADS, 0, st, g);
  B2_LAUNCH(ctx, k_gba_reduce, 1, RED_THREADS, 0, st, g, 1);
  B2_CHECK_LAUNCH(ctx);
  if (int rc = read_scal()) return rc;
  double nw = hs[2], lam = LM_LAMBDA0;
  int its = 0, ntrace = 0, trials = 0;
  if (trace) trace[ntrace] = nw;
  ++ntrace;
  if (nw > 0.0) {
    bool linearise = true;
    for (;;) {
      const double cur = nw;
      if (linearise) {
        B2_LAUNCH(ctx, k_gba_lin, gm, GB_THREADS, 0, st, g);
        B2_CHECK_LAUNCH(ctx);
        linearise = false;
      }
      for (;;) {  // tryLambda
        B2_CUDA(ctx, cudaMemsetAsync(g.flag, 0, 4, st));
        B2_CUDA(ctx, cudaMemsetAsync(g.S, 0, (size_t)np * np * 8, st));
        B2_LAUNCH(ctx, k_gba_point, gn, GB_THREADS, 0, st, g, lam);
        if (nblk) B2_LAUNCH(ctx, k_gba_blocks, (unsigned)nblk, GB_THREADS, 0, st, g);
        if (g.beta > 0.0 && g.gauge == B2_BA_KARCHER)
          B2_LAUNCH(ctx, k_gba_karcher, (unsigned)((nb_all * 6 + 255) / 256), 256, 0, st, g);
        B2_LAUNCH(ctx, k_gba_diag, (unsigned)cdiv(np, 256), 256, 0, st, g, lam);
        B2_LAUNCH(ctx, k_gba_rhs, (unsigned)cdiv(np, GB_THREADS), GB_THREADS, 0, st, g);
        B2_CHECK_LAUNCH(ctx);
        if (int rc = dense_chol_solve(ctx, g.S, np, g.b, g.y, g.dc, g.flag, st)) return rc;
        B2_LAUNCH(ctx, k_gba_cams, (unsigned)cdiv(C, GB_THREADS), GB_THREADS, 0, st, g);
        B2_LAUNCH(ctx, k_gba_points, gn, GB_THREADS, 0, st, g);
        B2_LAUNCH(ctx, k_gba_reduce, 1, RED_THREADS, 0, st, g, 0);
        B2_CHECK_LAUNCH(ctx);
        if (int rc = read_scal()) return rc;
        bool success = false, stop = false;
        const bool failed = hs[3] != 0.0;
        if (!failed) lm_trial(hs[0], hs[1], cur, hs[2], success, stop);
        if (trials < trial_cap) trial_out[trials] = failed ? -1 : success ? 1 : stop ? 2 : 0;
        ++trials;
        if (success) {
          std::swap(g.cur, g.cand);
          std::swap(g.pts, g.ptsn);
          lam /= LM_FACTOR, ++its, nw = hs[2];
          linearise = true;
          break;
        }
        if (stop) break;
        lam *= LM_FACTOR;
        if (lam >= LM_LAMBDA_MAX) break;
      }
      if (trace) trace[ntrace] = nw;
      ++ntrace;
      if (!lm_continue(its, prm->max_iters, cur, nw, LM_ABS_TOL)) break;
    }
  }
  B2_LAUNCH(ctx, k_gba_reproj, gm, GB_THREADS, 0, st, g, d_err);
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaMemcpyAsync(cams_out, g.cur, (size_t)C * sizeof(Cam), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(points_out, g.pts, (size_t)N * 24, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(reproj_err, d_err, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memset(result, 0, sizeof(*result));
  result->iterations = its, result->trace_len = ntrace, result->trials = trials, result->final_error = nw;
  return B2_OK;
}
