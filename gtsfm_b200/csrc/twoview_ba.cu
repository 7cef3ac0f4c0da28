// Two-view refinement for sm_90a: triangulation, two-view bundle adjustment and inlier support for a batch of verified
// pairs, the per-pair CPU stage of the reference's TwoViewEstimator.run_2view (gtsfm/two_view_estimator.py:350-481) that
// follows verification when bundle_adjust_2view is set.  oracle/twoview_ba_ref.py states the same maths in NumPy.
//   k_tv_triangulate  one thread per putative row of every pair: gathers the row's pixels and, for a verified row, DLT +
//                     gtsam's point refinement + the cheirality / reprojection / angle checks (twoview_math.cuh)
//   k_tv_ba           one CTA per pair: the whole Levenberg-Marquardt loop (gtsam's schedule) on the device.  The points
//                     are eliminated track by track (their 3 x 3 blocks live in registers), each track's Schur terms
//                     go to shared memory in tiles of TV_TILE and are reduced in fixed order, one thread per entry of the
//                     18 x 18 reduced camera system; one warp factors it.  Accept / reject and lambda stay on the device.
//   k_tv_finish       one CTA per pair: the indeterminate-system test, the 0.5 px filter, the surviving rows compacted
//                     in row order, and the inlier-support decision
// A sub-batch is these 3 launches, one copy of the problem table in, one copy of the results out and one synchronisation.
// Every reduction has a fixed order that does not depend on the other pairs of the batch, so a pair's result is the same
// bit for bit whatever it is batched with.
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "twoview_math.cuh"
#include "../../include/gtsfm_b200.h"

using namespace tvmath;

namespace {
constexpr int TV_THREADS = 256;
constexpr int TV_TILE = 128;   // tracks whose Schur terms are in shared memory at once
constexpr int TV_TERMS = 97;   // per track: A [4][9] (sqrt(w) J over the camera's unknowns), sqrt(w) r [4], W [18][3], z [3]
constexpr int TV_NS = 171;     // lower triangle of the 18 x 18 reduced system
constexpr int TV_TRI_THREADS = 128;

struct TvOut {
  int status, num_rows, num_verified, num_tracks, iterations, bundle_adjusted, indeterminate, trace_len;
  double R[9], t[3], final_error;
};

struct TvProb {
  const float *kp1, *kp2;
  const long long* matches;
  const uint8_t* vmask;
  uint8_t* out_mask;
  long long* out_rows;
  int k;
  Cam cam0[2];       // initial cameras: Pose3(), Pose3(R, t)^-1
  double R0[9], t0[3];
  double* uv;        // [k][4] pixels of the row in both images
  double* pts;       // [2][k][3] current / candidate points (which is current: TvOut-independent `sel`)
  int* flag;         // [k] 1 = verified row that triangulated
  Cam* cams;         // [2] the optimised cameras (k_tv_ba -> k_tv_finish)
  int* sel;          // which half of pts holds the optimised points
  int* first;        // the first track's row
  double* anchor;    // [3] the first track's triangulated point (PriorFactorPoint3)
  double* trace;     // [max_iters + 2]
  TvOut* out;
};

struct TvParams {
  int max_iters, min_inliers;
  double min_ratio, ba_thr, tri_thr, min_angle;
};

// one track's terms in camera c: whitened residual r, J over the camera's 9 unknowns, J over the point, Huber weight
// (GeneralSFMFactor2: a point behind the camera contributes nothing)
__device__ __forceinline__ void track_cam(const Cam& cam, const double* uv, const double* X, double* r, double* Jc, double* Jp,
                                          double& w) {
  double pr[2];
  const double z = project(cam.R, cam.t, cam.cal, X, pr, Jc, Jp);
  if (!(z > 0.0)) {
    r[0] = r[1] = 0.0, w = 1.0;
    for (int i = 0; i < 18; ++i) Jc[i] = 0.0;
    for (int i = 0; i < 6; ++i) Jp[i] = 0.0;
    return;
  }
  r[0] = pr[0] - uv[0], r[1] = pr[1] - uv[1];
  w = huber_weight(sqrt(r[0] * r[0] + r[1] * r[1]));
}

__device__ __forceinline__ double track_cost(const Cam* cams, const double* uv, const double* X) {
  double c = 0.0;
  for (int k = 0; k < 2; ++k) {
    double pr[2];
    if (!(project(cams[k].R, cams[k].t, cams[k].cal, X, pr, nullptr, nullptr) > 0.0)) continue;
    const double a = pr[0] - uv[2 * k], b = pr[1] - uv[2 * k + 1];
    c += huber_loss(sqrt(a * a + b * b));
  }
  return c;
}

// the Hessian block of a track's point (undamped), its gradient, and the camera-point coupling Hcp [18][3]
struct TrackLin {
  double r[4], Jc[2][18], Jp[2][6], w[2];
};
__device__ __forceinline__ void track_lin(const Cam* cams, const double* uv, const double* X, TrackLin& t) {
  for (int c = 0; c < 2; ++c) track_cam(cams[c], uv + 2 * c, X, t.r + 2 * c, t.Jc[c], t.Jp[c], t.w[c]);
}
__device__ __forceinline__ void point_block(const TrackLin& t, bool first, const double* X, const double* pt0, double lam,
                                            double* H, double* g) {
  for (int i = 0; i < 9; ++i) H[i] = 0.0;
  for (int i = 0; i < 3; ++i) g[i] = 0.0;
  for (int c = 0; c < 2; ++c)
    for (int m = 0; m < 2; ++m) {
      const double* J = t.Jp[c] + 3 * m;
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) H[i * 3 + j] += t.w[c] * J[i] * J[j];
        g[i] += t.w[c] * J[i] * t.r[2 * c + m];
      }
    }
  if (first) {
    const double s2 = 1.0 / (POINT_PRIOR_SIGMA * POINT_PRIOR_SIGMA);
    for (int i = 0; i < 3; ++i) H[i * 4] += s2, g[i] += (X[i] - pt0[i]) * s2;
  }
  for (int i = 0; i < 3; ++i) H[i * 4] += lam;
}

__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < TV_THREADS / 32; ++i) s += red[i];
  return s;
}

// shared state of one pair's CTA
struct TvShared {
  double S[18][19], b[18], full[18], dc[18];
  Cam cur[2], cand[2];
  double cal0[2][3], pt0[3], red[TV_THREADS / 32];
  int bad, first;
};

// the lower triangle entry e < 171 -> (a, b), a >= b
__device__ __forceinline__ void tri_index(int e, int& a, int& b) {
  a = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
  while ((a + 1) * (a + 2) / 2 <= e) ++a;
  while (a * (a + 1) / 2 > e) --a;
  b = e - a * (a + 1) / 2;
}

// Pass A: the reduced camera system S (+ lam I) and b at the current values into sh.S / sh.b.  `check`: undamped, with
// the pivot test of every point block (sh.bad) and the full Hessian's camera diagonal (sh.full).
__device__ void build_system(const TvProb& p, const double* pts, TvShared& sh, double* terms, double lam, bool check) {
  const int tid = threadIdx.x;
  double acc = 0.0;
  int ea = 0, eb = 0;
  if (tid < TV_NS) tri_index(tid, ea, eb);
  for (int r0 = 0; r0 < p.k; r0 += TV_TILE) {
    if (tid < TV_TILE) {
      double* T = terms + tid * TV_TERMS;
      const int row = r0 + tid;
      if (row < p.k && p.flag[row]) {
        TrackLin t;
        const double* X = pts + 3 * row;
        track_lin(sh.cur, p.uv + 4 * row, X, t);
        double H[9], g[3];
        point_block(t, row == sh.first, X, sh.pt0, lam, H, g);
        const double d0 = H[0], d1 = H[4], d2 = H[8];
        if (!chol(H, 3, 3)) {
          sh.bad = 1;
          for (int i = 0; i < TV_TERMS; ++i) T[i] = 0.0;
        } else {
          if (check && !(H[0] * H[0] > INDETERMINATE_PIVOT * d0 && H[4] * H[4] > INDETERMINATE_PIVOT * d1 &&
                         H[8] * H[8] > INDETERMINATE_PIVOT * d2))
            sh.bad = 1;
          for (int c = 0; c < 2; ++c) {
            const double sw = sqrt(t.w[c]);
            for (int m = 0; m < 2; ++m) {
              for (int j = 0; j < 9; ++j) T[(2 * c + m) * 9 + j] = sw * t.Jc[c][9 * m + j];
              T[36 + 2 * c + m] = sw * t.r[2 * c + m];
            }
          }
          for (int a = 0; a < 18; ++a) {  // W row a = L^-1 (Hcp row a)
            const int c = a / 9, j = a % 9;
            double h[3];
            for (int i = 0; i < 3; ++i)
              h[i] = t.w[c] * (t.Jc[c][j] * t.Jp[c][i] + t.Jc[c][9 + j] * t.Jp[c][3 + i]);
            chol_fwd(H, 3, 3, h);
            for (int i = 0; i < 3; ++i) T[40 + a * 3 + i] = h[i];
          }
          chol_fwd(H, 3, 3, g);
          for (int i = 0; i < 3; ++i) T[94 + i] = g[i];
        }
      } else {
        for (int i = 0; i < TV_TERMS; ++i) T[i] = 0.0;
      }
    }
    __syncthreads();
    const int n = min(TV_TILE, p.k - r0);
    if (tid < TV_NS) {
      const bool same = ea / 9 == eb / 9;
      const int c = ea / 9, ja = ea % 9, jb = eb % 9;
      for (int j = 0; j < n; ++j) {
        const double* T = terms + j * TV_TERMS;
        double v = 0.0;
        if (same) v = T[(2 * c) * 9 + ja] * T[(2 * c) * 9 + jb] + T[(2 * c + 1) * 9 + ja] * T[(2 * c + 1) * 9 + jb];
        v -= T[40 + ea * 3] * T[40 + eb * 3] + T[40 + ea * 3 + 1] * T[40 + eb * 3 + 1] + T[40 + ea * 3 + 2] * T[40 + eb * 3 + 2];
        acc += v;
      }
    } else if (tid < TV_NS + 18) {
      const int a = tid - TV_NS, c = a / 9, ja = a % 9;
      for (int j = 0; j < n; ++j) {
        const double* T = terms + j * TV_TERMS;
        acc += T[(2 * c) * 9 + ja] * T[36 + 2 * c] + T[(2 * c + 1) * 9 + ja] * T[36 + 2 * c + 1];
        acc -= T[40 + a * 3] * T[94] + T[40 + a * 3 + 1] * T[95] + T[40 + a * 3 + 2] * T[96];
      }
    } else if (check && tid < TV_NS + 36) {
      const int a = tid - TV_NS - 18, c = a / 9, ja = a % 9;
      for (int j = 0; j < n; ++j) {
        const double* T = terms + j * TV_TERMS;
        acc += T[(2 * c) * 9 + ja] * T[(2 * c) * 9 + ja] + T[(2 * c + 1) * 9 + ja] * T[(2 * c + 1) * 9 + ja];
      }
    }
    __syncthreads();
  }
  if (tid < TV_NS) sh.S[ea][eb] = acc;
  else if (tid < TV_NS + 18) sh.b[tid - TV_NS] = acc;
  else if (check && tid < TV_NS + 36) sh.full[tid - TV_NS - 18] = acc;
  __syncthreads();
  if (tid == 0) {  // priors: pose of camera 0 (Jacobian I / sigma), calibrations; the damping
    double xi[6];
    se3_log(sh.cur[0].R, sh.cur[0].t, xi);
    const double ip = 1.0 / POSE_PRIOR_SIGMA, ic = 1.0 / CAL_PRIOR_SIGMA;
    for (int i = 0; i < 6; ++i) sh.S[i][i] += ip * ip, sh.b[i] += xi[i] * ip * ip, sh.full[i] += check ? ip * ip : 0.0;
    for (int c = 0; c < 2; ++c)
      for (int i = 0; i < 3; ++i) {
        const int a = 9 * c + 6 + i;
        sh.S[a][a] += ic * ic, sh.b[a] += (sh.cur[c].cal[i] - sh.cal0[c][i]) * ic * ic;
        if (check) sh.full[a] += ic * ic;
      }
    for (int a = 0; a < 18; ++a) sh.S[a][a] += lam;
  }
  __syncthreads();
}

// one warp: Cholesky of sh.S in place (lower), row i owned by lane i.  `rel` > 0: a pivot must also exceed rel * full[k].
__device__ bool warp_chol18(TvShared& sh, double rel) {
  const int lane = threadIdx.x & 31;
  bool ok = true;
  for (int k = 0; k < 18; ++k) {
    const double piv = sh.S[k][k];
    ok = ok && piv > 0.0 && isfinite(piv) && !(rel > 0.0 && !(piv > rel * sh.full[k]));
    if (!ok) return false;
    const double l = sqrt(piv);
    __syncwarp();
    if (lane > k && lane < 18) sh.S[lane][k] /= l;
    __syncwarp();
    if (lane == 0) sh.S[k][k] = l;
    if (lane > k && lane < 18)
      for (int j = k + 1; j <= lane; ++j) sh.S[lane][j] -= sh.S[lane][k] * sh.S[j][k];
    __syncwarp();
  }
  return true;
}

__device__ double prior_cost(const TvShared& sh, const Cam* cams) {
  double xi[6], c = 0.0;
  se3_log(cams[0].R, cams[0].t, xi);
  for (int i = 0; i < 6; ++i) c += 0.5 * (xi[i] / POSE_PRIOR_SIGMA) * (xi[i] / POSE_PRIOR_SIGMA);
  for (int k = 0; k < 2; ++k)
    for (int i = 0; i < 3; ++i) {
      const double e = (cams[k].cal[i] - sh.cal0[k][i]) / CAL_PRIOR_SIGMA;
      c += 0.5 * e * e;
    }
  return c;
}

__device__ double full_cost(const TvProb& p, const double* pts, const Cam* cams, TvShared& sh) {
  double c = 0.0;
  for (int row = threadIdx.x; row < p.k; row += TV_THREADS) {
    if (!p.flag[row]) continue;
    const double* X = pts + 3 * row;
    c += track_cost(cams, p.uv + 4 * row, X);
    if (row == sh.first)
      for (int i = 0; i < 3; ++i) c += 0.5 * ((X[i] - sh.pt0[i]) / POINT_PRIOR_SIGMA) * ((X[i] - sh.pt0[i]) / POINT_PRIOR_SIGMA);
  }
  return block_sum(c, sh.red) + prior_cost(sh, cams);
}

}  // namespace

__global__ void __launch_bounds__(TV_TRI_THREADS) k_tv_triangulate(const TvProb* __restrict__ tab, TvParams prm) {
  const TvProb& p = tab[blockIdx.y];
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= p.k) return;
  const long long i1 = p.matches[2 * row], i2 = p.matches[2 * row + 1];
  double uv[4] = {(double)p.kp1[2 * i1], (double)p.kp1[2 * i1 + 1], (double)p.kp2[2 * i2], (double)p.kp2[2 * i2 + 1]};
  for (int i = 0; i < 4; ++i) p.uv[4 * row + i] = uv[i];
  double X[3] = {0.0, 0.0, 0.0};
  const int ok = p.vmask[row] && triangulate(p.cam0, uv, prm.tri_thr, prm.min_angle, X);
  p.flag[row] = ok;
  for (int i = 0; i < 3; ++i) p.pts[3 * row + i] = X[i];
}

__global__ void __launch_bounds__(TV_THREADS) k_tv_ba(const TvProb* __restrict__ tab, TvParams prm) {
  extern __shared__ double terms[];
  __shared__ TvShared sh;
  __shared__ int s_go;
  const TvProb& p = tab[blockIdx.x];
  const int tid = threadIdx.x;
  int nv = 0, nt = 0, first = INT_MAX;
  for (int row = tid; row < p.k; row += TV_THREADS) {
    nv += p.vmask[row] != 0;
    if (p.flag[row]) ++nt, first = min(first, row);
  }
  nv = (int)block_sum((double)nv, sh.red);
  nt = (int)block_sum((double)nt, sh.red);
  for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_down_sync(0xffffffffu, first, o));
  __syncthreads();
  if ((tid & 31) == 0) sh.red[tid >> 5] = (double)first;
  __syncthreads();
  if (tid == 0) {
    int f = INT_MAX;
    for (int i = 0; i < TV_THREADS / 32; ++i) f = min(f, (int)sh.red[i]);
    sh.first = f;
    TvOut& o = *p.out;
    o.num_verified = nv, o.num_tracks = nt, o.iterations = 0, o.trace_len = 0, o.indeterminate = 0, o.final_error = 0.0;
    o.bundle_adjusted = nv >= prm.min_inliers;  // two_view_estimator.py:412
    s_go = o.bundle_adjusted && nt > 0;
    *p.sel = 0;
    *p.first = f;
    for (int c = 0; c < 2; ++c) {
      sh.cur[c] = p.cam0[c];
      for (int i = 0; i < 3; ++i) sh.cal0[c][i] = p.cam0[c].cal[i];
    }
    if (f < p.k)
      for (int i = 0; i < 3; ++i) sh.pt0[i] = p.anchor[i] = p.pts[3 * f + i];
  }
  __syncthreads();
  if (!s_go) {
    if (tid == 0) p.cams[0] = sh.cur[0], p.cams[1] = sh.cur[1];
    return;
  }
  int sel = 0;
  double lam = LM_LAMBDA0, nw = full_cost(p, p.pts, sh.cur, sh);
  int its = 0, ntrace = 0;
  if (tid == 0) p.trace[ntrace] = nw;
  ++ntrace;
  if (nw > 0.0) {
    for (;;) {
      const double cur = nw;
      for (;;) {  // tryLambda
        double* P = p.pts + (size_t)sel * 3 * p.k;
        double* Q = p.pts + (size_t)(1 - sel) * 3 * p.k;
        if (tid == 0) sh.bad = 0;
        __syncthreads();
        build_system(p, P, sh, terms, lam, false);
        bool solved = !sh.bad;
        if (solved && tid < 32) {
          const bool ok = warp_chol18(sh, 0.0);
          if (tid == 0) {
            if (ok) {
              for (int a = 0; a < 18; ++a) sh.dc[a] = -sh.b[a];
              chol_solve(&sh.S[0][0], 18, 19, sh.dc);
              for (int c = 0; c < 2; ++c) {
                sh.cand[c] = sh.cur[c];
                retract_pose(sh.cand[c].R, sh.cand[c].t, sh.dc + 9 * c);
                for (int i = 0; i < 3; ++i) sh.cand[c].cal[i] += sh.dc[9 * c + 6 + i];
              }
            } else {
              sh.bad = 1;
            }
          }
        }
        __syncthreads();
        solved = !sh.bad;
        bool success = false, stop = false;
        double e_new = 0.0;
        if (solved) {  // Pass B: back-substitution, linearised decrease, cost at the candidate
          double lin = 0.0, old = 0.0, cn = 0.0;
          for (int row = tid; row < p.k; row += TV_THREADS) {
            if (!p.flag[row]) continue;
            TrackLin t;
            const double* X = P + 3 * row;
            const bool fst = row == sh.first;
            track_lin(sh.cur, p.uv + 4 * row, X, t);
            double H[9], g[3];
            point_block(t, fst, X, sh.pt0, lam, H, g);
            for (int c = 0; c < 2; ++c)  // g += Hpc dc
              for (int m = 0; m < 2; ++m) {
                double jd = 0.0;
                for (int j = 0; j < 9; ++j) jd += t.Jc[c][9 * m + j] * sh.dc[9 * c + j];
                for (int i = 0; i < 3; ++i) g[i] += t.w[c] * t.Jp[c][3 * m + i] * jd;
              }
            chol(H, 3, 3);
            double dp[3] = {-g[0], -g[1], -g[2]};
            chol_solve(H, 3, 3, dp);
            for (int c = 0; c < 2; ++c)
              for (int m = 0; m < 2; ++m) {
                double jd = t.Jp[c][3 * m] * dp[0] + t.Jp[c][3 * m + 1] * dp[1] + t.Jp[c][3 * m + 2] * dp[2];
                for (int j = 0; j < 9; ++j) jd += t.Jc[c][9 * m + j] * sh.dc[9 * c + j];
                const double r = t.r[2 * c + m];
                lin -= t.w[c] * (r * jd + 0.5 * jd * jd);
                old += 0.5 * t.w[c] * r * r;
              }
            double Xn[3];
            for (int i = 0; i < 3; ++i) Xn[i] = X[i] + dp[i], Q[3 * row + i] = Xn[i];
            cn += track_cost(sh.cand, p.uv + 4 * row, Xn);
            if (fst)
              for (int i = 0; i < 3; ++i) {
                const double e = (X[i] - sh.pt0[i]) / POINT_PRIOR_SIGMA, jd = dp[i] / POINT_PRIOR_SIGMA;
                const double en = (Xn[i] - sh.pt0[i]) / POINT_PRIOR_SIGMA;
                lin -= e * jd + 0.5 * jd * jd, old += 0.5 * e * e, cn += 0.5 * en * en;
              }
          }
          lin = block_sum(lin, sh.red);
          old = block_sum(old, sh.red);
          cn = block_sum(cn, sh.red);
          {  // the camera priors' share
            double xi[6];
            se3_log(sh.cur[0].R, sh.cur[0].t, xi);
            for (int i = 0; i < 6; ++i) {
              const double e = xi[i] / POSE_PRIOR_SIGMA, jd = sh.dc[i] / POSE_PRIOR_SIGMA;
              lin -= e * jd + 0.5 * jd * jd, old += 0.5 * e * e;
            }
            for (int c = 0; c < 2; ++c)
              for (int i = 0; i < 3; ++i) {
                const double e = (sh.cur[c].cal[i] - sh.cal0[c][i]) / CAL_PRIOR_SIGMA, jd = sh.dc[9 * c + 6 + i] / CAL_PRIOR_SIGMA;
                lin -= e * jd + 0.5 * jd * jd, old += 0.5 * e * e;
              }
            cn += prior_cost(sh, sh.cand);
          }
          e_new = cn;
          lm_trial(lin, old, cur, e_new, success, stop);
        }
        __syncthreads();
        if (success) {
          if (tid == 0) sh.cur[0] = sh.cand[0], sh.cur[1] = sh.cand[1];
          sel = 1 - sel, lam /= LM_FACTOR, ++its, nw = e_new;
          __syncthreads();
          break;
        }
        if (stop) break;
        lam *= LM_FACTOR;
        if (lam >= LM_LAMBDA_MAX) break;
      }
      if (tid == 0) p.trace[ntrace] = nw;
      ++ntrace;
      if (!lm_continue(its, prm.max_iters, cur, nw, LM_ABS_TOL)) break;
    }
  }
  if (tid == 0) {
    *p.sel = sel;
    p.cams[0] = sh.cur[0], p.cams[1] = sh.cur[1];
    p.out->iterations = its, p.out->trace_len = ntrace, p.out->final_error = nw;
  }
}

__global__ void __launch_bounds__(TV_THREADS) k_tv_finish(const TvProb* __restrict__ tab, TvParams prm) {
  extern __shared__ double terms[];
  __shared__ TvShared sh;
  __shared__ int s_warp[TV_THREADS / 32];
  const TvProb& p = tab[blockIdx.x];
  TvOut& o = *p.out;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mode_ba = o.bundle_adjusted, lm = mode_ba && o.num_tracks > 0;
  const double* P = p.pts + (size_t)(*p.sel) * 3 * p.k;
  if (tid == 0) {
    sh.cur[0] = p.cams[0], sh.cur[1] = p.cams[1];
    for (int c = 0; c < 2; ++c)
      for (int i = 0; i < 3; ++i) sh.cal0[c][i] = p.cam0[c].cal[i];
    sh.first = *p.first;
    if (lm)
      for (int i = 0; i < 3; ++i) sh.pt0[i] = p.anchor[i];
    sh.bad = 0;
  }
  __syncthreads();
  bool indeterminate = false;
  if (lm) {
    build_system(p, P, sh, terms, 0.0, true);
    if (tid < 32) {
      const bool ok = !sh.bad && warp_chol18(sh, INDETERMINATE_PIVOT);
      if (tid == 0) sh.bad = !ok;
    }
    __syncthreads();
    indeterminate = sh.bad;
  }
  // the rows that survive: verified rows (no BA), or tracks whose reprojection errors are all below the threshold
  int base = 0;
  for (int r0 = 0; r0 < p.k; r0 += TV_THREADS) {
    const int row = r0 + tid;
    int keep = 0;
    if (row < p.k) {
      if (!mode_ba) {
        keep = p.vmask[row] != 0;
      } else if (!indeterminate && p.flag[row]) {
        keep = 1;
        for (int c = 0; c < 2; ++c) {
          double pr[2];
          const double* uv = p.uv + 4 * row + 2 * c;
          const double z = project(sh.cur[c].R, sh.cur[c].t, sh.cur[c].cal, P + 3 * row, pr, nullptr, nullptr);
          const double e = sqrt((pr[0] - uv[0]) * (pr[0] - uv[0]) + (pr[1] - uv[1]) * (pr[1] - uv[1]));
          if (!(z > 0.0 && e < prm.ba_thr)) keep = 0;
        }
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    off += __popc(bal & ((1u << lane) - 1u));
    int tot = 0;
    for (int w = 0; w < TV_THREADS / 32; ++w) tot += s_warp[w];
    if (row < p.k) {
      if (p.out_mask) p.out_mask[row] = (uint8_t)keep;
      if (keep && p.out_rows) p.out_rows[2 * off] = p.matches[2 * row], p.out_rows[2 * off + 1] = p.matches[2 * row + 1];
    }
    base += tot;
    __syncthreads();
  }
  if (tid == 0) {
    o.indeterminate = indeterminate;
    const double ratio = p.k > 0 ? (double)o.num_verified / (double)p.k : 0.0;
    int n = base;
    bool ok = !indeterminate;
    if (lm && ok && n > 0) {  // wTi2.between(wTi1)
      const Cam& a = sh.cur[0];
      const Cam& b = sh.cur[1];
      double d[3] = {a.t[0] - b.t[0], a.t[1] - b.t[1], a.t[2] - b.t[2]}, nn = 0.0;
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) o.R[i * 3 + j] = b.R[i] * a.R[j] + b.R[3 + i] * a.R[3 + j] + b.R[6 + i] * a.R[6 + j];
        o.t[i] = b.R[i] * d[0] + b.R[3 + i] * d[1] + b.R[6 + i] * d[2];
        nn += o.t[i] * o.t[i];
      }
      nn = sqrt(nn);
      for (int i = 0; i < 3; ++i) o.t[i] /= nn;
    } else {
      for (int i = 0; i < 9; ++i) o.R[i] = p.R0[i];
      for (int i = 0; i < 3; ++i) o.t[i] = p.t0[i];
    }
    if (ratio < prm.min_ratio || (n > 0 && n < prm.min_inliers)) ok = false;  // InlierSupportProcessor
    o.status = ok ? 0 : 1;
    o.num_rows = ok ? n : 0;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct TwoViewState {
  DevBuf rows, tab, out;
  HostBuf htab, hout;
};

void tv_destroy(b2_context* ctx) {
  delete ctx->tv;
  ctx->tv = nullptr;
}

static size_t tv_row_bytes() { return 4 * 8 + 6 * 8 + 4; }
static size_t tv_problem_bytes(const b2_twoview_problem& q, const b2_twoview_params& prm) {
  return (size_t)q.k * tv_row_bytes() + (size_t)(prm.max_iters + 2) * 8 + 2 * sizeof(Cam) + 64 + sizeof(TvOut) + sizeof(TvProb);
}

static int tv_plan(const b2_twoview_problem* problems, int n, const b2_twoview_params& prm, size_t budget, int* first) {
  int count = 0;
  size_t used = 0;
  first[0] = 0;
  for (int i = 0; i < n; ++i) {
    const size_t b = tv_problem_bytes(problems[i], prm);
    if (i > first[count] && used + b > budget) first[++count] = i, used = 0;
    used += b;
  }
  if (n > 0) ++count;
  first[count] = n;
  return count;
}

static int tv_check(b2_context* ctx, const b2_twoview_problem* problems, int n, const b2_twoview_params* prm) {
  if (!prm) return b2_fail(ctx, B2_ERR_ARG, "twoview: params is NULL");
  if (prm->max_iters < 0 || prm->max_iters > 10000) return b2_fail(ctx, B2_ERR_ARG, "twoview: max_iters must be in 0..10000");
  if (!(prm->ba_reproj_error_threshold > 0.0)) return b2_fail(ctx, B2_ERR_ARG, "twoview: ba_reproj_error_threshold must be > 0");
  for (int i = 0; i < n; ++i) {
    const b2_twoview_problem& p = problems[i];
    const std::string at = "twoview problem " + std::to_string(i) + ": ";
    if (p.k < 0) return b2_fail(ctx, B2_ERR_ARG, at + "k < 0");
    if (p.k > 0 && (!p.kp1 || !p.kp2 || !p.matches || !p.mask)) return b2_fail(ctx, B2_ERR_ARG, at + "no points / matches / mask");
    if (!(p.cal1[0] > 0.0 && p.cal2[0] > 0.0)) return b2_fail(ctx, B2_ERR_ARG, at + "focal length must be > 0");
  }
  return B2_OK;
}

static int tv_run_sub(b2_context* ctx, const b2_twoview_problem* q, int L, const b2_twoview_params& prm, b2_twoview_result* res,
                      cudaStream_t st, double* trace_out) {
  TwoViewState* s = ctx->tv;
  size_t rows = 0;
  int max_k = 1;
  for (int i = 0; i < L; ++i) rows += (size_t)q[i].k, max_k = max(max_k, q[i].k);
  const size_t tr = (size_t)prm.max_iters + 2;
  const size_t row_bytes = rows * tv_row_bytes() + (size_t)L * (tr * 8 + 2 * sizeof(Cam) + 128 + 10 * 16) + 256;
  B2_CUDA(ctx, s->rows.ensure(row_bytes));
  B2_CUDA(ctx, s->tab.ensure((size_t)L * sizeof(TvProb)));
  B2_CUDA(ctx, s->out.ensure((size_t)L * sizeof(TvOut)));
  B2_CUDA(ctx, s->htab.ensure((size_t)L * sizeof(TvProb)));
  B2_CUDA(ctx, s->hout.ensure((size_t)L * sizeof(TvOut)));
  TvProb* ht = s->htab.as<TvProb>();
  TvOut* dout = s->out.as<TvOut>();
  char* w = s->rows.as<char>();
  auto take = [&](size_t bytes) {
    char* r = w;
    w += (bytes + 15) / 16 * 16;
    return r;
  };
  for (int i = 0; i < L; ++i) {
    const b2_twoview_problem& pq = q[i];
    TvProb& t = ht[i];
    memset(&t, 0, sizeof(t));
    t.kp1 = pq.kp1, t.kp2 = pq.kp2, t.matches = reinterpret_cast<const long long*>(pq.matches), t.vmask = pq.mask;
    t.out_mask = pq.out_mask, t.out_rows = reinterpret_cast<long long*>(pq.out_rows), t.k = pq.k;
    // Pose3() with K1, Pose3(R, t)^-1 = (R^T, -R^T t) with K2 (two_view_estimator.py:241-252)
    Cam c0{}, c1{};
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) c0.R[a * 3 + b] = a == b, c1.R[a * 3 + b] = pq.R[b * 3 + a];
    for (int a = 0; a < 3; ++a) c1.t[a] = -(pq.R[a] * pq.t[0] + pq.R[3 + a] * pq.t[1] + pq.R[6 + a] * pq.t[2]);
    const double* cals[2] = {pq.cal1, pq.cal2};
    Cam* cs[2] = {&c0, &c1};
    for (int c = 0; c < 2; ++c) {
      cs[c]->cal[0] = cals[c][0], cs[c]->cal[1] = cs[c]->cal[2] = 0.0, cs[c]->cal[3] = cals[c][1], cs[c]->cal[4] = cals[c][2];
    }
    t.cam0[0] = c0, t.cam0[1] = c1;
    memcpy(t.R0, pq.R, 72), memcpy(t.t0, pq.t, 24);
    t.uv = reinterpret_cast<double*>(take((size_t)pq.k * 32));
    t.pts = reinterpret_cast<double*>(take((size_t)pq.k * 48));
    t.flag = reinterpret_cast<int*>(take((size_t)pq.k * 4));
    t.cams = reinterpret_cast<Cam*>(take(2 * sizeof(Cam)));
    t.sel = reinterpret_cast<int*>(take(4));
    t.first = reinterpret_cast<int*>(take(4));
    t.anchor = reinterpret_cast<double*>(take(24));
    t.trace = reinterpret_cast<double*>(take(tr * 8));
    t.out = dout + i;
  }
  TvParams kp{prm.max_iters, prm.min_num_inliers, prm.min_inlier_ratio, prm.ba_reproj_error_threshold,
              prm.tri_reproj_error_threshold, prm.min_triangulation_angle};
  TvProb* dt = s->tab.as<TvProb>();
  B2_CUDA(ctx, cudaMemcpyAsync(dt, ht, (size_t)L * sizeof(TvProb), cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, k_tv_triangulate, dim3(cdiv(max_k, TV_TRI_THREADS), L), TV_TRI_THREADS, 0, st, dt, kp);
  B2_CHECK_LAUNCH(ctx);
  const size_t smem = (size_t)TV_TILE * TV_TERMS * 8;
  B2_CUDA(ctx, cudaFuncSetAttribute(k_tv_ba, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_tv_finish, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2_LAUNCH(ctx, k_tv_ba, dim3(L), TV_THREADS, smem, st, dt, kp);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_tv_finish, dim3(L), TV_THREADS, smem, st, dt, kp);
  B2_CHECK_LAUNCH(ctx);
  TvOut* ho = s->hout.as<TvOut>();
  B2_CUDA(ctx, cudaMemcpyAsync(ho, dout, (size_t)L * sizeof(TvOut), cudaMemcpyDeviceToHost, st));
  if (trace_out)
    for (int i = 0; i < L; ++i)
      B2_CUDA(ctx, cudaMemcpyAsync(trace_out + (size_t)i * tr, ht[i].trace, tr * 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (int i = 0; i < L; ++i) {
    const TvOut& o = ho[i];
    b2_twoview_result& r = res[i];
    memset(&r, 0, sizeof(r));
    r.status = o.status, r.num_rows = o.num_rows, r.num_verified = o.num_verified, r.num_tracks = o.num_tracks;
    r.iterations = o.iterations, r.bundle_adjusted = o.bundle_adjusted, r.indeterminate = o.indeterminate;
    r.trace_len = o.trace_len, r.final_error = o.final_error;
    memcpy(r.R, o.R, 72), memcpy(r.t, o.t, 24);
  }
  return B2_OK;
}

static int tv_run(b2_context* ctx, const b2_twoview_problem* problems, int n, const b2_twoview_params* params,
                  b2_twoview_result* results, void* stream, double* trace) {
  if (!ctx || n < 0 || (n > 0 && (!problems || !results))) return B2_ERR_ARG;
  if (int rc = tv_check(ctx, problems, n, params)) return rc;
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->tv) ctx->tv = new TwoViewState();
  std::vector<int> first(n + 1);
  const int subs = tv_plan(problems, n, *params, (size_t)ctx->rs_workspace_mb << 20, first.data());
  cudaStream_t st = stream ? (cudaStream_t)stream : cudaStreamLegacy;
  const size_t tr = (size_t)params->max_iters + 2;
  for (int b = 0; b < subs; ++b)
    if (int rc = tv_run_sub(ctx, problems + first[b], first[b + 1] - first[b], *params, results + first[b], st,
                            trace ? trace + (size_t)first[b] * tr : nullptr))
      return rc;
  return B2_OK;
}

extern "C" size_t b2_twoview_ba_workspace_bytes(const b2_twoview_problem* problem, const b2_twoview_params* params) {
  if (!problem || !params || problem->k < 0 || params->max_iters < 0) return 0;
  return tv_problem_bytes(*problem, *params);
}

extern "C" int b2_twoview_ba_plan(const b2_twoview_problem* problems, int n, const b2_twoview_params* params, size_t budget_bytes,
                                  int* out_first) {
  if (n < 0 || !out_first || !params || params->max_iters < 0 || (n > 0 && !problems)) return B2_ERR_ARG;
  for (int i = 0; i < n; ++i)
    if (problems[i].k < 0) return B2_ERR_ARG;
  return tv_plan(problems, n, *params, budget_bytes, out_first);
}

extern "C" int b2_twoview_ba_batched_dev(b2_context* ctx, const b2_twoview_problem* problems, int n, const b2_twoview_params* params,
                                         b2_twoview_result* results, void* stream) {
  return tv_run(ctx, problems, n, params, results, stream, nullptr);
}

extern "C" int b2_debug_twoview_ba_trace_host(b2_context* ctx, const b2_twoview_problem* problems, int n,
                                              const b2_twoview_params* params, b2_twoview_result* results, double* out_trace,
                                              void* stream) {
  if (!out_trace) return b2_fail(ctx, B2_ERR_ARG, "twoview trace: out_trace is NULL");
  return tv_run(ctx, problems, n, params, results, stream, out_trace);
}
