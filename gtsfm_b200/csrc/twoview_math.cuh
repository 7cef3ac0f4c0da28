// fp64 building blocks of the two-view refinement, usable from host and device (the host build is the unit-test harness in
// tests/cpp/test_twoview_math.cpp; the device build is twoview_ba.cu).  oracle/twoview_ba_ref.py states the same maths in
// NumPy.
//
// What they restate: gtsam's triangulatePoint3(cameras, measurements, rank_tol=1e-9, optimize=True) for two
// PinholeCamera<Cal3Bundler>, the projection and Jacobians of GeneralSFMFactor2<Cal3Bundler>, Pose3's retraction (gtsam's
// default build sets GTSAM_POSE3_EXPMAP, so retract is the full SE(3) exponential, compose(Expmap(xi)) with xi = [w, v]),
// the Block Huber reweighting of noiseModel::Robust, and the Levenberg-Marquardt step policy of gtsam's
// LevenbergMarquardtOptimizer (tryLambda with the fixed lambda factor).  The global bundle adjustment (global_ba.cu) uses
// the same projection, retraction, Huber and LM decision over N cameras.
#pragma once
#include <float.h>
#include <math.h>

#ifdef __CUDACC__
#define TV_HD __host__ __device__ __forceinline__
#else
#define TV_HD inline
#endif

namespace tvmath {

constexpr double HUBER_K = 1.345;
constexpr double POSE_PRIOR_SIGMA = 0.1;
constexpr double POINT_PRIOR_SIGMA = 0.1;
constexpr double CAL_PRIOR_SIGMA = 1e-5;
constexpr double DLT_RANK_TOL = 1e-9;
// gtsam.LevenbergMarquardtParams() defaults (relativeErrorTol, absoluteErrorTol, lambdaUpperBound, minModelFidelity)
constexpr double LM_LAMBDA0 = 1e-5, LM_FACTOR = 10.0, LM_LAMBDA_MAX = 1e5, LM_REL_TOL = 1e-5, LM_ABS_TOL = 1e-5;
constexpr double LM_MIN_FIDELITY = 1e-3;
// triangulation.h optimize(): lambdaInitial 1, absoluteErrorTol 1 (the rest as above)
constexpr double TRI_LAMBDA0 = 1.0, TRI_ABS_TOL = 1.0;
constexpr int TRI_MAX_ITERS = 100;
// indeterminate system: a Cholesky pivot of the undamped Hessian at or below this fraction of the unknown's diagonal
constexpr double INDETERMINATE_PIVOT = 1e-10;

// noiseModel::mEstimator::Huber(k) on a whitened error norm e: the IRLS weight and the loss (0.5 e^2 inside the basin)
TV_HD double huber_weight(double e, double k) { return e <= k ? 1.0 : k / e; }
TV_HD double huber_loss(double e, double k) { return e <= k ? 0.5 * e * e : k * (e - 0.5 * k); }
TV_HD double huber_weight(double e) { return huber_weight(e, HUBER_K); }
TV_HD double huber_loss(double e) { return huber_loss(e, HUBER_K); }

// One tryLambda decision of gtsam's LevenbergMarquardtOptimizer: `lin` the linearised cost decrease of the step, `old` the
// undamped linearised cost at dx = 0, `cur` the cost before and `e_new` the cost after the step (read only when lin >= 0).
// success: accept the step (lambda /= 10); otherwise stop: leave the lambda loop without a step, else lambda *= 10.
TV_HD void lm_trial(double lin, double old, double cur, double e_new, bool& success, bool& stop) {
  success = stop = false;
  if (!(lin >= 0.0)) return;
  const double dc = cur - e_new;
  success = lin > DBL_EPSILON * old ? dc / lin > LM_MIN_FIDELITY : true;
  stop = fabs(dc) < LM_REL_TOL * cur;
}
// After an outer iteration (cost cur before, nw after, its successful iterations so far): whether LM goes on
// (checkConvergence with the relative and the given absolute tolerance, maxIterations, a finite error)
TV_HD bool lm_continue(int its, int max_iters, double cur, double nw, double abs_tol) {
  const double dec = cur - nw;
  const bool conv = dec / cur <= LM_REL_TOL || dec <= abs_tol || nw <= 0.0;
  return its < max_iters && !conv && isfinite(cur);
}

TV_HD void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
TV_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1], c[1] = a[2] * b[0] - a[0] * b[2], c[2] = a[0] * b[1] - a[1] * b[0];
}

// Rot3::Expmap (first order below theta^2 = DBL_EPSILON, as gtsam's SO3 ExpmapFunctor)
TV_HD void so3_exp(const double* w, double* R) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double a = 1.0, b = 0.0;
  if (th2 > DBL_EPSILON) {
    const double th = sqrt(th2);
    a = sin(th) / th, b = (1.0 - cos(th)) / th2;
  }
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double WW[9];
  mat3_mul(W, W, WW);
  for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0 ? 1.0 : 0.0) + a * W[i] + b * WW[i];
}

// SO3::Logmap away from theta = pi (gtsam's normal and near-zero branches)
TV_HD void so3_log(const double* R, double* w) {
  const double tr = R[0] + R[4] + R[8], tr3 = tr - 3.0;
  double mag;
  if (tr3 < -1e-6) {
    const double c = fmin(1.0, fmax(-1.0, 0.5 * (tr - 1.0)));
    const double th = acos(c);
    mag = th / (2.0 * sin(th));
  } else {
    mag = 0.5 - tr3 / 12.0 + tr3 * tr3 / 60.0;
  }
  w[0] = mag * (R[7] - R[5]), w[1] = mag * (R[2] - R[6]), w[2] = mag * (R[3] - R[1]);
}

// V(w) v: the translation of Pose3::Expmap([w, v]) (series below theta = 1e-4)
TV_HD void se3_v(const double* w, const double* v, double* t) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double wv[3], wwv[3], a, b;
  cross3(w, v, wv);
  cross3(w, wv, wwv);
  if (th2 < 1e-8) {
    a = 0.5 - th2 / 24.0, b = 1.0 / 6.0 - th2 / 120.0;
  } else {
    const double th = sqrt(th2);
    a = (1.0 - cos(th)) / th2, b = (th - sin(th)) / (th2 * th);
  }
  for (int i = 0; i < 3; ++i) t[i] = v[i] + a * wv[i] + b * wwv[i];
}

// Pose3::Logmap -> [w, u] (Agrawal06iros eq. 14 as gtsam writes it)
TV_HD void se3_log(const double* R, const double* t, double* xi) {
  so3_log(R, xi);
  const double th = sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]);
  if (th < 1e-10) {
    xi[3] = t[0], xi[4] = t[1], xi[5] = t[2];
    return;
  }
  const double n[3] = {xi[0] / th, xi[1] / th, xi[2] / th};
  double WT[3], WWT[3];
  cross3(n, t, WT);
  cross3(n, WT, WWT);
  const double c = 1.0 - th / (2.0 * tan(0.5 * th));
  for (int i = 0; i < 3; ++i) xi[3 + i] = t[i] - (0.5 * th) * WT[i] + c * WWT[i];
}

// Pose3::retract(d) = compose(Expmap(d)): R <- R Exp(w), t <- t + R V(w) v
TV_HD void retract_pose(double* R, double* t, const double* d) {
  double E[9], Rn[9], tv[3];
  so3_exp(d, E);
  mat3_mul(R, E, Rn);
  se3_v(d, d + 3, tv);
  for (int i = 0; i < 3; ++i) t[i] += R[i * 3] * tv[0] + R[i * 3 + 1] * tv[1] + R[i * 3 + 2] * tv[2];
  for (int i = 0; i < 9; ++i) R[i] = Rn[i];
}

// PinholeCamera<Cal3Bundler>(Pose3(R, t), cal = {f, k1, k2, u0, v0}).project(p) -> uv; returns the depth.  Jacobians (any
// may be NULL) row-major: Jc [2][9] = pose [w, v] (right perturbation) then (f, k1, k2); Jp [2][3] the point.
TV_HD double project(const double* R, const double* t, const double* cal, const double* p, double* uv, double* Jc,
                     double* Jp) {
  const double d[3] = {p[0] - t[0], p[1] - t[1], p[2] - t[2]};
  double pc[3];
  for (int i = 0; i < 3; ++i) pc[i] = R[i] * d[0] + R[3 + i] * d[1] + R[6 + i] * d[2];  // R^T (p - t)
  const double z = pc[2], iz = 1.0 / z, x = pc[0] * iz, y = pc[1] * iz;
  const double f = cal[0], k1 = cal[1], k2 = cal[2];
  const double r = x * x + y * y, g = 1.0 + k1 * r + k2 * r * r;
  uv[0] = cal[3] + f * g * x, uv[1] = cal[4] + f * g * y;
  if (!Jc && !Jp) return z;
  const double dg = 2.0 * (k1 + 2.0 * k2 * r);
  const double A00 = f * (g + dg * x * x), A01 = f * dg * x * y, A11 = f * (g + dg * y * y);
  // D = Duv/dpn * Dpn/dpc (2 x 3)
  const double D[6] = {A00 * iz, A01 * iz, -(A00 * x + A01 * y) * iz, A01 * iz, A11 * iz, -(A01 * x + A11 * y) * iz};
  if (Jc) {
    for (int k = 0; k < 2; ++k) {
      const double* Dk = D + 3 * k;
      // d pc / d w = [pc]x under pose * Exp([w, v]), d pc / d v = -I
      Jc[9 * k + 0] = Dk[1] * pc[2] - Dk[2] * pc[1];
      Jc[9 * k + 1] = Dk[2] * pc[0] - Dk[0] * pc[2];
      Jc[9 * k + 2] = Dk[0] * pc[1] - Dk[1] * pc[0];
      Jc[9 * k + 3] = -Dk[0], Jc[9 * k + 4] = -Dk[1], Jc[9 * k + 5] = -Dk[2];
      const double q = k == 0 ? x : y;
      Jc[9 * k + 6] = g * q, Jc[9 * k + 7] = f * r * q, Jc[9 * k + 8] = f * r * r * q;
    }
  }
  if (Jp)
    for (int k = 0; k < 2; ++k)
      for (int j = 0; j < 3; ++j) Jp[3 * k + j] = D[3 * k] * R[3 * j] + D[3 * k + 1] * R[3 * j + 1] + D[3 * k + 2] * R[3 * j + 2];
  return z;
}

// In-place Cholesky of an n x n symmetric matrix (lower triangle used, row-major, leading dimension ld) -> false when a
// pivot is not positive (or not finite).
TV_HD bool chol(double* A, int n, int ld) {
  for (int k = 0; k < n; ++k) {
    double p = A[k * ld + k];
    for (int m = 0; m < k; ++m) p -= A[k * ld + m] * A[k * ld + m];
    if (!(p > 0.0) || !isfinite(p)) return false;
    const double l = sqrt(p);
    A[k * ld + k] = l;
    for (int i = k + 1; i < n; ++i) {
      double s = A[i * ld + k];
      for (int m = 0; m < k; ++m) s -= A[i * ld + m] * A[k * ld + m];
      A[i * ld + k] = s / l;
    }
  }
  return true;
}
// Solve L L^T x = b in place (L from chol)
TV_HD void chol_solve(const double* L, int n, int ld, double* b) {
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int m = 0; m < i; ++m) s -= L[i * ld + m] * b[m];
    b[i] = s / L[i * ld + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i];
    for (int m = i + 1; m < n; ++m) s -= L[m * ld + i] * b[m];
    b[i] = s / L[i * ld + i];
  }
}
// Forward substitution only: L y = b in place
TV_HD void chol_fwd(const double* L, int n, int ld, double* b) {
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int m = 0; m < i; ++m) s -= L[i * ld + m] * b[m];
    b[i] = s / L[i * ld + i];
  }
}

// One-sided Jacobi SVD of a 4 x 4 matrix (row-major A, destroyed): singular values s (unsorted) and V (columns).
TV_HD void svd4(double* A, double* s, double* V) {
  for (int i = 0; i < 16; ++i) V[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) {
        double a = 0, b = 0, c = 0;
        for (int i = 0; i < 4; ++i) a += A[i * 4 + p] * A[i * 4 + p], b += A[i * 4 + q] * A[i * 4 + q], c += A[i * 4 + p] * A[i * 4 + q];
        if (fabs(c) <= 1e-300 || fabs(c) <= 1e-17 * sqrt(a * b)) continue;
        off = fmax(off, fabs(c) / sqrt(a * b));
        const double zeta = (b - a) / (2.0 * c);
        const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
        for (int i = 0; i < 4; ++i) {
          const double x = A[i * 4 + p], y = A[i * 4 + q];
          A[i * 4 + p] = cs * x - sn * y, A[i * 4 + q] = sn * x + cs * y;
          const double vx = V[i * 4 + p], vy = V[i * 4 + q];
          V[i * 4 + p] = cs * vx - sn * vy, V[i * 4 + q] = sn * vx + cs * vy;
        }
      }
    if (off < 1e-15) break;
  }
  for (int j = 0; j < 4; ++j) {
    double n = 0;
    for (int i = 0; i < 4; ++i) n += A[i * 4 + j] * A[i * 4 + j];
    s[j] = sqrt(n);
  }
}

// camera.cameraProjectionMatrix() of Pose3(R, t) with calibration {f, *, *, u0, v0}: K [R^T | -R^T t]
TV_HD void projection_matrix(const double* R, const double* t, const double* cal, double* P) {
  double M[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) M[i * 4 + j] = R[j * 3 + i];
    M[i * 4 + 3] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
  }
  for (int j = 0; j < 4; ++j) {
    P[j] = cal[0] * M[j] + cal[3] * M[8 + j];
    P[4 + j] = cal[0] * M[4 + j] + cal[4] * M[8 + j];
    P[8 + j] = M[8 + j];
  }
}

// A camera of the two-view problem: Pose3(R, t) (world from camera) and {f, k1, k2, u0, v0}
struct Cam {
  double R[9], t[3], cal[5];
};

// The two rows of the DLT system one view contributes: u P[2] - P[0], v P[2] - P[1]
TV_HD void dlt_rows(const double* P, const double* uv, double* a) {
  for (int j = 0; j < 4; ++j) {
    a[j] = uv[0] * P[8 + j] - P[j];
    a[4 + j] = uv[1] * P[8 + j] - P[4 + j];
  }
}

// The null vector of a 4-column system reduced to 4 x 4 (A, destroyed) -> false when the rank (singular values above
// 1e-9) is below 3 or the point is at infinity
TV_HD bool dlt_solve(double* A, double* X) {
  double s[4], V[16];
  svd4(A, s, V);
  int rank = 0, jmin = 0;
  for (int j = 0; j < 4; ++j) {
    rank += s[j] > DLT_RANK_TOL;
    if (s[j] < s[jmin]) jmin = j;
  }
  if (rank < 3) return false;
  const double w = V[12 + jmin];
  for (int i = 0; i < 3; ++i) X[i] = V[i * 4 + jmin] / w;
  return isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
}

// triangulateDLT on two views
TV_HD bool dlt(const double* P0, const double* P1, const double* uv0, const double* uv1, double* X) {
  double A[16];
  dlt_rows(P0, uv0, A);
  dlt_rows(P1, uv1, A + 8);
  return dlt_solve(A, X);
}

// Folds one row a[4] (destroyed) into the upper-triangular R (row-major 4 x 4) by Givens rotations, so that R^T R gains
// a a^T: R then has the singular values and right singular vectors of every row folded in so far.
TV_HD void qr_fold_row(double* R, double* a) {
  for (int j = 0; j < 4; ++j) {
    if (a[j] == 0.0) continue;
    const double r = hypot(R[j * 4 + j], a[j]), c = R[j * 4 + j] / r, s = a[j] / r;
    R[j * 4 + j] = r;
    a[j] = 0.0;
    for (int k = j + 1; k < 4; ++k) {
      const double x = R[j * 4 + k], y = a[k];
      R[j * 4 + k] = c * x + s * y, a[k] = c * y - s * x;
    }
  }
}

// triangulateDLT on n >= 2 views given by `views` (see refine_point_views).  Two views go through dlt's 4 x 4 system as
// it is; more are reduced to 4 x 4 by a streamed QR of the 2n x 4 system first (same singular values, same null vector).
template <class Views>
TV_HD bool dlt_views(const Views& views, double* X) {
  const int n = views.size();
  double A[16], P[12];
  if (n == 2) {
    for (int k = 0; k < 2; ++k) {
      const Cam& c = views.cam(k);
      projection_matrix(c.R, c.t, c.cal, P);
      dlt_rows(P, views.uv(k), A + 8 * k);
    }
    return dlt_solve(A, X);
  }
  for (int i = 0; i < 16; ++i) A[i] = 0.0;
  for (int k = 0; k < n; ++k) {
    const Cam& c = views.cam(k);
    double a[8];
    projection_matrix(c.R, c.t, c.cal, P);
    dlt_rows(P, views.uv(k), a);
    qr_fold_row(A, a);
    qr_fold_row(A, a + 4);
  }
  return dlt_solve(A, X);
}

// TriangulationFactor residual of a point in one camera, Jacobian J [2][3] (may be NULL); a point behind the camera:
// residual (2f, 2f), zero Jacobian
TV_HD void tri_resid1(const Cam& c, const double* uv, const double* X, double* r, double* J) {
  double pr[2];
  const double z = project(c.R, c.t, c.cal, X, pr, nullptr, J);
  if (!(z > 0.0)) {
    r[0] = r[1] = 2.0 * c.cal[0];
    if (J)
      for (int i = 0; i < 6; ++i) J[i] = 0.0;
  } else {
    r[0] = pr[0] - uv[0], r[1] = pr[1] - uv[1];
  }
}

// TriangulationFactor residuals of a point in both cameras
TV_HD void tri_resid(const Cam* cams, const double* uv, const double* X, double* r, double* J) {
  for (int c = 0; c < 2; ++c) tri_resid1(cams[c], uv + 2 * c, X, r + 2 * c, J ? J + 6 * c : nullptr);
}
TV_HD double tri_cost(const Cam* cams, const double* uv, const double* X) {
  double r[4];
  tri_resid(cams, uv, X, r, nullptr);
  return 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
}

// The two views of the two-view problem, as refine_point_views and dlt_views take views: size(), cam(k), uv(k) and
// cost(X), the triangulation cost 0.5 sum |r|^2
struct TwoViews {
  const Cam* cams;
  const double* uvs;  // {u0, v0, u1, v1}
  TV_HD int size() const { return 2; }
  TV_HD const Cam& cam(int k) const { return cams[k]; }
  TV_HD const double* uv(int k) const { return uvs + 2 * k; }
  TV_HD double cost(const double* X) const { return tri_cost(cams, uvs, X); }
};

// triangulateNonlinear: gtsam's LM (lambda0 1, absolute tolerance 1, 100 iterations) on the point alone, over any number
// of views.  The normal equations and the linearised decrease are accumulated view by view, row by row, in view order
// (nothing is stored per view), so two views sum in the order of the 4-row two-view system.
template <class Views>
TV_HD void refine_point_views(const Views& views, double* X) {
  const int n = views.size();
  double err = views.cost(X);
  if (err <= 0.0) return;
  double lam = TRI_LAMBDA0, nw = err;
  int its = 0;
  for (;;) {
    const double cur = nw;
    for (;;) {
      double H[9] = {0}, g[3] = {0};
      for (int k = 0; k < n; ++k) {
        double r[2], J[6];
        tri_resid1(views.cam(k), views.uv(k), X, r, J);
        for (int m = 0; m < 2; ++m) {
          for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) H[i * 3 + j] += J[m * 3 + i] * J[m * 3 + j];
            g[i] += J[m * 3 + i] * r[m];
          }
        }
      }
      for (int i = 0; i < 3; ++i) H[i * 4] += lam;
      bool success = false, stop = false;
      double Xn[3];
      if (chol(H, 3, 3)) {
        double d[3] = {-g[0], -g[1], -g[2]};
        chol_solve(H, 3, 3, d);
        double lin = 0.0, old = 0.0;
        for (int k = 0; k < n; ++k) {
          double r[2], J[6];
          tri_resid1(views.cam(k), views.uv(k), X, r, J);
          for (int m = 0; m < 2; ++m) {
            const double jd = J[m * 3] * d[0] + J[m * 3 + 1] * d[1] + J[m * 3 + 2] * d[2];
            lin -= r[m] * jd + 0.5 * jd * jd;
            old += 0.5 * r[m] * r[m];
          }
        }
        if (lin >= 0.0) {
          for (int i = 0; i < 3; ++i) Xn[i] = X[i] + d[i];
          lm_trial(lin, old, cur, views.cost(Xn), success, stop);
        }
      }
      if (success) {
        X[0] = Xn[0], X[1] = Xn[1], X[2] = Xn[2];
        lam /= LM_FACTOR, ++its;
        break;
      }
      if (stop) break;
      lam *= LM_FACTOR;
      if (lam >= LM_LAMBDA_MAX) break;
    }
    nw = views.cost(X);
    if (!lm_continue(its, TRI_MAX_ITERS, cur, nw, TRI_ABS_TOL)) return;
  }
}

TV_HD void refine_point(const Cam* cams, const double* uv, double* X) { refine_point_views(TwoViews{cams, uv}, X); }

// Point3dInitializer.triangulate (NO_RANSAC) for one correspondence uv = {u0, v0, u1, v1} -> false when dropped
TV_HD bool triangulate(const Cam* cams, const double* uv, double reproj_thr, double min_angle_deg, double* X) {
  double P0[12], P1[12];
  projection_matrix(cams[0].R, cams[0].t, cams[0].cal, P0);
  projection_matrix(cams[1].R, cams[1].t, cams[1].cal, P1);
  if (!dlt(P0, P1, uv, uv + 2, X)) return false;
  refine_point(cams, uv, X);
  for (int c = 0; c < 2; ++c) {
    double pr[2];
    if (!(project(cams[c].R, cams[c].t, cams[c].cal, X, pr, nullptr, nullptr) > 0.0)) return false;  // cheirality
    const double e = sqrt((pr[0] - uv[2 * c]) * (pr[0] - uv[2 * c]) + (pr[1] - uv[2 * c + 1]) * (pr[1] - uv[2 * c + 1]));
    if (!(e < reproj_thr)) return false;
  }
  double a[3], b[3], ab = 0, aa = 0, bb = 0;
  for (int i = 0; i < 3; ++i) a[i] = X[i] - cams[0].t[i], b[i] = X[i] - cams[1].t[i];
  for (int i = 0; i < 3; ++i) ab += a[i] * b[i], aa += a[i] * a[i], bb += b[i] * b[i];
  const double ang = acos(fmin(1.0, fmax(-1.0, ab / (sqrt(aa) * sqrt(bb))))) * (180.0 / M_PI);
  return !(ang < min_angle_deg);
}

}  // namespace tvmath
