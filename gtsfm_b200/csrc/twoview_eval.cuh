// fp64 maths of the two-view reports' ground-truth metrics, usable from host and device (the host build is the unit-test
// harness in tests/cpp/test_twoview_eval.cpp; the device build is twoview_eval.cu).  oracle/twoview_report_ref.py states
// the same maths in NumPy, in the same operation order.
//
// What they restate (GTSfM):
//   gt_relative        Pose3 wTi2.between(wTi1)                         two_view_estimator.py:705-731, utils/metrics.py:91
//   gt_fundamental     EssentialMatrix(R, Unit3(t)).matrix() = [u]x R, then F = K2^-T E K1^-1
//                                                                     utils/metrics.py:119-120, utils/verification.py:115
//   sampson_sq         compute_epipolar_distances_sq_sampson            utils/verification.py:172-216
//   rotation_angle_deg norm of the rotation vector of Ra.between(Rb)    utils/geometry_comparisons.py:137-159
//   unit_angle_deg     arccos(clip(dot(a, b), -1, 1))                    utils/geometry_comparisons.py:162-180
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define TE_HD __host__ __device__ __forceinline__
#else
#define TE_HD inline
#endif

namespace tveval {

constexpr double RAD2DEG = 57.29577951308232;  // np.rad2deg: x * (180 / pi)

// wTi = (R, t) with R row-major world-from-camera and t the camera centre: i2Ti1 = wTi2^-1 wTi1 -> (R, t)
TE_HD void gt_relative(const double* R1, const double* t1, const double* R2, const double* t2, double* R, double* t) {
  const double d[3] = {t1[0] - t2[0], t1[1] - t2[1], t1[2] - t2[2]};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = R2[i] * R1[j] + R2[3 + i] * R1[3 + j] + R2[6 + i] * R1[6 + j];
    t[i] = R2[i] * d[0] + R2[3 + i] * d[1] + R2[6 + i] * d[2];
  }
}

// F = K2^-T [t / |t|]x R K1^-1, K = [[f, 0, u0], [0, f, v0], [0, 0, 1]] (Cal3Bundler without distortion: cal = f, u0, v0)
TE_HD void gt_fundamental(const double* R, const double* t, const double* cal1, const double* cal2, double* F) {
  const double n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  const double u[3] = {t[0] / n, t[1] / n, t[2] / n};
  const double S[9] = {0.0, -u[2], u[1], u[2], 0.0, -u[0], -u[1], u[0], 0.0};
  double E[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[i * 3 + j] = S[i * 3] * R[j] + S[i * 3 + 1] * R[3 + j] + S[i * 3 + 2] * R[6 + j];
  // K^-1 = [[1/f, 0, -u0/f], [0, 1/f, -v0/f], [0, 0, 1]]
  const double a1 = 1.0 / cal1[0], b1 = -cal1[1] / cal1[0], c1 = -cal1[2] / cal1[0];
  const double a2 = 1.0 / cal2[0], b2 = -cal2[1] / cal2[0], c2 = -cal2[2] / cal2[0];
  double G[9];  // K2^-T E: row 0 = a2 E0, row 1 = a2 E1, row 2 = b2 E0 + c2 E1 + E2
  for (int j = 0; j < 3; ++j) {
    G[j] = a2 * E[j];
    G[3 + j] = a2 * E[3 + j];
    G[6 + j] = b2 * E[j] + c2 * E[3 + j] + E[6 + j];
  }
  for (int i = 0; i < 3; ++i) {  // (K2^-T E) K1^-1: col 0 = a1 G0, col 1 = a1 G1, col 2 = b1 G0 + c1 G1 + G2
    F[i * 3] = G[i * 3] * a1;
    F[i * 3 + 1] = G[i * 3 + 1] * a1;
    F[i * 3 + 2] = G[i * 3] * b1 + G[i * 3 + 1] * c1 + G[i * 3 + 2];
  }
}

// squared Sampson distance of (x1, y1) <-> (x2, y2) under i2Fi1: (x1^T l1)^2 / (|l1.xy|^2 + |l2.xy|^2), l2 = F x1, l1 = F^T x2
TE_HD double sampson_sq(const double* F, double x1, double y1, double x2, double y2) {
  const double l2x = x1 * F[0] + y1 * F[1] + F[2], l2y = x1 * F[3] + y1 * F[4] + F[5];
  const double l1x = x2 * F[0] + y2 * F[3] + F[6], l1y = x2 * F[1] + y2 * F[4] + F[7], l1z = x2 * F[2] + y2 * F[5] + F[8];
  const double d = x1 * l1x + y1 * l1y + l1z;
  return (d * d) / ((l1x * l1x + l1y * l1y) + (l2x * l2x + l2y * l2y));
}

// the angle of Ra^T Rb in degrees: atan2(|axis part|, cos part) keeps full accuracy near 0 and near 180 degrees, where
// acos((tr - 1) / 2) alone loses half the digits
TE_HD double rotation_angle_deg(const double* Ra, const double* Rb) {
  double M[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i * 3 + j] = Ra[i] * Rb[j] + Ra[3 + i] * Rb[3 + j] + Ra[6 + i] * Rb[6 + j];
  const double x = M[7] - M[5], y = M[2] - M[6], z = M[3] - M[1];
  const double s = 0.5 * sqrt(x * x + y * y + z * z), c = 0.5 * (M[0] + M[4] + M[8] - 1.0);
  return atan2(s, c) * RAD2DEG;
}

// angle between the directions of a and b (each normalised first, as Unit3 does), in degrees
TE_HD double unit_angle_deg(const double* a, const double* b) {
  const double na = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]), nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  double d = (a[0] / na) * (b[0] / nb) + (a[1] / na) * (b[1] / nb) + (a[2] / na) * (b[2] / nb);
  d = d < -1.0 ? -1.0 : (d > 1.0 ? 1.0 : d);
  return acos(d) * RAD2DEG;
}

}  // namespace tveval
