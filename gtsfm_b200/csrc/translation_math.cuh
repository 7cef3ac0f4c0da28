// fp64 factor maths of gtsam's TranslationRecovery as 1DSfM runs it (averaging_1dsfm.py:__run_averaging), usable from host
// and device: the device build is translation_recovery.cu.  oracle/translation_recovery_ref.py states the same in NumPy.
//
//   TranslationFactor(a, b, m)   error normalize(x_b - x_a) - m, whitened by 1 / sigma, Jacobians -N (a) and +N (b) with
//                                N = (|d|^2 I - d d^T) / |d|^3, gtsam's normalize() derivative
//   Robust(Huber(k))             the block reweighting: weight and loss on the norm of the whole whitened 3-vector
//   addPrior                     PriorFactor<Point3>(a_0, 0, Isotropic(3, prior_sigma)), not robust (prior 0), and
//                                PriorFactor<Point3>(b_0, scale m_0, the edges' own model) (prior 1)
// Every prior is isotropic with an identity Jacobian, so its block in the normal equations is h I.
#pragma once
#include "twoview_math.cuh"

namespace trmath {

// the whitened error's loss and IRLS weight: Huber(k), or the Gaussian model when k == 0
TV_HD double loss(double e, double k) { return k > 0.0 ? tvmath::huber_loss(e, k) : 0.5 * e * e; }
TV_HD double weight(double e, double k) { return k > 0.0 ? tvmath::huber_weight(e, k) : 1.0; }
TV_HD double norm3(const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// gtsam's normalize(p, H): p / |p| and, when H is given, its derivative (row-major)
TV_HD void normalize(const double* p, double* n, double* H) {
  const double r = norm3(p);
  for (int i = 0; i < 3; ++i) n[i] = p[i] / r;
  if (!H) return;
  const double x2 = p[0] * p[0], y2 = p[1] * p[1], z2 = p[2] * p[2];
  const double xy = p[0] * p[1], xz = p[0] * p[2], yz = p[1] * p[2];
  const double d = pow(x2 + y2 + z2, 1.5);
  H[0] = (y2 + z2) / d, H[1] = -xy / d, H[2] = -xz / d;
  H[3] = -xy / d, H[4] = (x2 + z2) / d, H[5] = -yz / d;
  H[6] = -xz / d, H[7] = -yz / d, H[8] = (x2 + y2) / d;
}

// TranslationFactor's whitened error e at (x_a, x_b) and, when M is given, its whitened Jacobian in x_b (N / sigma; the
// Jacobian in x_a is -M)
TV_HD void edge_error(const double* xa, const double* xb, const double* m, double inv_sigma, double* e, double* M) {
  const double d[3] = {xb[0] - xa[0], xb[1] - xa[1], xb[2] - xa[2]};
  double n[3];
  normalize(d, n, M);
  for (int i = 0; i < 3; ++i) e[i] = (n[i] - m[i]) * inv_sigma;
  if (M)
    for (int i = 0; i < 9; ++i) M[i] *= inv_sigma;
}

// the two priors of addPrior: prior 0 holds node n0 at the origin (Isotropic(3, 1 / inv_p)); prior 1 holds node n1 at t1
// under the edges' model (1 / inv_s, Huber huber_k)
struct Priors {
  int n0, n1;
  double inv_p, inv_s, huber_k;
  double t1[3];
};

// prior k's whitened error at x, the square root of its IRLS weight and its Jacobian scale (J = jac I before reweighting)
TV_HD void prior_err(const Priors& P, int k, const double* x, double* e, double& sw, double& jac) {
  if (k == 0) {
    for (int i = 0; i < 3; ++i) e[i] = x[i] * P.inv_p;
    sw = 1.0, jac = P.inv_p;
    return;
  }
  for (int i = 0; i < 3; ++i) e[i] = (x[i] - P.t1[i]) * P.inv_s;
  sw = sqrt(weight(norm3(e), P.huber_k)), jac = P.inv_s;
}

TV_HD double prior_cost(const Priors& P, int k, const double* x) {
  double e[3], sw, jac;
  prior_err(P, k, x, e, sw, jac);
  return k == 0 ? 0.5 * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]) : loss(norm3(e), P.huber_k);
}

// the priors on `node`, linearised at x: h I onto its Hessian block, their gradient J^T r onto g
TV_HD void prior_hg(const Priors& P, int node, const double* x, double& h, double* g) {
  for (int k = 0; k < 2; ++k) {
    if (node != (k == 0 ? P.n0 : P.n1)) continue;
    double e[3], sw, jac;
    prior_err(P, k, x, e, sw, jac);
    const double j = sw * jac;
    h += j * j;
    for (int i = 0; i < 3; ++i) g[i] += j * (sw * e[i]);
  }
}

// prior k's share of the linearised decrease (-(r . Jd + |Jd|^2 / 2)) and of the old linearised cost, for the step d of
// its node from the linearisation point x
TV_HD void prior_lin(const Priors& P, int k, const double* x, const double* d, double& lin, double& old) {
  double e[3], sw, jac;
  prior_err(P, k, x, e, sw, jac);
  for (int i = 0; i < 3; ++i) {
    const double r = sw * e[i], jd = sw * jac * d[i];
    lin -= r * jd + 0.5 * jd * jd, old += 0.5 * r * r;
  }
}

}  // namespace trmath
