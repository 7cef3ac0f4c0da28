// Host build of the LMedS verifier's fp64 primitives (gtsfm_b200/csrc/ransac_math.cuh) as a C ABI, for oracle/lmeds_ref.py
// and the LMedS tests.  Built with g++ (-DB2_FIVEPT_QR: the 5-point variant libgtsfm_b200.so compiles) by
// oracle/lmeds_ref.build_shim.
#include "../../gtsfm_b200/csrc/ransac_math.cuh"

using namespace rmath;

extern "C" {

// mode 0: 5 correspondences -> up to 10 E (every real root); mode 1: 7 -> up to 3 F.  [.][2] in, [10][9] out.
int lm_solve(int mode, const double* x1, const double* x2, double* out) {
  auto a = reinterpret_cast<const double(*)[2]>(x1);
  auto b = reinterpret_cast<const double(*)[2]>(x2);
  auto o = reinterpret_cast<double(*)[9]>(out);
  return mode == 0 ? fivept_solve_all(a, b, o) : sevenpt_solve(a, b, o);
}

// the RANSAC verifier's 5-point solver, for comparison
int lm_fivept_sampled(const double* x1, const double* x2, double* out) {
  return fivept_solve(reinterpret_cast<const double(*)[2]>(x1), reinterpret_cast<const double(*)[2]>(x2),
                      reinterpret_cast<double(*)[9]>(out));
}

// the complete-root 5-point solver's degree-10 polynomial (ascending, scaled) -> poly [11]; returns the solution count
int lm_fivept_poly(const double* x1, const double* x2, double* poly) {
  double E[10][9];
  for (int i = 0; i <= 10; ++i) poly[i] = 0.0;
  return fivept_solve_t<true>(reinterpret_cast<const double(*)[2]>(x1), reinterpret_cast<const double(*)[2]>(x2), E, poly);
}

// real roots of p (ascending coefficients, degree <= 10)
int lm_poly_roots(const double* p, int deg, double* roots) { return upoly_all_real_roots(p, deg, roots); }

int lm_subsets(const double* x1, const double* x2, int k, int mode, int niters, int* idx) {
  return lmeds_subsets(x1, x2, k, mode, niters, idx);
}

int lm_niters(double confidence, int m, int max_iters) { return lmeds_niters(confidence, m, max_iters); }

void lm_errors(int mode, const double* M, const double* x1, const double* x2, int k, float* out) {
  for (int i = 0; i < k; ++i)
    out[i] = mode == 0 ? sampson_sq_cv(M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1])
                       : epiline_sq_cv(M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
}
}
