// Host build of the verifier's fp64 primitives (gtsfm_b200/csrc/ransac_math.cuh) as a C ABI, so the Python tests can pin
// oracle/ransac_ref.py to the arithmetic the kernels compile.  Built with g++ by tests/test_ransac_ref_cpu.py and by
// tests/test_ransac_stages_gpu.py (with -DB2_FIVEPT_QR, the shipped 5-point variant).
#include "../../gtsfm_b200/csrc/ransac_math.cuh"

using namespace rmath;

extern "C" {

// samples [count][m] of sample_distinct(seed, stream0 + s, n, m)
void shim_sample_distinct(unsigned long long seed, unsigned long long stream0, int count, int n, int m, int* out) {
  for (int s = 0; s < count; ++s) sample_distinct(seed, stream0 + (unsigned long long)s, n, m, out + (size_t)s * m);
}

// mode 0: sampson_sq, 1: epiline_sq of M at k points x1 / x2 [k][2]
void shim_error(int mode, const double* M, const double* x1, const double* x2, int k, double* out) {
  for (int i = 0; i < k; ++i)
    out[i] = mode == 0 ? sampson_sq(M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1])
                       : epiline_sq(M, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
}

// 8 correspondences [8][2] -> F [9]; returns the solution count (0 or 1)
int shim_eightpt(const double* x1, const double* x2, double* F) {
  return eightpt_solve(reinterpret_cast<const double(*)[2]>(x1), reinterpret_cast<const double(*)[2]>(x2), F);
}

// 5 correspondences [5][2] -> up to 10 E [10][9]; returns the solution count
int shim_fivept(const double* x1, const double* x2, double* E) {
  return fivept_solve(reinterpret_cast<const double(*)[2]>(x1), reinterpret_cast<const double(*)[2]>(x2),
                      reinterpret_cast<double(*)[9]>(E));
}
}
