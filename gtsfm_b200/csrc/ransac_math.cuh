// Two-view geometry primitives in fp64, usable from host and device (the host build is the unit-test harness in
// tests/cpp/test_ransac_math.cpp; the device build is ransac.cu).
//
// What they restate: the arithmetic the reference delegates to OpenCV (opencv-python 4.12.0.88 pinned, uv.lock:1911)
// at gtsfm/frontend/verifier/ransac.py:74-81 (findEssentialMat: 5-point minimal solver of Nister, TPAMI 2004, inside a
// RANSAC loop with squared-Sampson inlier test), :103-110 (findFundamentalMat) and gtsfm/utils/verification.py:83
// (recoverPose: decompose E, cheirality vote).  Published algorithms, written from their definitions.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define RM_HD __host__ __device__ __forceinline__
#define RM_HDN __host__ __device__
#else
#define RM_HD inline
#define RM_HDN inline
#endif

namespace rmath {

// ---- small dense linear algebra -----------------------------------------------------------------------------------

// Cyclic Jacobi eigen-decomposition of a symmetric N x N matrix (row-major, destroyed).  V columns = eigenvectors.
// On the device the rotation loops of the small instances (N <= 4: svd3, the cheirality triangulation) are fully unrolled,
// so every index is static and A / V stay in registers; with run-time (p, q) they live in local memory and each of the
// ~200 accesses per rotation is a dependent L1 round trip - that, not the arithmetic, is what made the fp64 kernels slow.
#if defined(__CUDA_ARCH__)
#define RM_UNROLL_SMALL _Pragma("unroll")
#else
#define RM_UNROLL_SMALL
#endif
template <int N>
RM_HDN void jacobi_eig(double* A, double* V, double* w) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i * N + j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 40; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < N; ++i) {
      diag += A[i * N + i] * A[i * N + i];
      for (int j = i + 1; j < N; ++j) off += A[i * N + j] * A[i * N + j];
    }
    if (off <= 1e-30 * (diag + 1e-300)) break;
    if (N <= 4) {
      RM_UNROLL_SMALL
      for (int p = 0; p < N - 1; ++p) {
        RM_UNROLL_SMALL
        for (int q = p + 1; q < N; ++q) {
          double apq = A[p * N + q];
          if (fabs(apq) < 1e-300) continue;
          double theta = (A[q * N + q] - A[p * N + p]) / (2.0 * apq);
          double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
          RM_UNROLL_SMALL
          for (int k = 0; k < N; ++k) {
            double akp = A[k * N + p], akq = A[k * N + q];
            A[k * N + p] = c * akp - s * akq;
            A[k * N + q] = s * akp + c * akq;
          }
          RM_UNROLL_SMALL
          for (int k = 0; k < N; ++k) {
            double apk = A[p * N + k], aqk = A[q * N + k];
            A[p * N + k] = c * apk - s * aqk;
            A[q * N + k] = s * apk + c * aqk;
          }
          RM_UNROLL_SMALL
          for (int k = 0; k < N; ++k) {
            double vkp = V[k * N + p], vkq = V[k * N + q];
            V[k * N + p] = c * vkp - s * vkq;
            V[k * N + q] = s * vkp + c * vkq;
          }
        }
      }
      continue;
    }
    for (int p = 0; p < N - 1; ++p) {
      for (int q = p + 1; q < N; ++q) {
        double apq = A[p * N + q];
        if (fabs(apq) < 1e-300) continue;
        double theta = (A[q * N + q] - A[p * N + p]) / (2.0 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {
          double akp = A[k * N + p], akq = A[k * N + q];
          A[k * N + p] = c * akp - s * akq;
          A[k * N + q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {
          double apk = A[p * N + k], aqk = A[q * N + k];
          A[p * N + k] = c * apk - s * aqk;
          A[q * N + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {
          double vkp = V[k * N + p], vkq = V[k * N + q];
          V[k * N + p] = c * vkp - s * vkq;
          V[k * N + q] = s * vkp + c * vkq;
        }
      }
    }
  }
  for (int i = 0; i < N; ++i) w[i] = A[i * N + i];
}

RM_HD void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
RM_HD double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}
RM_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// SVD of a 3x3 matrix M = U diag(s) V^T with s0 >= s1 >= s2 >= 0, det(U) = det(V) = +1 not enforced.
RM_HDN void svd3(const double* M, double* U, double* s, double* V) {
  double A[9], Ev[9], w[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i * 3 + j] = M[i] * M[j] + M[3 + i] * M[3 + j] + M[6 + i] * M[6 + j];  // M^T M
  jacobi_eig<3>(A, Ev, w);
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (w[o[b]] > w[o[a]]) {
        int tt = o[a];
        o[a] = o[b];
        o[b] = tt;
      }
  for (int c = 0; c < 3; ++c) {
    s[c] = sqrt(w[o[c]] > 0 ? w[o[c]] : 0.0);
    for (int r = 0; r < 3; ++r) V[r * 3 + c] = Ev[r * 3 + o[c]];
  }
  // U columns: M v / s for the two leading singular values, third by cross product
  double u[3][3];
  for (int c = 0; c < 2; ++c) {
    double n = 0;
    for (int r = 0; r < 3; ++r) {
      u[c][r] = M[r * 3] * V[c] + M[r * 3 + 1] * V[3 + c] + M[r * 3 + 2] * V[6 + c];
      n += u[c][r] * u[c][r];
    }
    n = sqrt(n);
    if (n < 1e-300) n = 1;
    for (int r = 0; r < 3; ++r) u[c][r] /= n;
  }
  // re-orthogonalise u1 against u0 (guards the degenerate s1 ~ 0 case)
  double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
  double n = 0;
  for (int r = 0; r < 3; ++r) {
    u[1][r] -= d * u[0][r];
    n += u[1][r] * u[1][r];
  }
  n = sqrt(n);
  if (n < 1e-300) n = 1;
  for (int r = 0; r < 3; ++r) u[1][r] /= n;
  cross3(u[0], u[1], u[2]);
  // keep M v2 = s2 u2: flip v2 when the cross product picked the opposite sign
  double mv2 = 0;
  for (int r = 0; r < 3; ++r) mv2 += u[2][r] * (M[r * 3] * V[2] + M[r * 3 + 1] * V[5] + M[r * 3 + 2] * V[8]);
  if (mv2 < 0)
    for (int r = 0; r < 3; ++r) V[r * 3 + 2] = -V[r * 3 + 2];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) U[r * 3 + c] = u[c][r];
}

// ---- error metrics --------------------------------------------------------------------------------------------------

// squared Sampson distance of x2^T M x1 = 0 (what cv2 USAC thresholds against thr^2 for E; checked against the golden
// masks in tests/golden/verifier_*.npz).
RM_HD double sampson_sq(const double* M, double x1, double y1, double x2, double y2) {
  double l2x = M[0] * x1 + M[1] * y1 + M[2], l2y = M[3] * x1 + M[4] * y1 + M[5], l2z = M[6] * x1 + M[7] * y1 + M[8];
  double l1x = M[0] * x2 + M[3] * y2 + M[6], l1y = M[1] * x2 + M[4] * y2 + M[7];
  double num = x2 * l2x + y2 * l2y + l2z;
  double den = l2x * l2x + l2y * l2y + l1x * l1x + l1y * l1y;
  return den > 0 ? num * num / den : 1e300;
}
// symmetric squared point-to-epipolar-line distance, max of the two images (cv2 FM_RANSAC's computeError).
RM_HD double epiline_sq(const double* M, double x1, double y1, double x2, double y2) {
  double l2x = M[0] * x1 + M[1] * y1 + M[2], l2y = M[3] * x1 + M[4] * y1 + M[5], l2z = M[6] * x1 + M[7] * y1 + M[8];
  double l1x = M[0] * x2 + M[3] * y2 + M[6], l1y = M[1] * x2 + M[4] * y2 + M[7], l1z = M[2] * x2 + M[5] * y2 + M[8];
  double n2 = x2 * l2x + y2 * l2y + l2z, n1 = x1 * l1x + y1 * l1y + l1z;
  double d2 = n2 * n2 / (l2x * l2x + l2y * l2y + 1e-300), d1 = n1 * n1 / (l1x * l1x + l1y * l1y + 1e-300);
  return d1 > d2 ? d1 : d2;
}

// ---- polynomials in (x, y, z) of total degree <= 3, dense exponent-indexed ----------------------------------------
struct Poly {
  double c[4][4][4];
};
RM_HD void poly_zero(Poly& p) {
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b)
      for (int d = 0; d < 4; ++d) p.c[a][b][d] = 0.0;
}
// r += s * p * q, deg(p) = dp, deg(q) = dq, dp + dq <= 3
RM_HDN void poly_muladd(Poly& r, const Poly& p, int dp, const Poly& q, int dq, double s) {
  for (int a = 0; a <= dp; ++a)
    for (int b = 0; a + b <= dp; ++b)
      for (int d = 0; a + b + d <= dp; ++d) {
        double pc = p.c[a][b][d];
        if (pc == 0.0) continue;
        pc *= s;
        for (int e = 0; e <= dq; ++e)
          for (int f = 0; e + f <= dq; ++f)
            for (int g = 0; e + f + g <= dq; ++g) r.c[a + e][b + f][d + g] += pc * q.c[e][f][g];
      }
}

// univariate helpers (coefficients by ascending power)
RM_HD double upoly_eval(const double* p, int deg, double z) {
  double v = p[deg];
  for (int i = deg - 1; i >= 0; --i) v = v * z + p[i];
  return v;
}
// r (deg da+db) = a * b
RM_HD void upoly_mul(const double* a, int da, const double* b, int db, double* r) {
  for (int i = 0; i <= da + db; ++i) r[i] = 0.0;
  for (int i = 0; i <= da; ++i)
    for (int j = 0; j <= db; ++j) r[i + j] += a[i] * b[j];
}

// real roots of a degree-`deg` polynomial by sign-change bracketing on [-1, 1] for p(z) and for the reversed
// polynomial (roots 1/z), then bisection.  Returns the number of roots written (<= max_roots).
// Two phases per pass so that the 32 hypotheses of a warp stay in lock-step: (1) all 161 sample points are evaluated and
// the bracketing intervals recorded, (2) a fixed-trip loop bisects the recorded intervals.  With the bisection nested inside
// the scan (round 1) a warp ran it for the UNION of its lanes' hit intervals - ~100 bisections per pass instead of ~5 -
// which was most of k_rs_hyp_E's 1.1 ms.
RM_HDN int upoly_real_roots(const double* p, int deg, double* roots, int max_roots) {
  const int NS = 160;
  const int MAXB = 10;   // brackets per pass (a degree-10 polynomial has at most 10 real roots)
  const int NBIS = 60;   // 2 / 160 * 2^-60 is far below the spacing of doubles in [-1, 1]
  int n = 0;
  double rev[16];
  for (int i = 0; i <= deg; ++i) rev[i] = p[deg - i];
  for (int pass = 0; pass < 2 && n < max_roots; ++pass) {
    const double* q = pass == 0 ? p : rev;
    double blo[MAXB], bhi[MAXB], bflo[MAXB];
    int nb = 0;
    double a = -1.0, fa = upoly_eval(q, deg, a);
    for (int i = 1; i <= NS; ++i) {
      double b = -1.0 + 2.0 * i / NS, fb = upoly_eval(q, deg, b);
      bool hit = (fa == 0.0) || (fa < 0) != (fb < 0);
      if (fb == 0.0 && i < NS) hit = false;  // will be caught as fa == 0 of the next interval
      if (hit && nb < MAXB) {
        blo[nb] = a, bhi[nb] = (fa == 0.0) ? a : b, bflo[nb] = fa;
        ++nb;
      }
      a = b;
      fa = fb;
    }
    for (int r = 0; r < MAXB; ++r) {  // fixed trip count: lanes without an r-th bracket idle through it
      if (r >= nb || n >= max_roots) continue;
      double lo = blo[r], hi = bhi[r], flo = bflo[r];
      if (lo != hi) {
        for (int it = 0; it < NBIS; ++it) {
          double mid = 0.5 * (lo + hi), fm = upoly_eval(q, deg, mid);
          if (fm == 0.0) {
            lo = hi = mid;
          } else if ((fm < 0) == (flo < 0)) {
            lo = mid, flo = fm;
          } else {
            hi = mid;
          }
        }
      }
      double rt = 0.5 * (lo + hi);
      if (pass == 0) {
        roots[n++] = rt;
      } else if (fabs(rt) > 1e-12 && fabs(rt) < 1.0) {  // |z| > 1 strictly (|z| == 1 belongs to pass 0)
        roots[n++] = 1.0 / rt;
      }
    }
  }
  return n;
}

// EVERY real root of p (degree <= 10) in [-1, 1], ascending.  Between two consecutive real roots of p' the polynomial is
// monotone, so the roots of p' split [-1, 1] into intervals holding at most one root each; the roots of p' come from p''
// the same way, down to the linear derivative.  Unlike sampling for sign changes this finds close pairs of roots (a pair
// closer than the sampling step gives no sign change at the samples, but the root of p' between them separates it).
RM_HDN int upoly_roots_in_unit(const double* p, int deg, double* roots) {
  double d[11][11];  // d[j] = j-th derivative / j!, ascending, degree deg - j
  double crit[12], nxt[12];
  for (int i = 0; i <= deg; ++i) d[0][i] = p[i];
  for (int j = 1; j <= deg; ++j)
    for (int i = 0; i <= deg - j; ++i) d[j][i] = d[j - 1][i + 1] * (double)(i + 1);
  int nc = 0;  // roots of the current derivative in (-1, 1), ascending
  for (int j = deg - 1; j >= 0; --j) {
    const double* q = d[j];
    const int dq = deg - j;
    double a = -1.0, fa = upoly_eval(q, dq, a);
    int nn = 0;
    for (int s = 0; s <= nc; ++s) {
      const double b = s < nc ? crit[s] : 1.0, fb = upoly_eval(q, dq, b);
      if (fa == 0.0) {
        if (nn == 0 || nxt[nn - 1] != a) nxt[nn++] = a;
      } else if (fb != 0.0 && (fa < 0) != (fb < 0)) {
        double lo = a, hi = b, flo = fa;
        for (int it = 0; it < 200; ++it) {
          const double mid = 0.5 * (lo + hi);
          if (mid == lo || mid == hi) break;
          const double fm = upoly_eval(q, dq, mid);
          if (fm == 0.0) {
            lo = hi = mid;
            break;
          }
          if ((fm < 0) == (flo < 0)) lo = mid, flo = fm;
          else hi = mid;
        }
        nxt[nn++] = 0.5 * (lo + hi);
      }
      a = b, fa = fb;
    }
    if (fa == 0.0 && (nn == 0 || nxt[nn - 1] != a)) nxt[nn++] = a;  // a root at +1
    for (int i = 0; i < nn; ++i) crit[i] = nxt[i];
    nc = nn;
  }
  for (int i = 0; i < nc; ++i) roots[i] = crit[i];
  return nc;
}
// every real root of p: [-1, 1] directly, |z| > 1 as 1 / z of the reversed polynomial's roots in (-1, 1) \ {0}.
RM_HDN int upoly_all_real_roots(const double* p, int deg, double* roots) {
  int n = upoly_roots_in_unit(p, deg, roots);
  double rev[11], rr[10];
  for (int i = 0; i <= deg; ++i) rev[i] = p[deg - i];
  const int nr = upoly_roots_in_unit(rev, deg, rr);
  for (int i = 0; i < nr; ++i)
    if (rr[i] != 0.0 && fabs(rr[i]) < 1.0) roots[n++] = 1.0 / rr[i];
  return n;
}

// ---- 5-point essential-matrix solver (Nister 2004) -------------------------------------------------------------
// x1, x2: 5 normalised correspondences; E_out: up to 10 solutions, row-major, x2^T E x1 = 0, Frobenius norm 1.
// kAllRoots = false (fivept_solve, the RANSAC verifier): the degree-10 polynomial's roots are bracketed by sign changes at
// 161 samples, which can miss a close pair.  kAllRoots = true (fivept_solve_all, the LMedS verifier, which must visit
// every solution cv2 visits): upoly_all_real_roots.
// poly_out (kAllRoots only, may be null): receives the scaled degree-10 polynomial in z, ascending (for tests).
template <bool kAllRoots>
RM_HDN int fivept_solve_t(const double (*x1)[2], const double (*x2)[2], double (*E_out)[9], double* poly_out = nullptr) {
#ifdef B2_FIVEPT_QR
  // (opt-in, host-validated, not yet run on the GPU: see DESIGN.md section 8) null space of the 5 x 9 epipolar constraint
  // matrix A by Householder QR of A^T (9 x 5): A^T = Q [R; 0], columns 5..8 of Q are an orthonormal basis of null(A).
  // Five reflections instead of Jacobi sweeps on the 9 x 9 Gram matrix, which is half of the solver's arithmetic.
  double basis[4][9];  // X, Y, Z, W
  {
    double a[9][5], hv[5][9], beta[5];
    for (int p = 0; p < 5; ++p) {
      const double q[9] = {x2[p][0] * x1[p][0], x2[p][0] * x1[p][1], x2[p][0], x2[p][1] * x1[p][0], x2[p][1] * x1[p][1],
                           x2[p][1],            x1[p][0],            x1[p][1], 1.0};
      for (int i = 0; i < 9; ++i) a[i][p] = q[i];
    }
    for (int j = 0; j < 5; ++j) {
      double n2 = 0.0;
      for (int i = j; i < 9; ++i) n2 += a[i][j] * a[i][j];
      for (int i = 0; i < 9; ++i) hv[j][i] = 0.0;
      beta[j] = 0.0;
      if (!(n2 > 1e-300)) continue;  // rank-deficient sample: the reflection is the identity
      const double alpha = a[j][j] > 0.0 ? -sqrt(n2) : sqrt(n2);
      double v2 = 0.0;
      for (int i = j; i < 9; ++i) {
        hv[j][i] = a[i][j] - (i == j ? alpha : 0.0);
        v2 += hv[j][i] * hv[j][i];
      }
      if (!(v2 > 1e-300)) continue;
      beta[j] = 2.0 / v2;
      for (int c = j; c < 5; ++c) {
        double sdot = 0.0;
        for (int i = j; i < 9; ++i) sdot += hv[j][i] * a[i][c];
        sdot *= beta[j];
        for (int i = j; i < 9; ++i) a[i][c] -= sdot * hv[j][i];
      }
    }
    for (int k = 0; k < 4; ++k) {
      double qv[9];
      for (int i = 0; i < 9; ++i) qv[i] = (i == 5 + k) ? 1.0 : 0.0;
      for (int j = 4; j >= 0; --j) {
        double sdot = 0.0;
        for (int i = j; i < 9; ++i) sdot += hv[j][i] * qv[i];
        sdot *= beta[j];
        for (int i = j; i < 9; ++i) qv[i] -= sdot * hv[j][i];
      }
      for (int i = 0; i < 9; ++i) basis[k][i] = qv[i];
    }
  }
#else
  // null space of the 5 x 9 epipolar constraint matrix via the 4 smallest eigenvectors of Q^T Q
  double QtQ[81], Vn[81], wn[9];
  for (int i = 0; i < 81; ++i) QtQ[i] = 0.0;
  for (int p = 0; p < 5; ++p) {
    double q[9] = {x2[p][0] * x1[p][0], x2[p][0] * x1[p][1], x2[p][0], x2[p][1] * x1[p][0], x2[p][1] * x1[p][1],
                   x2[p][1],            x1[p][0],            x1[p][1], 1.0};
    for (int i = 0; i < 9; ++i)
      for (int j = 0; j < 9; ++j) QtQ[i * 9 + j] += q[i] * q[j];
  }
  jacobi_eig<9>(QtQ, Vn, wn);
  int ord[9];
  for (int i = 0; i < 9; ++i) ord[i] = i;
  for (int a = 0; a < 4; ++a)
    for (int b = a + 1; b < 9; ++b)
      if (wn[ord[b]] < wn[ord[a]]) {
        int t = ord[a];
        ord[a] = ord[b];
        ord[b] = t;
      }
  double basis[4][9];  // X, Y, Z, W
  for (int k = 0; k < 4; ++k)
    for (int i = 0; i < 9; ++i) basis[k][i] = Vn[i * 9 + ord[k]];

#endif

  // E(x,y,z) = x X + y Y + z Z + W, entries are degree-1 polynomials
  Poly E[9];
  for (int i = 0; i < 9; ++i) {
    poly_zero(E[i]);
    E[i].c[1][0][0] = basis[0][i];
    E[i].c[0][1][0] = basis[1][i];
    E[i].c[0][0][1] = basis[2][i];
    E[i].c[0][0][0] = basis[3][i];
  }
  Poly EEt[9];  // E E^T, degree 2
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      poly_zero(EEt[i * 3 + j]);
      for (int k = 0; k < 3; ++k) poly_muladd(EEt[i * 3 + j], E[i * 3 + k], 1, E[j * 3 + k], 1, 1.0);
    }
  Poly tr;
  poly_zero(tr);
  for (int a = 0; a < 3; ++a)
    for (int b = 0; a + b < 3; ++b)
      for (int d = 0; a + b + d < 3; ++d) tr.c[a][b][d] = EEt[0].c[a][b][d] + EEt[4].c[a][b][d] + EEt[8].c[a][b][d];
  Poly eq[10];
  // 2 E E^T E - trace(E E^T) E = 0  (9 cubics)
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      Poly& r = eq[i * 3 + j];
      poly_zero(r);
      for (int k = 0; k < 3; ++k) poly_muladd(r, EEt[i * 3 + k], 2, E[k * 3 + j], 1, 2.0);
      poly_muladd(r, tr, 2, E[i * 3 + j], 1, -1.0);
    }
  // det(E) = 0
  {
    Poly& r = eq[9];
    poly_zero(r);
    Poly m;
    const int idx[3][2][2] = {{{4, 8}, {5, 7}}, {{3, 8}, {5, 6}}, {{3, 7}, {4, 6}}};
    for (int t = 0; t < 3; ++t) {
      poly_zero(m);
      poly_muladd(m, E[idx[t][0][0]], 1, E[idx[t][0][1]], 1, 1.0);
      poly_muladd(m, E[idx[t][1][0]], 1, E[idx[t][1][1]], 1, -1.0);
      poly_muladd(r, m, 2, E[t], 1, (t == 1) ? -1.0 : 1.0);
    }
  }
  // 10 x 20 coefficient matrix, columns ordered so that Gauss-Jordan on the first 10 leaves polynomials in z
  const int mono[20][3] = {{3, 0, 0}, {0, 3, 0}, {2, 1, 0}, {1, 2, 0}, {2, 0, 1}, {2, 0, 0}, {0, 2, 1}, {0, 2, 0}, {1, 1, 1}, {1, 1, 0},
                           {1, 0, 2}, {1, 0, 1}, {1, 0, 0}, {0, 1, 2}, {0, 1, 1}, {0, 1, 0}, {0, 0, 3}, {0, 0, 2}, {0, 0, 1}, {0, 0, 0}};
  double M[10][20];
  for (int r = 0; r < 10; ++r)
    for (int c = 0; c < 20; ++c) M[r][c] = eq[r].c[mono[c][0]][mono[c][1]][mono[c][2]];
  for (int c = 0; c < 10; ++c) {
    int piv = c;
    double best = fabs(M[c][c]);
    for (int r = c + 1; r < 10; ++r)
      if (fabs(M[r][c]) > best) best = fabs(M[r][c]), piv = r;
    if (best < 1e-14) return 0;
    if (piv != c)
      for (int k = 0; k < 20; ++k) {
        double t = M[c][k];
        M[c][k] = M[piv][k];
        M[piv][k] = t;
      }
    double inv = 1.0 / M[c][c];
    for (int k = c; k < 20; ++k) M[c][k] *= inv;
    for (int r = 0; r < 10; ++r) {
      if (r == c) continue;
      double f = M[r][c];
      if (f == 0.0) continue;
      for (int k = c; k < 20; ++k) M[r][k] -= f * M[c][k];
    }
  }
  // rows 4..9 = leading monomials x^2 z, x^2, y^2 z, y^2, xyz, xy.  k = e - z f, l = g - z h, m = i - z j
  double B[3][3][5];  // [row][column: x, y, 1][power of z]
  for (int r = 0; r < 3; ++r) {
    const double* hi = &M[4 + 2 * r][10];  // e, g, i : coefficients of [xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1]
    const double* lo = &M[5 + 2 * r][10];  // f, h, j
    for (int col = 0; col < 2; ++col) {
      const double* a = hi + 3 * col;
      const double* b = lo + 3 * col;
      B[r][col][0] = a[2];
      B[r][col][1] = a[1] - b[2];
      B[r][col][2] = a[0] - b[1];
      B[r][col][3] = -b[0];
      B[r][col][4] = 0.0;
    }
    const double* a = hi + 6;
    const double* b = lo + 6;
    B[r][2][0] = a[3];
    B[r][2][1] = a[2] - b[3];
    B[r][2][2] = a[1] - b[2];
    B[r][2][3] = a[0] - b[1];
    B[r][2][4] = -b[0];
  }
  // det B(z): degree 10
  double detp[11];
  for (int i = 0; i <= 10; ++i) detp[i] = 0.0;
  const int perm[3][2] = {{1, 2}, {0, 2}, {0, 1}};  // cofactor expansion along the third column (degree 4 entries)
  for (int r = 0; r < 3; ++r) {
    int r1 = perm[r][0], r2 = perm[r][1];
    double m1[7], m2[7], minor[7], term[11];
    upoly_mul(B[r1][0], 3, B[r2][1], 3, m1);
    upoly_mul(B[r1][1], 3, B[r2][0], 3, m2);
    for (int i = 0; i <= 6; ++i) minor[i] = m1[i] - m2[i];
    upoly_mul(minor, 6, B[r][2], 4, term);
    double sgn = (r == 1) ? -1.0 : 1.0;  // (-1)^(r+2)
    for (int i = 0; i <= 10; ++i) detp[i] += sgn * term[i];
  }
  double scale = 0.0;
  for (int i = 0; i <= 10; ++i) scale = fabs(detp[i]) > scale ? fabs(detp[i]) : scale;
  if (!(scale > 0.0) || !(scale < 1e300)) return 0;
  for (int i = 0; i <= 10; ++i) detp[i] /= scale;
  if (kAllRoots && poly_out)
    for (int i = 0; i <= 10; ++i) poly_out[i] = detp[i];
  double roots[10];
  int nr = kAllRoots ? upoly_all_real_roots(detp, 10, roots) : upoly_real_roots(detp, 10, roots, 10);
  int ns = 0;
  for (int ri = 0; ri < nr; ++ri) {
    double z = roots[ri];
    double b[3][3];
    for (int r = 0; r < 3; ++r) {
      b[r][0] = upoly_eval(B[r][0], 3, z);
      b[r][1] = upoly_eval(B[r][1], 3, z);
      b[r][2] = upoly_eval(B[r][2], 4, z);
    }
    // (x, y, 1) spans the null space of B(z): take the best-conditioned cross product of two rows
    double bestv[3] = {0, 0, 0}, bestn = -1.0;
    for (int a = 0; a < 3; ++a)
      for (int c = a + 1; c < 3; ++c) {
        double v[3];
        cross3(b[a], b[c], v);
        double na = b[a][0] * b[a][0] + b[a][1] * b[a][1] + b[a][2] * b[a][2];
        double nc = b[c][0] * b[c][0] + b[c][1] * b[c][1] + b[c][2] * b[c][2];
        double q = (v[2] * v[2]) / (na * nc + 1e-300);
        if (q > bestn) bestn = q, bestv[0] = v[0], bestv[1] = v[1], bestv[2] = v[2];
      }
    if (!(fabs(bestv[2]) > 1e-300)) continue;
    double x = bestv[0] / bestv[2], y = bestv[1] / bestv[2];
    double nrm = 0.0, e[9];
    for (int i = 0; i < 9; ++i) {
      e[i] = x * basis[0][i] + y * basis[1][i] + z * basis[2][i] + basis[3][i];
      nrm += e[i] * e[i];
    }
    nrm = sqrt(nrm);
    if (!(nrm > 1e-300) || !(nrm < 1e300)) continue;
    for (int i = 0; i < 9; ++i) E_out[ns][i] = e[i] / nrm;
    ++ns;
  }
  return ns;
}
RM_HDN int fivept_solve(const double (*x1)[2], const double (*x2)[2], double (*E_out)[9]) {
  return fivept_solve_t<false>(x1, x2, E_out);
}
RM_HDN int fivept_solve_all(const double (*x1)[2], const double (*x2)[2], double (*E_out)[9]) {
  return fivept_solve_t<true>(x1, x2, E_out);
}

// ---- cv2's LMedS arithmetic (the LMedS verifier, lmeds.cu) ------------------------------------------------------------
// Products and sums rounded one at a time (no FMA contraction on the device), so the float cast of an error sees the
// double cv2 computes.
#if defined(__CUDA_ARCH__)
#define RM_MUL(a, b) __dmul_rn((a), (b))
#define RM_ADD(a, b) __dadd_rn((a), (b))
#else
#define RM_MUL(a, b) ((a) * (b))
#define RM_ADD(a, b) ((a) + (b))
#endif
// squared Sampson error of cv2's EMEstimatorCallback::computeError, as float
RM_HD float sampson_sq_cv(const double* E, double x1, double y1, double x2, double y2) {
  const double e0 = RM_ADD(RM_ADD(RM_MUL(E[0], x1), RM_MUL(E[1], y1)), E[2]);
  const double e1 = RM_ADD(RM_ADD(RM_MUL(E[3], x1), RM_MUL(E[4], y1)), E[5]);
  const double e2 = RM_ADD(RM_ADD(RM_MUL(E[6], x1), RM_MUL(E[7], y1)), E[8]);
  const double t0 = RM_ADD(RM_ADD(RM_MUL(E[0], x2), RM_MUL(E[3], y2)), E[6]);
  const double t1 = RM_ADD(RM_ADD(RM_MUL(E[1], x2), RM_MUL(E[4], y2)), E[7]);
  const double r = RM_ADD(RM_ADD(RM_MUL(x2, e0), RM_MUL(y2, e1)), e2);
  const double den = RM_ADD(RM_ADD(RM_ADD(RM_MUL(e0, e0), RM_MUL(e1, e1)), RM_MUL(t0, t0)), RM_MUL(t1, t1));
  return (float)(RM_MUL(r, r) / den);
}
// symmetric squared epipolar-line error of cv2's FMEstimatorCallback::computeError (points already float-valued), as float
RM_HD float epiline_sq_cv(const double* F, double x1, double y1, double x2, double y2) {
  double a = RM_ADD(RM_ADD(RM_MUL(F[0], x1), RM_MUL(F[1], y1)), F[2]);
  double b = RM_ADD(RM_ADD(RM_MUL(F[3], x1), RM_MUL(F[4], y1)), F[5]);
  double c = RM_ADD(RM_ADD(RM_MUL(F[6], x1), RM_MUL(F[7], y1)), F[8]);
  const double s2 = 1. / RM_ADD(RM_MUL(a, a), RM_MUL(b, b));
  const double d2 = RM_ADD(RM_ADD(RM_MUL(x2, a), RM_MUL(y2, b)), c);
  a = RM_ADD(RM_ADD(RM_MUL(F[0], x2), RM_MUL(F[3], y2)), F[6]);
  b = RM_ADD(RM_ADD(RM_MUL(F[1], x2), RM_MUL(F[4], y2)), F[7]);
  c = RM_ADD(RM_ADD(RM_MUL(F[2], x2), RM_MUL(F[5], y2)), F[8]);
  const double s1 = 1. / RM_ADD(RM_MUL(a, a), RM_MUL(b, b));
  const double d1 = RM_ADD(RM_ADD(RM_MUL(x1, a), RM_MUL(y1, b)), c);
  const double u = RM_MUL(RM_MUL(d1, d1), s1), v = RM_MUL(RM_MUL(d2, d2), s2);
  return (float)(u < v ? v : u);
}
// cv2's haveCollinearPoints for the last of the first `count` points of p [.][2] (float-valued): is it on a line through two
// earlier points (or on top of one)?
RM_HD bool collinear_last(const double (*p)[2], int count) {
  const int i = count - 1;
  const double eps = 1.1920928955078125e-07;  // FLT_EPSILON
  for (int j = 0; j < i; ++j) {
    const double dx1 = (double)(float)(p[j][0] - p[i][0]), dy1 = (double)(float)(p[j][1] - p[i][1]);
    for (int k = 0; k < j; ++k) {
      const double dx2 = (double)(float)(p[k][0] - p[i][0]), dy2 = (double)(float)(p[k][1] - p[i][1]);
      if (fabs(RM_ADD(RM_MUL(dx2, dy1), -RM_MUL(dy2, dx1))) <= eps * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2))) return true;
    }
  }
  return false;
}

// 7-point fundamental-matrix solver (Hartley & Zisserman 11.1.2) on float-valued pixels: Hartley normalisation, the
// two-dimensional null space of the 7 x 9 constraint matrix (F = lambda f1 + (1 - lambda) f2), det F = 0 as a cubic in
// lambda, every real root, de-normalised and scaled so that F33 = 1 (as cv2's run7Point).  Returns 0..3 solutions.
RM_HDN int sevenpt_solve(const double (*x1)[2], const double (*x2)[2], double (*F_out)[9]) {
  double c1x = 0, c1y = 0, c2x = 0, c2y = 0;
  for (int i = 0; i < 7; ++i) c1x += x1[i][0], c1y += x1[i][1], c2x += x2[i][0], c2y += x2[i][1];
  const double t = 1. / 7;
  c1x *= t, c1y *= t, c2x *= t, c2y *= t;
  double s1 = 0, s2 = 0;
  for (int i = 0; i < 7; ++i) {
    s1 += sqrt((x1[i][0] - c1x) * (x1[i][0] - c1x) + (x1[i][1] - c1y) * (x1[i][1] - c1y));
    s2 += sqrt((x2[i][0] - c2x) * (x2[i][0] - c2x) + (x2[i][1] - c2y) * (x2[i][1] - c2y));
  }
  s1 *= t, s2 *= t;
  if (s1 < 1.1920928955078125e-07 || s2 < 1.1920928955078125e-07) return 0;
  s1 = 1.4142135623730951 / s1, s2 = 1.4142135623730951 / s2;
  double A[81];
  for (int i = 0; i < 81; ++i) A[i] = 0;
  for (int p = 0; p < 7; ++p) {
    const double ax = (x1[p][0] - c1x) * s1, ay = (x1[p][1] - c1y) * s1;
    const double bx = (x2[p][0] - c2x) * s2, by = (x2[p][1] - c2y) * s2;
    const double q[9] = {bx * ax, bx * ay, bx, by * ax, by * ay, by, ax, ay, 1.0};
    for (int i = 0; i < 9; ++i)
      for (int j = 0; j < 9; ++j) A[i * 9 + j] += q[i] * q[j];
  }
  double V[81], w[9];
  jacobi_eig<9>(A, V, w);
  int o0 = 0, o1 = -1;  // the two smallest eigenvalues span the null space
  for (int i = 1; i < 9; ++i)
    if (w[i] < w[o0]) o0 = i;
  for (int i = 0; i < 9; ++i)
    if (i != o0 && (o1 < 0 || w[i] < w[o1])) o1 = i;
  double f1[9], f2[9];
  for (int i = 0; i < 9; ++i) f2[i] = V[i * 9 + o1], f1[i] = V[i * 9 + o0] - f2[i];
  // det(lambda f1 + f2) = c3 lambda^3 + c2 lambda^2 + c1 lambda + c0, ascending in cf
  double cf[4];
  {
    double t0 = f2[4] * f2[8] - f2[5] * f2[7], t1 = f2[3] * f2[8] - f2[5] * f2[6], t2 = f2[3] * f2[7] - f2[4] * f2[6];
    cf[0] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
    cf[1] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 - f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
            f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) -
            f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) + f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
    t0 = f1[4] * f1[8] - f1[5] * f1[7], t1 = f1[3] * f1[8] - f1[5] * f1[6], t2 = f1[3] * f1[7] - f1[4] * f1[6];
    cf[2] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 - f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
            f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) -
            f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) + f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
    cf[3] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
  }
  double scale = 0.0;
  for (int i = 0; i < 4; ++i) scale = fabs(cf[i]) > scale ? fabs(cf[i]) : scale;
  if (!(scale > 0.0) || !(scale < 1e300)) return 0;
  for (int i = 0; i < 4; ++i) cf[i] /= scale;
  double r[6];
  const int n = upoly_all_real_roots(cf, 3, r);
  const double T1[9] = {s1, 0, -s1 * c1x, 0, s1, -s1 * c1y, 0, 0, 1}, T2t[9] = {s2, 0, 0, 0, s2, 0, -s2 * c2x, -s2 * c2y, 1};
  int ns = 0;
  for (int k = 0; k < n && ns < 3; ++k) {
    double lambda = r[k], mu = 1.0, Fn[9];
    const double s = f1[8] * r[k] + f2[8];
    if (fabs(s) > 2.220446049250313e-16) {
      mu = 1. / s, lambda *= mu, Fn[8] = 1.0;
    } else {
      Fn[8] = 0.0;
    }
    for (int i = 0; i < 8; ++i) Fn[i] = f1[i] * lambda + f2[i] * mu;
    double tmp[9], F[9];
    mat3_mul(T2t, Fn, tmp);
    mat3_mul(tmp, T1, F);
    if (fabs(F[8]) > 1.1920928955078125e-07) {
      const double inv = 1. / F[8];
      for (int i = 0; i < 9; ++i) F[i] *= inv;
    }
    for (int i = 0; i < 9; ++i) F_out[ns][i] = F[i];
    ++ns;
  }
  return ns;
}

// ---- cv2's RNG (cv::RNG, multiply-with-carry) and its LMedS subset draw -------------------------------------------
RM_HD unsigned cvrng_next(unsigned long long& state) {
  state = (unsigned long long)(unsigned)state * 4164903690ull + (unsigned)(state >> 32);
  return (unsigned)state;
}
// cv2's LMeDS sample table: `niters` subsets of m = 5 (mode 0) or 7 (mode 1) indices of [0, k), one RNG stream seeded with
// 2^64 - 1.  An index equal to an earlier one of its subset is drawn again.  Mode 1 rejects a subset whose last point is
// collinear with two earlier ones in either image and draws a whole new one, at most 1000 times per subset.  Returns the
// subsets drawn: niters, fewer when the attempts ran out (cv2 stops sampling there), 0 when that happened on the first.
RM_HDN int lmeds_subsets(const double* x1, const double* x2, int k, int mode, int niters, int* idx) {
  const int m = mode == 0 ? 5 : 7;
  unsigned long long st = ~0ull;
  for (int it = 0; it < niters; ++it) {
    int* s = idx + (size_t)it * m;
    int attempt = 0;
    for (; attempt < 1000; ++attempt) {
      for (int i = 0; i < m; ++i) {
        int v;
        bool dup;
        do {
          v = (int)(cvrng_next(st) % (unsigned)k);
          dup = false;
          for (int j = 0; j < i; ++j) dup |= s[j] == v;
        } while (dup);
        s[i] = v;
      }
      if (mode == 0) break;
      double p1[7][2], p2[7][2];
      for (int i = 0; i < 7; ++i)  // cv2 casts F's points to float32
        for (int c = 0; c < 2; ++c) p1[i][c] = (double)(float)x1[2 * s[i] + c], p2[i][c] = (double)(float)x2[2 * s[i] + c];
      if (!collinear_last(p1, 7) && !collinear_last(p2, 7)) break;
    }
    if (attempt == 1000) return it;
  }
  return niters;
}
// cv2's RANSACUpdateNumIters(confidence, 0.45, m, max_iters), at least 3 (LMeDSPointSetRegistrator::run)
RM_HD int lmeds_niters(double confidence, int m, int max_iters) {
  const double num = log(fmax(1. - confidence, 2.2250738585072014e-308));
  const double denom = 1. - pow(0.55, (double)m);
  int n;
  if (denom < 2.2250738585072014e-308) n = 0;
  else {
    const double ld = log(denom);
    n = (ld >= 0 || -num >= max_iters * (-ld)) ? max_iters : (int)floor(num / ld + 0.5);
  }
  return n > 3 ? n : 3;
}

// ---- linear (8+ point) estimation helpers ---------------------------------------------------------------------------
// Given the 9x9 moment matrix A = sum q q^T of Hartley-normalised constraints, returns the smallest eigenvector as a
// 3x3 matrix (row-major).
RM_HDN void smallest_eigvec9(double* A, double* M) {
  double V[81], w[9];
  jacobi_eig<9>(A, V, w);
  int k = 0;
  for (int i = 1; i < 9; ++i)
    if (w[i] < w[k]) k = i;
  for (int i = 0; i < 9; ++i) M[i] = V[i * 9 + k];
}
// project onto the essential manifold (singular values (1,1,0)) / the rank-2 manifold (s2 = 0)
RM_HDN void enforce_essential(double* E) {
  double U[9], s[3], V[9];
  svd3(E, U, s, V);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[i * 3 + j] = (U[i * 3] * V[j * 3] + U[i * 3 + 1] * V[j * 3 + 1]) * 0.70710678118654752440;
}
RM_HDN void enforce_rank2(double* F) {
  double U[9], s[3], V[9];
  svd3(F, U, s, V);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) F[i * 3 + j] = U[i * 3] * s[0] * V[j * 3] + U[i * 3 + 1] * s[1] * V[j * 3 + 1];
}

// normalised 8-point algorithm (Hartley 1997) on 8 correspondences: F (unit Frobenius norm, rank 2) with x2^T F x1 = 0.
// Returns 1, or 0 for a degenerate sample (coincident points, zero F).
RM_HDN int eightpt_solve(const double (*x1)[2], const double (*x2)[2], double* F_out) {
  double c1x = 0, c1y = 0, c2x = 0, c2y = 0;
  for (int i = 0; i < 8; ++i) c1x += x1[i][0], c1y += x1[i][1], c2x += x2[i][0], c2y += x2[i][1];
  c1x /= 8, c1y /= 8, c2x /= 8, c2y /= 8;
  double d1 = 0, d2 = 0;
  for (int i = 0; i < 8; ++i) {
    d1 += sqrt((x1[i][0] - c1x) * (x1[i][0] - c1x) + (x1[i][1] - c1y) * (x1[i][1] - c1y));
    d2 += sqrt((x2[i][0] - c2x) * (x2[i][0] - c2x) + (x2[i][1] - c2y) * (x2[i][1] - c2y));
  }
  if (d1 < 1e-12 || d2 < 1e-12) return 0;
  double s1 = 1.4142135623730951 * 8 / d1, s2 = 1.4142135623730951 * 8 / d2;
  double A[81];
  for (int i = 0; i < 81; ++i) A[i] = 0;
  for (int p = 0; p < 8; ++p) {
    double ax = (x1[p][0] - c1x) * s1, ay = (x1[p][1] - c1y) * s1;
    double bx = (x2[p][0] - c2x) * s2, by = (x2[p][1] - c2y) * s2;
    double q[9] = {bx * ax, bx * ay, bx, by * ax, by * ay, by, ax, ay, 1.0};
    for (int i = 0; i < 9; ++i)
      for (int j = 0; j < 9; ++j) A[i * 9 + j] += q[i] * q[j];
  }
  double Fn[9];
  smallest_eigvec9(A, Fn);
  enforce_rank2(Fn);
  // F = T2^T Fn T1, T = [s 0 -s c; 0 s -s c; 0 0 1]
  double T1[9] = {s1, 0, -s1 * c1x, 0, s1, -s1 * c1y, 0, 0, 1}, T2t[9] = {s2, 0, 0, 0, s2, 0, -s2 * c2x, -s2 * c2y, 1};
  double tmp[9], F[9];
  mat3_mul(T2t, Fn, tmp);
  mat3_mul(tmp, T1, F);
  double n = 0;
  for (int i = 0; i < 9; ++i) n += F[i] * F[i];
  n = sqrt(n);
  if (!(n > 1e-300)) return 0;
  for (int i = 0; i < 9; ++i) F_out[i] = F[i] / n;
  return 1;
}

// ---- pose from E -----------------------------------------------------------------------------------------------
// The four (R, t) decompositions of E (Hartley & Zisserman 9.6.2): R = U W V^T or U W^T V^T, t = +-u3.
RM_HDN void decompose_E(const double* E, double* R1, double* R2, double* t) {
  double U[9], s[3], V[9];
  svd3(E, U, s, V);
  if (det3(U) < 0)
    for (int i = 0; i < 9; ++i) U[i] = -U[i];
  if (det3(V) < 0)
    for (int i = 0; i < 9; ++i) V[i] = -V[i];
  const double W[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};  // cv2's convention
  double Vt[9], Wt[9], T[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Vt[i * 3 + j] = V[j * 3 + i], Wt[i * 3 + j] = W[j * 3 + i];
  mat3_mul(U, W, T);
  mat3_mul(T, Vt, R1);
  mat3_mul(U, Wt, T);
  mat3_mul(T, Vt, R2);
  t[0] = U[2], t[1] = U[5], t[2] = U[8];
}
// cheirality of one correspondence under P1 = [I|0], P2 = [R|t]: linear triangulation (DLT 4x4 via normal equations
// smallest eigenvector), both depths positive and below `dist` (cv2.recoverPose uses 50).
RM_HDN bool cheirality_ok(const double* R, const double* t, double x1, double y1, double x2, double y2, double dist) {
  double rows[4][4] = {{-1, 0, x1, 0},
                       {0, -1, y1, 0},
                       {x2 * R[6] - R[0], x2 * R[7] - R[1], x2 * R[8] - R[2], x2 * t[2] - t[0]},
                       {y2 * R[6] - R[3], y2 * R[7] - R[4], y2 * R[8] - R[5], y2 * t[2] - t[1]}};
  double A[16], V[16], w[4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += rows[k][i] * rows[k][j];
      A[i * 4 + j] = s;
    }
  jacobi_eig<4>(A, V, w);
  int k = 0;
  for (int i = 1; i < 4; ++i)
    if (w[i] < w[k]) k = i;
  double X[4] = {V[k], V[4 + k], V[8 + k], V[12 + k]};
  if (fabs(X[3]) < 1e-300) return false;
  double px = X[0] / X[3], py = X[1] / X[3], pz = X[2] / X[3];
  double z2 = R[6] * px + R[7] * py + R[8] * pz + t[2];
  return pz > 0 && pz < dist && z2 > 0 && z2 < dist;
}

// ---- counter-based RNG (per call seed, per sample stream) -------------------------------------------------------
RM_HD unsigned long long splitmix64(unsigned long long& s) {
  unsigned long long z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// m distinct indices in [0, n)
RM_HDN void sample_distinct(unsigned long long seed, unsigned long long stream, int n, int m, int* out) {
  unsigned long long s = seed * 0xD1342543DE82EF95ull + stream * 0x2545F4914F6CDD1Dull + 0x1234567ull;
  for (int i = 0; i < m; ++i) {
    int v;
    bool dup;
    do {
      v = (int)(splitmix64(s) % (unsigned long long)n);
      dup = false;
      for (int j = 0; j < i; ++j) dup |= (out[j] == v);
    } while (dup);
    out[i] = v;
  }
}

}  // namespace rmath
