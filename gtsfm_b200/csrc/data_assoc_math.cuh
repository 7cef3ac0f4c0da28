// fp64 per-track pieces of data association's triangulation (gtsfm/data_association/point3d_initializer.py:139-295), usable
// from host and device: the device build is data_assoc.cu, the host build the unit-test harness
// tests/cpp/test_triangulation_math.cpp.  oracle/data_assoc_ref.py states the same maths in NumPy.
//
// A track is n measurements (image, uv).  RANSAC_SAMPLE_UNIFORM draws min(num_hypotheses, C(n, 2)) measurement pairs
// without replacement; each pair index follows the lexicographic order of itertools.combinations(range(n), 2).  When
// C(n, 2) <= num_hypotheses every pair is drawn, hypothesis h taking pair h.  Otherwise hypothesis h takes pair pi(h),
// pi a bijection of [0, C(n, 2)) keyed by (seed, the track's position in the input): a 4-round Feistel network on the
// smallest even bit width that covers C(n, 2), cycle-walked back into range.  Each hypothesis finds its pair alone.
#pragma once
#include <stdint.h>

#include "twoview_math.cuh"

namespace damath {

using tvmath::Cam;

enum ExitCode {  // TriangulationExitCode
  SUCCESS = 0,
  CHEIRALITY_FAILURE = 1,
  INLIERS_UNDERCONSTRAINED = 2,
  POSES_UNDERCONSTRAINED = 3,
  EXCEEDS_REPROJ_THRESH = 4,
  LOW_TRIANGULATION_ANGLE = 5,
};

// splitmix64's finaliser
TV_HD uint64_t mix64(uint64_t x) {
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}

TV_HD uint64_t sampler_key(uint64_t seed, uint64_t track) { return mix64(seed ^ mix64(track + 0x9e3779b97f4a7c15ull)); }

// Pair index of hypothesis h of a track with `pairs` = C(n, 2) pairs and `hyps` = min(num_hypotheses, pairs) hypotheses
TV_HD int64_t sample_pair(uint64_t key, int64_t h, int64_t pairs, int64_t hyps) {
  if (hyps >= pairs) return h;
  int bits = 1;
  while ((1ll << bits) < pairs) ++bits;
  const int half = (bits + 1) / 2;
  const uint64_t mask = (1ull << half) - 1ull;
  uint64_t x = (uint64_t)h;
  do {
    uint64_t L = x >> half, R = x & mask;
    for (uint64_t r = 0; r < 4; ++r) {
      const uint64_t F = mix64(key ^ (r * 0xd6e8feb86659fd93ull) ^ R) & mask;
      const uint64_t nl = R;
      R = L ^ F, L = nl;
    }
    x = (L << half) | R;
  } while (x >= (uint64_t)pairs);
  return (int64_t)x;
}

// Pair index p -> (k1, k2), k1 < k2 < n, in itertools.combinations order
TV_HD void pair_of(int64_t p, int n, int* k1, int* k2) {
  int a = 0;
  while (p >= n - 1 - a) p -= n - 1 - a, ++a;
  *k1 = a, *k2 = a + 1 + (int)p;
}

// projectSafe's reprojection error of X in camera c (NaN: no camera, or a depth <= 0), as
// reprojection.compute_point_reprojection_errors
TV_HD double reproj_error(const Cam* c, const double* uv, const double* X) {
  if (!c) return NAN;
  double pr[2];
  if (!(tvmath::project(c->R, c->t, c->cal, X, pr, nullptr, nullptr) > 0.0)) return NAN;
  const double du = uv[0] - pr[0], dv = uv[1] - pr[1];
  return sqrt(du * du + dv * dv);
}

// gtsam.triangulatePoint3(rank_tol=1e-9, optimize=True) on the views, throwing nothing: false where it raises (DLT rank
// below 3, a point at infinity, a point behind a camera after refinement)
template <class Views>
TV_HD bool triangulate_views(const Views& v, double* X) {
  if (!tvmath::dlt_views(v, X)) return false;
  tvmath::refine_point_views(v, X);
  for (int k = 0; k < v.size(); ++k) {
    double pr[2];
    const Cam& c = v.cam(k);
    if (!(tvmath::project(c.R, c.t, c.cal, X, pr, nullptr, nullptr) > 0.0)) return false;
  }
  return true;
}

// Two measurements of a track as views
struct PairViews {
  const Cam* c[2];
  const double* u[2];
  TV_HD int size() const { return 2; }
  TV_HD const Cam& cam(int k) const { return *c[k]; }
  TV_HD const double* uv(int k) const { return u[k]; }
  TV_HD double cost(const double* X) const {
    double r[4];
    tvmath::tri_resid1(*c[0], u[0], X, r, nullptr);
    tvmath::tri_resid1(*c[1], u[1], X, r + 2, nullptr);
    return 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
  }
};

// The views of a list of measurement indices sel[0..n) into (camera of measurement, uv): cams[cam_of[i]]
struct ListViews {
  const Cam* cams;
  const int32_t* cam_of;
  const double* uvs;  // [M][2]
  const int32_t* sel;
  int n;
  TV_HD int size() const { return n; }
  TV_HD const Cam& cam(int k) const { return cams[cam_of[sel[k]]]; }
  TV_HD const double* uv(int k) const { return uvs + 2 * (int64_t)sel[k]; }
  TV_HD double cost(const double* X) const {
    double s = 0.0;
    for (int k = 0; k < n; ++k) {
      double r[2];
      tvmath::tri_resid1(cam(k), uv(k), X, r, nullptr);
      s += r[0] * r[0];
      s += r[1] * r[1];
    }
    return 0.5 * s;
  }
};

// get_max_triangulation_angle >= min_angle_deg for the cameras of the views: the angle between Unit3(X - centre) of two
// views, in degrees (compute_relative_unit_translation_angle)
template <class Views>
TV_HD bool angle_at_least(const Views& v, const double* X, double min_angle_deg) {
  if (!(min_angle_deg > 0.0)) return true;
  for (int a = 0; a < v.size(); ++a) {
    double ra[3], na = 0.0;
    for (int i = 0; i < 3; ++i) ra[i] = X[i] - v.cam(a).t[i], na += ra[i] * ra[i];
    na = sqrt(na);
    for (int b = a + 1; b < v.size(); ++b) {
      double rb[3], nb = 0.0, dot = 0.0;
      for (int i = 0; i < 3; ++i) rb[i] = X[i] - v.cam(b).t[i], nb += rb[i] * rb[i];
      nb = sqrt(nb);
      for (int i = 0; i < 3; ++i) dot += (ra[i] / na) * (rb[i] / nb);
      const double ang = acos(fmin(1.0, fmax(-1.0, dot))) * (180.0 / M_PI);
      if (!(ang < min_angle_deg)) return true;
    }
  }
  return false;
}

}  // namespace damath
