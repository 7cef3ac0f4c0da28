// Host build of gtsfm_b200/csrc/data_assoc_math.cuh and the n-view DLT of twoview_math.cuh (what k_da_hyp and k_da_track
// compile), driven from tests/test_data_assoc_cpu.py: one command per stdin line, one line of %.17g numbers out.
//   pair seed track pairs hyps          -> the pair index of every hypothesis
//   dlt2 cam0[17] cam1[17] uv[4]         -> ok X[3] of dlt, then ok X[3] of dlt_views on the same two views
//   qr   m rows[m][4]                    -> the 4 singular values of the QR-reduced system, ascending, then its null vector
//                                           (unit, last entry >= 0)
//   tri  n cams[n][17] uv[n][2]          -> ok X[3] of triangulate_views
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../gtsfm_b200/csrc/data_assoc_math.cuh"

using tvmath::Cam;

static bool rd(double* v, int n) {
  for (int i = 0; i < n; ++i)
    if (scanf("%lf", v + i) != 1) return false;
  return true;
}
static void wr(const double* v, int n) {
  for (int i = 0; i < n; ++i) printf(" %.17g", v[i]);
}
static bool rd_cam(Cam& c) { return rd(c.R, 9) && rd(c.t, 3) && rd(c.cal, 5); }

struct VecViews {
  const std::vector<Cam>* cams;
  const std::vector<double>* uvs;
  int size() const { return (int)cams->size(); }
  const Cam& cam(int k) const { return (*cams)[k]; }
  const double* uv(int k) const { return uvs->data() + 2 * k; }
  double cost(const double* X) const {
    double s = 0.0;
    for (int k = 0; k < size(); ++k) {
      double r[2];
      tvmath::tri_resid1(cam(k), uv(k), X, r, nullptr);
      s += r[0] * r[0];
      s += r[1] * r[1];
    }
    return 0.5 * s;
  }
};

int main() {
  char cmd[16];
  while (scanf("%15s", cmd) == 1) {
    if (!strcmp(cmd, "pair")) {
      unsigned long long seed, track;
      long long pairs, hyps;
      if (scanf("%llu %llu %lld %lld", &seed, &track, &pairs, &hyps) != 4) return 2;
      const uint64_t key = damath::sampler_key(seed, track);
      for (long long h = 0; h < hyps; ++h) printf("%s%lld", h ? " " : "", (long long)damath::sample_pair(key, h, pairs, hyps));
    } else if (!strcmp(cmd, "dlt2")) {
      Cam c[2];
      double uv[4], P0[12], P1[12], X[3] = {0, 0, 0}, Y[3] = {0, 0, 0};
      if (!rd_cam(c[0]) || !rd_cam(c[1]) || !rd(uv, 4)) return 2;
      tvmath::projection_matrix(c[0].R, c[0].t, c[0].cal, P0);
      tvmath::projection_matrix(c[1].R, c[1].t, c[1].cal, P1);
      const bool a = tvmath::dlt(P0, P1, uv, uv + 2, X);
      const bool b = tvmath::dlt_views(tvmath::TwoViews{c, uv}, Y);
      printf("%d", a ? 1 : 0), wr(X, 3), printf(" %d", b ? 1 : 0), wr(Y, 3);
    } else if (!strcmp(cmd, "qr")) {
      int m;
      if (scanf("%d", &m) != 1) return 2;
      double A[16] = {0}, s[4], V[16];
      for (int r = 0; r < m; ++r) {
        double a[4];
        if (!rd(a, 4)) return 2;
        tvmath::qr_fold_row(A, a);
      }
      tvmath::svd4(A, s, V);
      int o[4] = {0, 1, 2, 3};
      for (int i = 0; i < 4; ++i)
        for (int j = i + 1; j < 4; ++j)
          if (s[o[j]] < s[o[i]]) { const int x = o[i]; o[i] = o[j], o[j] = x; }
      double ss[4], v[4], nrm = 0.0;
      for (int i = 0; i < 4; ++i) ss[i] = s[o[i]], v[i] = V[i * 4 + o[0]], nrm += v[i] * v[i];
      nrm = sqrt(nrm) * (v[3] < 0 ? -1.0 : 1.0);
      for (int i = 0; i < 4; ++i) v[i] /= nrm;
      wr(ss, 4), wr(v, 4);
    } else if (!strcmp(cmd, "tri")) {
      int n;
      if (scanf("%d", &n) != 1) return 2;
      std::vector<Cam> cams(n);
      std::vector<double> uvs(2 * n);
      for (int k = 0; k < n; ++k)
        if (!rd_cam(cams[k])) return 2;
      if (!rd(uvs.data(), 2 * n)) return 2;
      double X[3] = {0, 0, 0};
      const bool ok = damath::triangulate_views(VecViews{&cams, &uvs}, X);
      printf("%d", ok ? 1 : 0), wr(X, 3);
    } else {
      return 3;
    }
    printf("\n");
    fflush(stdout);
  }
  return 0;
}
