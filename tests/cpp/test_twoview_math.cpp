// Host build of gtsfm_b200/csrc/twoview_math.cuh (the source the device two-view refinement compiles), driven from
// tests/test_twoview_ba_cpu.py: one command per stdin line, one line of %.17g numbers out per command.
//   dlt  P0[12] P1[12] uv0[2] uv1[2]          -> ok X[3]
//   proj R[9] t[3] cal[5] p[3]                -> z uv[2] Jc[18] Jp[6]
//   tri  R0[9] t0[3] cal0[5] R1[9] t1[3] cal1[5] uv[4] thr angle -> ok X[3]
//   exp  R[9] t[3] d[6]                       -> R'[9] t'[3]   (Pose3::retract)
//   log  R[9] t[3]                            -> xi[6]         (Pose3::Logmap)
#include <stdio.h>
#include <string.h>

#include "../../gtsfm_b200/csrc/twoview_math.cuh"

using namespace tvmath;

static bool rd(double* v, int n) {
  for (int i = 0; i < n; ++i)
    if (scanf("%lf", v + i) != 1) return false;
  return true;
}
static void wr(const double* v, int n) {
  for (int i = 0; i < n; ++i) printf(" %.17g", v[i]);
}

int main() {
  char cmd[16];
  while (scanf("%15s", cmd) == 1) {
    if (!strcmp(cmd, "dlt")) {
      double P0[12], P1[12], a[2], b[2], X[3] = {0, 0, 0};
      if (!rd(P0, 12) || !rd(P1, 12) || !rd(a, 2) || !rd(b, 2)) return 2;
      const bool ok = dlt(P0, P1, a, b, X);
      printf("%d", ok ? 1 : 0);
      wr(X, 3);
    } else if (!strcmp(cmd, "proj")) {
      double R[9], t[3], cal[5], p[3], uv[2], Jc[18], Jp[6];
      if (!rd(R, 9) || !rd(t, 3) || !rd(cal, 5) || !rd(p, 3)) return 2;
      const double z = project(R, t, cal, p, uv, Jc, Jp);
      printf("%.17g", z);
      wr(uv, 2), wr(Jc, 18), wr(Jp, 6);
    } else if (!strcmp(cmd, "tri")) {
      Cam c[2];
      double uv[4], thr, ang, X[3] = {0, 0, 0};
      for (int k = 0; k < 2; ++k)
        if (!rd(c[k].R, 9) || !rd(c[k].t, 3) || !rd(c[k].cal, 5)) return 2;
      if (!rd(uv, 4) || !rd(&thr, 1) || !rd(&ang, 1)) return 2;
      const bool ok = triangulate(c, uv, thr, ang, X);
      printf("%d", ok ? 1 : 0);
      wr(X, 3);
    } else if (!strcmp(cmd, "exp")) {
      double R[9], t[3], d[6];
      if (!rd(R, 9) || !rd(t, 3) || !rd(d, 6)) return 2;
      retract_pose(R, t, d);
      wr(R, 9), wr(t, 3);
    } else if (!strcmp(cmd, "log")) {
      double R[9], t[3], xi[6];
      if (!rd(R, 9) || !rd(t, 3)) return 2;
      se3_log(R, t, xi);
      wr(xi, 6);
    } else {
      return 3;
    }
    printf("\n");
  }
  return 0;
}
