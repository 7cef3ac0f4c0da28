// Host build of gtsfm_b200/csrc/twoview_eval.cuh (the source k_tv_eval compiles), driven from
// tests/test_twoview_report_cpu.py: one command per stdin line, one line of %.17g numbers out per command.
//   F    R1[9] t1[3] R2[9] t2[3] cal1[3] cal2[3]   -> F[9]        (ground-truth F of wTi1, wTi2)
//   samp F[9] x1 y1 x2 y2                          -> d2
//   rot  Ra[9] Rb[9]                               -> degrees
//   unit a[3] b[3]                                 -> degrees
#include <stdio.h>
#include <string.h>

#include "../../gtsfm_b200/csrc/twoview_eval.cuh"

using namespace tveval;

static bool rd(double* v, int n) {
  for (int i = 0; i < n; ++i)
    if (scanf("%lf", v + i) != 1) return false;
  return true;
}

int main() {
  char cmd[16];
  while (scanf("%15s", cmd) == 1) {
    if (!strcmp(cmd, "F")) {
      double R1[9], t1[3], R2[9], t2[3], c1[3], c2[3], R[9], t[3], F[9];
      if (!rd(R1, 9) || !rd(t1, 3) || !rd(R2, 9) || !rd(t2, 3) || !rd(c1, 3) || !rd(c2, 3)) return 2;
      gt_relative(R1, t1, R2, t2, R, t);
      gt_fundamental(R, t, c1, c2, F);
      for (int i = 0; i < 9; ++i) printf(" %.17g", F[i]);
    } else if (!strcmp(cmd, "samp")) {
      double F[9], x[4];
      if (!rd(F, 9) || !rd(x, 4)) return 2;
      printf(" %.17g", sampson_sq(F, x[0], x[1], x[2], x[3]));
    } else if (!strcmp(cmd, "rot")) {
      double a[9], b[9];
      if (!rd(a, 9) || !rd(b, 9)) return 2;
      printf(" %.17g", rotation_angle_deg(a, b));
    } else if (!strcmp(cmd, "unit")) {
      double a[3], b[3];
      if (!rd(a, 3) || !rd(b, 3)) return 2;
      printf(" %.17g", unit_angle_deg(a, b));
    } else {
      return 3;
    }
    printf("\n");
  }
  return 0;
}
