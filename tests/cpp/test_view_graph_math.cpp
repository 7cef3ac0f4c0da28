// Host build of gtsfm_b200/csrc/view_graph_math.cuh (the cycle error k_vg_count and k_vg_fill compile), driven from
// tests/test_view_graph_cpu.py: one triplet per stdin line, R01[9] R12[9] R02[9] (row-major), one %.17g error out per line.
#include <stdio.h>

#include "../../gtsfm_b200/csrc/view_graph_math.cuh"

int main() {
  double R[27];
  for (;;) {
    for (int i = 0; i < 27; ++i)
      if (scanf("%lf", R + i) != 1) return i == 0 ? 0 : 2;
    printf("%.17g\n", vgraph::cycle_error_deg(R, R + 9, R + 18));
  }
}
