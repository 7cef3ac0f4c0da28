// Host build of gtsfm_b200/csrc/mfas_math.cuh (the per-direction maths k_mfas_order compiles), driven from
// tests/test_mfas_cpu.py.  stdin: V E K, then E lines "a b mx my mz" (map order), then K lines "dx dy dz" (%.17g).
// stdout per direction: the V node ids in removal order, then the E violated flags.
#include <stdio.h>

#include <vector>

#include "../../gtsfm_b200/csrc/mfas_math.cuh"

int main() {
  int V, E, K;
  if (scanf("%d %d %d", &V, &E, &K) != 3) return 2;
  std::vector<int32_t> ea(E), eb(E), off(V + 1, 0), inc(2 * (size_t)E), fill(V);
  std::vector<double> meas(3 * (size_t)E), d(3);
  for (int e = 0; e < E; ++e)
    if (scanf("%d %d %lf %lf %lf", &ea[e], &eb[e], &meas[3 * e], &meas[3 * e + 1], &meas[3 * e + 2]) != 5) return 2;
  for (int e = 0; e < E; ++e) ++off[ea[e] + 1], ++off[eb[e] + 1];
  for (int v = 0; v < V; ++v) off[v + 1] += off[v], fill[v] = off[v];
  for (int e = 0; e < E; ++e) inc[fill[ea[e]]++] = e, inc[fill[eb[e]]++] = e;
  std::vector<int32_t> order(V);
  std::vector<uint8_t> bad(E);
  for (int k = 0; k < K; ++k) {
    if (scanf("%lf %lf %lf", &d[0], &d[1], &d[2]) != 3) return 2;
    mfas::greedy(V, E, ea.data(), eb.data(), meas.data(), off.data(), inc.data(), d.data(), order.data(), bad.data());
    for (int v = 0; v < V; ++v) printf("%d ", order[v]);
    printf("\n");
    for (int e = 0; e < E; ++e) printf("%d ", bad[e]);
    printf("\n");
  }
  return 0;
}
