// fp64 maths of 1DSfM's per-direction MFAS (gtsam's MFAS::computeOutlierWeights, as the reference's
// averaging_1dsfm.py:216-232 calls it), usable from host and device: the device build is mfas.cu (compiled with
// -fmad=false), the host build is the harness tests/cpp/test_mfas_math.cpp.  oracle/mfas_ref.py states the same in NumPy.
//
// Nodes are dense ids in gtsam key order (cameras, then landmarks) and edges come in std::map<KeyPair> order, i.e.
// strictly increasing in (a, b).  For one projection direction d:
//   edge_weight   w = m . d as (mx*dx + my*dy) + mz*dz, no contraction; the edge points a -> b when w >= 0, else b -> a
//   pick_key      +inf for a node with inWeightSum < 1e-8 (a source), else (out + 1) / (in + 1)
//   better        the greedy picks the largest key; a tie (several sources, or equal ratios) goes to the lowest id, where
//                 gtsam takes the first node in its unordered_map's hash order
// Removing the picked node subtracts each live neighbour's edge |w| from that neighbour's in- or out-sum.  An edge s -> d
// is violated when d is removed before s; its outlier weight is then |w|, else 0.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define MFAS_HD __host__ __device__ __forceinline__
#else
#define MFAS_HD inline
#endif

namespace mfas {

constexpr double SOURCE_IN_WEIGHT = 1e-8;  // MFAS.cpp: a node whose inWeightSum is below this is a source

MFAS_HD double edge_weight(const double* m, const double* d) {
  const double xy = m[0] * d[0] + m[1] * d[1];
  return xy + m[2] * d[2];
}

MFAS_HD double pick_key(double in, double out) { return in < SOURCE_IN_WEIGHT ? INFINITY : (out + 1.0) / (in + 1.0); }

// (key a, id ia) is picked before (key b, id ib)
MFAS_HD bool better(double a, int ia, double b, int ib) { return a > b || (a == b && ia < ib); }

// Node v's initial (in, out) sums: its incident edges inc[0..n) in map order, as gtsam's graphFromEdges adds them.
MFAS_HD void node_sums(int v, const int32_t* inc, int n, const int32_t* ea, const double* meas, const double* d, double* in,
                       double* out) {
  double si = 0.0, so = 0.0;
  for (int k = 0; k < n; ++k) {
    const int e = inc[k];
    const double w = edge_weight(meas + 3 * (int64_t)e, d);
    const bool v_is_a = ea[e] == v;
    if ((w >= 0.0) == v_is_a) so += fabs(w);  // v is the source
    else si += fabs(w);
  }
  *in = si;
  *out = so;
}

#ifndef __CUDA_ARCH__
// The plain sequential greedy for one direction (O(V^2); the host test's statement of what the kernel computes).
// inc_off [V + 1] / inc_edge: each node's incident edges in map order.  -> order [V] (node removed at each step) and
// violated [E] (0/1).
inline void greedy(int V, int E, const int32_t* ea, const int32_t* eb, const double* meas, const int32_t* inc_off,
                   const int32_t* inc_edge, const double* d, int32_t* order, uint8_t* violated) {
  double* in = new double[V > 0 ? V : 1];
  double* out = new double[V > 0 ? V : 1];
  int32_t* pos = new int32_t[V > 0 ? V : 1];
  for (int v = 0; v < V; ++v) {
    node_sums(v, inc_edge + inc_off[v], inc_off[v + 1] - inc_off[v], ea, meas, d, in + v, out + v);
    pos[v] = -1;
  }
  for (int step = 0; step < V; ++step) {
    int u = -1;
    double best = -INFINITY;
    for (int v = 0; v < V; ++v) {
      if (pos[v] >= 0) continue;
      const double k = pick_key(in[v], out[v]);
      if (u < 0 || better(k, v, best, u)) u = v, best = k;
    }
    pos[u] = step;
    order[step] = u;
    for (int k = inc_off[u]; k < inc_off[u + 1]; ++k) {
      const int e = inc_edge[k];
      const int v = ea[e] == u ? eb[e] : ea[e];
      if (pos[v] >= 0) continue;
      const double w = edge_weight(meas + 3 * (int64_t)e, d);
      const bool u_is_source = (w >= 0.0) == (ea[e] == u);
      if (u_is_source) in[v] -= fabs(w);
      else out[v] -= fabs(w);
    }
  }
  for (int e = 0; e < E; ++e) {
    const double w = edge_weight(meas + 3 * (int64_t)e, d);
    const int s = w >= 0.0 ? ea[e] : eb[e], t = w >= 0.0 ? eb[e] : ea[e];
    violated[e] = pos[t] < pos[s];
  }
  delete[] in;
  delete[] out;
  delete[] pos;
}
#endif

}  // namespace mfas
