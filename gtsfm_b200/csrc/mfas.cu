// 1DSfM's outlier rejection for sm_90a: gtsam's MFAS outlier weights for every projection direction of
// TranslationAveraging1DSFM.compute_inliers (gtsfm/averaging/translation/averaging_1dsfm.py:234-296), and their sum over
// the directions, fp64, compiled with -fmad=false.  The per-direction maths is mfas_math.cuh; oracle/mfas_ref.py states
// the same in NumPy.
//
//   k_mfas_order  one warp per direction.  The node state (in- and out-sums, the pick key, the removal step) and a
//                 32-ary tournament tree over the pick keys live in the direction's slice of the workspace (global memory:
//                 at the sizes 1DSfM runs, tens of thousands of nodes, a direction's state does not fit shared memory).
//                 Each step takes the tree's root, removes that node, subtracts its edges from its live neighbours (each
//                 neighbour once, through the CSR of incident edges) and recomputes only the tree paths of the changed
//                 leaves: O((V + E) log32 V) per direction, not gtsam's O(V^2).  Writes the violated-edge bitmask.
//   k_mfas_sum    one thread per edge: walks the chunk's directions in order and adds |m . d_k| where edge e was
//                 violated, onto the sum carried over from the previous chunk: the reference's summation order, without
//                 K x E doubles in memory.
// Directions are cut into chunks under "mfas_workspace_mb"; each direction's ordering does not depend on its chunk, and the
// sums carry across chunks, so a chunked run returns the bits of an unchunked one.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "common.cuh"
#include "mfas_math.cuh"
#include "../../include/gtsfm_b200.h"

namespace {
constexpr int MF_WARPS = 4;       // directions per CTA of k_mfas_order
constexpr int MF_SUM_THREADS = 256;
constexpr int MF_MAX_LEVELS = 7;  // tree levels above the leaves: 32^6 = 2^30 >= V
constexpr unsigned FULL = 0xffffffffu;

struct MfasChunk {
  const int32_t* ea;
  const int32_t* eb;
  const double* meas;       // [E][3]
  const int32_t* inc_off;   // [V + 1]
  const int32_t* inc_edge;  // [2E]: each node's incident edges in map order
  const double* dirs;       // [Kc][3]
  char* ws;                 // [Kc] slices of ws_stride bytes
  uint32_t* violated;       // [Kc][W]
  int32_t* order;           // [Kc][V] or NULL
  int64_t ws_stride;
  int64_t off_out, off_leaf, off_pos;
  int64_t off_r[MF_MAX_LEVELS + 1], off_id[MF_MAX_LEVELS + 1];  // level l >= 1: best key and its node of each group of 32
  int n[MF_MAX_LEVELS + 1];                                     // entries per level; n[0] = V
  int L;                                                        // levels above the leaves; n[L] <= 32
  int V, E, W, Kc;
};

__device__ __forceinline__ void warp_best(double& r, int& id) {
  for (int o = 16; o; o >>= 1) {
    const double r2 = __shfl_xor_sync(FULL, r, o);
    const int i2 = __shfl_xor_sync(FULL, id, o);
    if (mfas::better(r2, i2, r, id)) r = r2, id = i2;
  }
}

// Entry c of level l (leaves at l = 0, whose node is their index); past the end: a key nothing loses to.
__device__ __forceinline__ void level_entry(const MfasChunk& c, char* base, int l, int idx, double& r, int& id) {
  if (idx >= c.n[l]) {
    r = -INFINITY, id = 0x7fffffff;
  } else if (l == 0) {
    r = reinterpret_cast<const double*>(base + c.off_leaf)[idx], id = idx;
  } else {
    r = reinterpret_cast<const double*>(base + c.off_r[l])[idx], id = reinterpret_cast<const int*>(base + c.off_id[l])[idx];
  }
}

// Recompute entry p of level l >= 1 from its 32 children (the whole warp; lane 0 writes).
__device__ __forceinline__ void refresh(const MfasChunk& c, char* base, int l, int p, int lane) {
  double r;
  int id;
  level_entry(c, base, l - 1, 32 * p + lane, r, id);
  warp_best(r, id);
  if (lane == 0) {
    reinterpret_cast<double*>(base + c.off_r[l])[p] = r;
    reinterpret_cast<int*>(base + c.off_id[l])[p] = id;
  }
  __syncwarp();
}

__global__ void __launch_bounds__(MF_WARPS * 32) k_mfas_order(MfasChunk c) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * MF_WARPS + (threadIdx.x >> 5);
  if (k >= c.Kc) return;
  char* base = c.ws + (int64_t)k * c.ws_stride;
  double* in = reinterpret_cast<double*>(base);
  double* out = reinterpret_cast<double*>(base + c.off_out);
  double* leaf = reinterpret_cast<double*>(base + c.off_leaf);
  int* pos = reinterpret_cast<int*>(base + c.off_pos);
  const double d[3] = {c.dirs[3 * k], c.dirs[3 * k + 1], c.dirs[3 * k + 2]};

  for (int v = lane; v < c.V; v += 32) {
    double si, so;
    mfas::node_sums(v, c.inc_edge + c.inc_off[v], c.inc_off[v + 1] - c.inc_off[v], c.ea, c.meas, d, &si, &so);
    in[v] = si, out[v] = so, leaf[v] = mfas::pick_key(si, so), pos[v] = -1;
  }
  __syncwarp();
  for (int l = 1; l <= c.L; ++l)
    for (int p = 0; p < c.n[l]; ++p) refresh(c, base, l, p, lane);

  for (int step = 0; step < c.V; ++step) {
    double r;
    int u;
    level_entry(c, base, c.L, lane, r, u);
    warp_best(r, u);
    if (lane == 0) {
      pos[u] = step;
      leaf[u] = -INFINITY;
      if (c.order) c.order[(int64_t)k * c.V + step] = u;
    }
    __syncwarp();
    // item 0 is u itself (its leaf changed), item t >= 1 its t-th incident edge; 32 items per round
    const int e0 = c.inc_off[u], deg = c.inc_off[u + 1] - e0;
    for (int t0 = 0; t0 <= deg; t0 += 32) {
      const int t = t0 + lane;
      int dirty = -1;
      if (t == 0) {
        dirty = u;
      } else if (t <= deg) {
        const int e = c.inc_edge[e0 + t - 1];
        const int v = c.ea[e] == u ? c.eb[e] : c.ea[e];
        if (pos[v] < 0) {
          const double w = mfas::edge_weight(c.meas + 3 * (int64_t)e, d);
          if ((w >= 0.0) == (c.ea[e] == u)) in[v] -= fabs(w);  // u -> v: v loses in-weight
          else out[v] -= fabs(w);
          leaf[v] = mfas::pick_key(in[v], out[v]);
          dirty = v;
        }
      }
      __syncwarp();
      for (int l = 1; l <= c.L; ++l) {  // the parents of this round's dirty entries, each group refreshed once
        const int parent = dirty >= 0 ? dirty >> 5 : -1;
        const unsigned same = __match_any_sync(FULL, parent);
        const bool leader = parent >= 0 && (__ffs(same) - 1) == lane;
        unsigned todo = __ballot_sync(FULL, leader);
        while (todo) {
          const int src = __ffs(todo) - 1;
          todo &= todo - 1;
          refresh(c, base, l, __shfl_sync(FULL, parent, src), lane);
        }
        dirty = leader ? parent : -1;
      }
    }
  }

  uint32_t* vk = c.violated + (int64_t)k * c.W;
  for (int e0 = 0; e0 < c.E; e0 += 32) {
    const int e = e0 + lane;
    bool bad = false;
    if (e < c.E) {
      const double w = mfas::edge_weight(c.meas + 3 * (int64_t)e, d);
      const int s = w >= 0.0 ? c.ea[e] : c.eb[e], t = w >= 0.0 ? c.eb[e] : c.ea[e];
      bad = pos[t] < pos[s];
    }
    const unsigned word = __ballot_sync(FULL, bad);
    if (lane == 0) vk[e0 >> 5] = word;
  }
}

__global__ void __launch_bounds__(MF_SUM_THREADS) k_mfas_sum(const double* meas, const double* dirs, const uint32_t* violated,
                                                           int E, int W, int Kc, double* sum) {
  const int e = blockIdx.x * MF_SUM_THREADS + threadIdx.x;
  if (e >= E) return;
  const double m[3] = {meas[3 * (int64_t)e], meas[3 * (int64_t)e + 1], meas[3 * (int64_t)e + 2]};
  double s = sum[e];
  for (int k = 0; k < Kc; ++k)
    if ((violated[(int64_t)k * W + (e >> 5)] >> (e & 31)) & 1u) s += fabs(mfas::edge_weight(m, dirs + 3 * k));
  sum[e] = s;
}
}  // namespace

struct MfasState {
  DevBuf ea, eb, meas, inc_off, inc_edge, dirs, ws, violated, order, sum;
};

void mf_destroy(b2_context* ctx) {
  delete ctx->mf;
  ctx->mf = nullptr;
}

extern "C" int b2_mfas_outlier_weights_host(b2_context* ctx, int V, int E, const int32_t* edge_a, const int32_t* edge_b,
                                            const double* meas, int K, const double* dirs, double* weight_sum, int32_t* order_out,
                                            uint32_t* violated_out, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (V < 0 || E < 0 || K < 0) return b2_fail(ctx, B2_ERR_ARG, "mfas: V, E and K must be >= 0");
  if (V > (1 << 30) || E > (1 << 29)) return b2_fail(ctx, B2_ERR_ARG, "mfas: at most 2^30 nodes and 2^29 edges");
  if (E > 0 && (!edge_a || !edge_b || !meas || !weight_sum)) return b2_fail(ctx, B2_ERR_ARG, "mfas: an edge array is NULL");
  if (K > 0 && !dirs) return b2_fail(ctx, B2_ERR_ARG, "mfas: dirs is NULL");
  std::vector<uint64_t> pairs((size_t)E);
  for (int e = 0; e < E; ++e) {
    const int a = edge_a[e], b = edge_b[e];
    if (a < 0 || a >= V || b < 0 || b >= V) return b2_fail(ctx, B2_ERR_ARG, "mfas: an edge's node id is outside [0, V)");
    if (a == b) return b2_fail(ctx, B2_ERR_ARG, "mfas: an edge from a node to itself");
    if (e > 0 && (a < edge_a[e - 1] || (a == edge_a[e - 1] && b <= edge_b[e - 1])))
      return b2_fail(ctx, B2_ERR_ARG, "mfas: edges must be strictly increasing in (a, b)");
    pairs[e] = (uint64_t)std::min(a, b) << 32 | (uint32_t)std::max(a, b);
    for (int j = 0; j < 3; ++j)
      if (!isfinite(meas[3 * (int64_t)e + j])) return b2_fail(ctx, B2_ERR_ARG, "mfas: a measurement is not finite");
  }
  std::sort(pairs.begin(), pairs.end());
  if (std::adjacent_find(pairs.begin(), pairs.end()) != pairs.end())
    return b2_fail(ctx, B2_ERR_ARG, "mfas: the same node pair is given twice, as (a, b) and (b, a)");
  for (int64_t j = 0; j < 3 * (int64_t)K; ++j)
    if (!isfinite(dirs[j])) return b2_fail(ctx, B2_ERR_ARG, "mfas: a direction is not finite");
  for (int e = 0; e < E; ++e) weight_sum[e] = 0.0;
  if (V == 0 || K == 0) return B2_OK;

  // each node's incident edges in map order: the order gtsam's graphFromEdges adds them in
  std::vector<int32_t> inc_off((size_t)V + 1, 0), inc_edge(2 * (size_t)E), fill((size_t)V);
  for (int e = 0; e < E; ++e) ++inc_off[edge_a[e] + 1], ++inc_off[edge_b[e] + 1];
  for (int v = 0; v < V; ++v) inc_off[v + 1] += inc_off[v];
  for (int v = 0; v < V; ++v) fill[v] = inc_off[v];
  for (int e = 0; e < E; ++e) inc_edge[fill[edge_a[e]]++] = e, inc_edge[fill[edge_b[e]]++] = e;

  MfasChunk c{};
  c.V = V, c.E = E, c.W = (E + 31) / 32;
  c.n[0] = V;
  while (c.n[c.L] > 32) ++c.L, c.n[c.L] = (c.n[c.L - 1] + 31) / 32;
  auto al = [](int64_t x) { return (x + 15) & ~(int64_t)15; };
  int64_t o = al(8 * (int64_t)V);
  c.off_out = o, o = al(o + 8 * (int64_t)V);
  c.off_leaf = o, o = al(o + 8 * (int64_t)V);
  c.off_pos = o, o = al(o + 4 * (int64_t)V);
  for (int l = 1; l <= c.L; ++l) c.off_r[l] = o, o = al(o + 8 * (int64_t)c.n[l]), c.off_id[l] = o, o = al(o + 4 * (int64_t)c.n[l]);
  c.ws_stride = o;
  const int64_t per_dir = c.ws_stride + 4 * (int64_t)c.W + (order_out ? 4 * (int64_t)V : 0) + 24;
  const int64_t budget = (int64_t)ctx->mf_workspace_mb << 20;
  const int Kc = (int)std::max<int64_t>(1, std::min<int64_t>(K, budget / per_dir));

  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  if (!ctx->mf) ctx->mf = new MfasState();
  MfasState* s = ctx->mf;
  const size_t e1 = std::max(1, E);
  B2_CUDA(ctx, s->ea.ensure(e1 * 4));
  B2_CUDA(ctx, s->eb.ensure(e1 * 4));
  B2_CUDA(ctx, s->meas.ensure(e1 * 24));
  B2_CUDA(ctx, s->sum.ensure(e1 * 8));
  B2_CUDA(ctx, s->inc_off.ensure(((size_t)V + 1) * 4));
  B2_CUDA(ctx, s->inc_edge.ensure(2 * e1 * 4));
  B2_CUDA(ctx, s->dirs.ensure((size_t)Kc * 24));
  B2_CUDA(ctx, s->ws.ensure((size_t)Kc * c.ws_stride));
  B2_CUDA(ctx, s->violated.ensure((size_t)Kc * std::max(1, c.W) * 4));
  if (order_out) B2_CUDA(ctx, s->order.ensure((size_t)Kc * V * 4));
  if (E > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(s->ea.p, edge_a, (size_t)E * 4, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->eb.p, edge_b, (size_t)E * 4, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->meas.p, meas, (size_t)E * 24, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->inc_edge.p, inc_edge.data(), 2 * (size_t)E * 4, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemsetAsync(s->sum.p, 0, (size_t)E * 8, st));
  }
  B2_CUDA(ctx, cudaMemcpyAsync(s->inc_off.p, inc_off.data(), ((size_t)V + 1) * 4, cudaMemcpyHostToDevice, st));
  c.ea = s->ea.as<int32_t>(), c.eb = s->eb.as<int32_t>(), c.meas = s->meas.as<double>();
  c.inc_off = s->inc_off.as<int32_t>(), c.inc_edge = s->inc_edge.as<int32_t>();
  c.dirs = s->dirs.as<double>(), c.ws = s->ws.as<char>(), c.violated = s->violated.as<uint32_t>();
  c.order = order_out ? s->order.as<int32_t>() : nullptr;
  for (int k0 = 0; k0 < K; k0 += Kc) {
    c.Kc = std::min(Kc, K - k0);
    B2_CUDA(ctx, cudaMemcpyAsync(s->dirs.p, dirs + 3 * (int64_t)k0, (size_t)c.Kc * 24, cudaMemcpyHostToDevice, st));
    B2_LAUNCH(ctx, k_mfas_order, (unsigned)((c.Kc + MF_WARPS - 1) / MF_WARPS), MF_WARPS * 32, 0, st, c);
    B2_CHECK_LAUNCH(ctx);
    if (E > 0) {
      B2_LAUNCH(ctx, k_mfas_sum, (unsigned)((E + MF_SUM_THREADS - 1) / MF_SUM_THREADS), MF_SUM_THREADS, 0, st, c.meas, c.dirs,
                c.violated, E, c.W, c.Kc, s->sum.as<double>());
      B2_CHECK_LAUNCH(ctx);
    }
    if (violated_out && c.W > 0)
      B2_CUDA(ctx, cudaMemcpyAsync(violated_out + (int64_t)k0 * c.W, c.violated, (size_t)c.Kc * c.W * 4, cudaMemcpyDeviceToHost, st));
    if (order_out)
      B2_CUDA(ctx, cudaMemcpyAsync(order_out + (int64_t)k0 * V, c.order, (size_t)c.Kc * V * 4, cudaMemcpyDeviceToHost, st));
  }
  if (E > 0) B2_CUDA(ctx, cudaMemcpyAsync(weight_sum, s->sum.p, (size_t)E * 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B2_OK;
}
