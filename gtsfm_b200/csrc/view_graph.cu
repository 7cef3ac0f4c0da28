// Cycle-consistent rotation view-graph filter for sm_90a: GTSfM's CycleConsistentRotationViewGraphEstimator.run
// (gtsfm/view_graph_estimator/cycle_consistent_rotation_estimator.py:80-157, 224-240) over the relative rotations of a
// graph's edges, fp64 throughout.  oracle/view_graph_ref.py states the same maths in NumPy.
//
// Adjacency (once per call): the 2E half-edge keys (node << B | neighbour), each carrying its edge id, are sorted by an
// LSD radix sort with 8-bit digits (k_vg_hist, the exclusive scan, k_vg_scatter; stable, so the sort is deterministic).
// A node's row is then the run of keys with its prefix, found by binary search, so nothing is indexed by node id and
// memory stays O(edges) however large the image indices are.
// Triplets: the warp of edge (a, b) walks the shorter of the two rows and binary-searches the longer; each common
// neighbour c is one triplet.  Its error is evaluated from the triplet's sorted node order by one call site, so the three
// edges of a triplet hold bit-identical values.
//   k_vg_count<false>  per edge: duplicate check and the triplet count (MEDIAN)
//   k_vg_count<true>   per edge: duplicate check, count and the running minimum of the errors (MIN: no segments)
//   k_vg_fill          MEDIAN, per chunk: the errors of the chunk's edges into their segments (offsets: exclusive scan of
//                      the counts)
//   k_vg_select        MEDIAN, per chunk: the exact median of each segment (ranked in registers up to 32 values, radix
//                      select on the uint64 bit patterns of the non-negative doubles above), the decision
// A NaN anywhere in a segment makes the aggregate NaN and rejects the edge, as np.median / np.amin and `<` do; an edge in
// no triplet is kept with aggregate NaN.
// Chunks cut the segment space into windows of "viewgraph_workspace_mb"; an edge belongs to the window holding its first
// entry, so a chunked run computes every edge's segment and aggregate exactly as an unchunked one.  The number of chunks
// is planned from the most triplets any graph with E edges can have, (sqrt(2) / 3) E^1.5 (a clique attains it), so the
// host never waits for the counts: chunks past the last segment return at once.  One synchronisation per call.
#include <math.h>
#include <string.h>

#include <string>

#include "common.cuh"
#include "view_graph_math.cuh"
#include "../../include/gtsfm_b200.h"

namespace {
typedef unsigned long long u64;
constexpr int VG_SORT_THREADS = 256, VG_SORT_ROUNDS = 8, VG_TILE = VG_SORT_THREADS * VG_SORT_ROUNDS;  // half-edges per sort CTA
constexpr int VG_SCAN_THREADS = 1024;
constexpr int VG_WARPS = 8;  // warps per CTA of the per-edge kernels (one warp per edge)
constexpr unsigned FULL = 0xffffffffu;
enum { VG_FLAG_DUP = 1, VG_FLAG_OVERFLOW = 2 };

struct VgGraph {  // the sorted adjacency
  const int* edges;
  const double* R;
  const u64* keys;
  const int* vals;
  int n, n2, B;
};
}  // namespace

// ---- adjacency: half-edges and their radix sort -----------------------------------------------------------------------
__global__ void k_vg_halfedges(const int* __restrict__ edges, int n, int B, u64* __restrict__ keys, int* __restrict__ vals) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const u64 a = (unsigned)edges[2 * e], b = (unsigned)edges[2 * e + 1];
  keys[2 * e] = (a << B) | b, vals[2 * e] = e;
  keys[2 * e + 1] = (b << B) | a, vals[2 * e + 1] = e;
}

// digit counts of one tile, digit-major: counts[d * nblk + tile], so their exclusive scan is each (digit, tile)'s base
__global__ void __launch_bounds__(VG_SORT_THREADS) k_vg_hist(const u64* __restrict__ keys, int n2, int shift,
                                                             long long* __restrict__ counts, int nblk) {
  __shared__ int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int base = blockIdx.x * VG_TILE;
  for (int r = 0; r < VG_SORT_ROUNDS; ++r) {
    const int i = base + r * VG_SORT_THREADS + threadIdx.x;
    if (i < n2) atomicAdd(&h[(keys[i] >> shift) & 255], 1);
  }
  __syncthreads();
  counts[(size_t)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

// stable scatter of one tile: in each round of 256 keys a key's rank is its rank among equal digits in its warp
// (__match_any_sync), after the earlier warps of the round and the earlier rounds of the tile
__global__ void __launch_bounds__(VG_SORT_THREADS) k_vg_scatter(const u64* __restrict__ kin, const int* __restrict__ vin,
                                                                u64* __restrict__ kout, int* __restrict__ vout, int n2, int shift,
                                                                const long long* __restrict__ offs, int nblk) {
  __shared__ int s_base[256];
  __shared__ int s_cnt[VG_SORT_THREADS / 32][256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  s_base[tid] = (int)offs[(size_t)tid * nblk + blockIdx.x];
  const int base = blockIdx.x * VG_TILE;
  for (int r = 0; r < VG_SORT_ROUNDS; ++r) {
    for (int d = tid; d < (VG_SORT_THREADS / 32) * 256; d += VG_SORT_THREADS) (&s_cnt[0][0])[d] = 0;
    __syncthreads();
    const int i = base + r * VG_SORT_THREADS + tid;
    const bool valid = i < n2;
    const u64 k = valid ? kin[i] : 0ull;
    const int dig = valid ? (int)((k >> shift) & 255) : 256;
    const unsigned peers = __match_any_sync(FULL, dig);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) s_cnt[warp][dig] = __popc(peers);
    __syncthreads();
    if (valid) {
      int pos = s_base[dig] + rank;
      for (int w = 0; w < warp; ++w) pos += s_cnt[w][dig];
      kout[pos] = k;
      vout[pos] = vin[i];
    }
    __syncthreads();
    int add = 0;
    for (int w = 0; w < VG_SORT_THREADS / 32; ++w) add += s_cnt[w][tid];
    s_base[tid] += add;
    __syncthreads();
  }
}

// ---- exclusive scan of int64 (the radix digit counts and the per-edge triplet counts) ---------------------------------
__device__ __forceinline__ long long vg_block_inclusive(long long v, long long* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(FULL, v, o);
    if (lane >= o) v += y;
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    long long w = lane < (int)(blockDim.x >> 5) ? s_warp[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(FULL, w, o);
      if (lane >= o) w += y;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  const long long r = v + (warp > 0 ? s_warp[warp - 1] : 0);
  __syncthreads();  // s_warp is reused by the next call
  return r;
}

__global__ void __launch_bounds__(VG_SCAN_THREADS) k_vg_scan_tiles(const long long* in, long long* out, long long n,
                                                                   long long* __restrict__ tile_sums) {
  __shared__ long long s_warp[32];
  const long long i = (long long)blockIdx.x * VG_SCAN_THREADS + threadIdx.x;
  const long long x = i < n ? in[i] : 0;
  const long long inc = vg_block_inclusive(x, s_warp);
  if (i < n) out[i] = inc - x;
  if (threadIdx.x == VG_SCAN_THREADS - 1) tile_sums[blockIdx.x] = inc;
}

// one CTA: the tile sums in place (exclusive); tile_sums[ntiles] = the total
__global__ void __launch_bounds__(VG_SCAN_THREADS) k_vg_scan_top(long long* __restrict__ tile_sums, int ntiles) {
  __shared__ long long s_warp[32];
  __shared__ long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int b = 0; b < ntiles; b += VG_SCAN_THREADS) {
    const int i = b + threadIdx.x;
    const long long x = i < ntiles ? tile_sums[i] : 0;
    const long long inc = vg_block_inclusive(x, s_warp);
    const long long carry = s_carry;
    if (i < ntiles) tile_sums[i] = carry + inc - x;
    __syncthreads();
    if (threadIdx.x == VG_SCAN_THREADS - 1) s_carry = carry + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) tile_sums[ntiles] = s_carry;
}

__global__ void __launch_bounds__(VG_SCAN_THREADS) k_vg_scan_add(long long* __restrict__ out, long long n,
                                                                 const long long* __restrict__ tile_sums) {
  const long long i = (long long)blockIdx.x * VG_SCAN_THREADS + threadIdx.x;
  if (i < n) out[i] += tile_sums[blockIdx.x];
}

// ---- triplets ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int vg_lower(const u64* __restrict__ keys, int lo, int hi, u64 x) {
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (keys[m] < x) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// Calls f(hit, c, e_ac, e_bc) warp-uniformly once per 32 entries of the shorter row of edge (a, b); `hit` marks the lanes
// whose neighbour c is common to a and b, in increasing c.
template <class F>
__device__ __forceinline__ void vg_for_common(const VgGraph& g, int a, int b, F&& f) {
  const int lane = threadIdx.x & 31;
  const u64 mask = (1ull << g.B) - 1ull;
  const int ra0 = vg_lower(g.keys, 0, g.n2, (u64)a << g.B), ra1 = vg_lower(g.keys, ra0, g.n2, ((u64)a + 1) << g.B);
  const int rb0 = vg_lower(g.keys, 0, g.n2, (u64)b << g.B), rb1 = vg_lower(g.keys, rb0, g.n2, ((u64)b + 1) << g.B);
  const bool a_short = ra1 - ra0 <= rb1 - rb0;
  const int s0 = a_short ? ra0 : rb0, s1 = a_short ? ra1 : rb1, l0 = a_short ? rb0 : ra0, l1 = a_short ? rb1 : ra1;
  const u64 other = (u64)(a_short ? b : a) << g.B;
  for (int p = s0; p < s1; p += 32) {
    const int q = p + lane;
    bool hit = false;
    int c = 0, e_s = 0, e_l = 0;
    if (q < s1) {
      c = (int)(g.keys[q] & mask);
      const u64 x = other | (u64)c;
      const int pos = vg_lower(g.keys, l0, l1, x);
      if (pos < l1 && g.keys[pos] == x) hit = true, e_s = g.vals[q], e_l = g.vals[pos];
    }
    f(hit, c, a_short ? e_s : e_l, a_short ? e_l : e_s);
  }
}

// the error of triplet {a, b, c} (a < b), from its sorted node order i0 < i1 < i2
__device__ __forceinline__ double vg_triplet_error(const double* __restrict__ R, int a, int b, int c, int e_ab, int e_ac, int e_bc) {
  int e01, e12, e02;
  if (c < a) e01 = e_ac, e12 = e_ab, e02 = e_bc;       // (c, a, b)
  else if (c < b) e01 = e_ac, e12 = e_bc, e02 = e_ab;  // (a, c, b)
  else e01 = e_ab, e12 = e_bc, e02 = e_ac;             // (a, b, c)
  return vgraph::cycle_error_deg(R + 9 * (size_t)e01, R + 9 * (size_t)e12, R + 9 * (size_t)e02);
}

__device__ __forceinline__ void vg_check_dup(const VgGraph& g, int a, int b, int* flags) {
  const u64 x = ((u64)a << g.B) | (u64)b;
  const int pos = vg_lower(g.keys, 0, g.n2, x);
  if (pos + 1 < g.n2 && g.keys[pos + 1] == x) atomicOr(flags, VG_FLAG_DUP);
}

template <bool kMin>
__global__ void __launch_bounds__(VG_WARPS * 32) k_vg_count(VgGraph g, double thr, long long* __restrict__ cnt,
                                                            int* __restrict__ ncyc, uint8_t* __restrict__ keep,
                                                            double* __restrict__ agg, int* __restrict__ flags) {
  const int lane = threadIdx.x & 31, e = blockIdx.x * VG_WARPS + (threadIdx.x >> 5);
  if (e >= g.n) return;
  const int a = g.edges[2 * e], b = g.edges[2 * e + 1];
  if (lane == 0) vg_check_dup(g, a, b, flags);
  int count = 0;
  bool nan = false;
  double mn = INFINITY;
  vg_for_common(g, a, b, [&](bool hit, int c, int e_ac, int e_bc) {
    count += __popc(__ballot_sync(FULL, hit));
    if (kMin && hit) {
      const double err = vg_triplet_error(g.R, a, b, c, e, e_ac, e_bc);
      nan |= isnan(err);
      mn = fmin(mn, err);
    }
  });
  if (kMin) {
    for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(FULL, mn, o));
    nan = __any_sync(FULL, nan);
  }
  if (lane == 0) {
    if (cnt) cnt[e] = count;
    ncyc[e] = count;
    if (count == 0) {
      agg[e] = NAN, keep[e] = 1;
    } else if (kMin) {
      const double v = nan ? NAN : mn;
      agg[e] = v, keep[e] = v < thr;
    }
  }
}

// the edges of a chunk: a triplet in the window [lo, hi) of the segment space starts there
__device__ __forceinline__ bool vg_in_chunk(const long long* cnt, const long long* off, int e, long long lo, long long hi) {
  return cnt[e] > 0 && off[e] >= lo && off[e] < hi;
}

__global__ void __launch_bounds__(VG_WARPS * 32) k_vg_fill(VgGraph g, const long long* __restrict__ cnt,
                                                           const long long* __restrict__ off, long long lo, long long hi,
                                                           double* __restrict__ seg) {
  const int lane = threadIdx.x & 31, e = blockIdx.x * VG_WARPS + (threadIdx.x >> 5);
  if (e >= g.n || !vg_in_chunk(cnt, off, e, lo, hi)) return;
  const int a = g.edges[2 * e], b = g.edges[2 * e + 1];
  double* s = seg + (off[e] - lo);
  int w = 0;
  vg_for_common(g, a, b, [&](bool hit, int c, int e_ac, int e_bc) {
    const unsigned bal = __ballot_sync(FULL, hit);
    if (hit) s[w + __popc(bal & ((1u << lane) - 1u))] = vg_triplet_error(g.R, a, b, c, e, e_ac, e_bc);
    w += __popc(bal);
  });
}

// the k-th smallest (0-based) of m non-negative doubles by their bit patterns, one warp, `hist` its 256 shared counters
__device__ double vg_radix_select(const double* __restrict__ s, int m, int k, int* hist) {
  const int lane = threadIdx.x & 31;
  u64 prefix = 0, pmask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int d = lane; d < 256; d += 32) hist[d] = 0;
    __syncwarp();
    for (int i = lane; i < m; i += 32) {
      const u64 u = (u64)__double_as_longlong(s[i]);
      if ((u & pmask) == prefix) atomicAdd(&hist[(u >> shift) & 255], 1);
    }
    __syncwarp();
    int loc[8], sum = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) loc[j] = hist[8 * lane + j], sum += loc[j];
    int inc = sum;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(FULL, inc, o);
      if (lane >= o) inc += y;
    }
    const int exc = inc - sum;
    const bool mine = exc <= k && k < inc;
    const int src = __ffs(__ballot_sync(FULL, mine)) - 1;
    int dsel = 0, before = 0;
    if (mine) {
      int c = exc;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (c <= k && k < c + loc[j]) dsel = 8 * lane + j, before = c;  // one digit's interval holds k
        c += loc[j];
      }
    }
    dsel = __shfl_sync(FULL, dsel, src);
    before = __shfl_sync(FULL, before, src);
    prefix |= (u64)dsel << shift;
    pmask |= 255ull << shift;
    k -= before;
    __syncwarp();
  }
  return __longlong_as_double((long long)prefix);
}

// the k-th smallest of m <= 32 values held one per lane (x on lanes >= m is ignored): rank by counting
__device__ __forceinline__ double vg_rank_select(double x, int m, int k) {
  const int lane = threadIdx.x & 31;
  int rank = 0;
  for (int j = 0; j < m; ++j) {
    const double y = __shfl_sync(FULL, x, j);
    rank += (y < x) || (y == x && j < lane);
  }
  const int src = __ffs(__ballot_sync(FULL, lane < m && rank == k)) - 1;
  return __shfl_sync(FULL, x, src);
}

__global__ void __launch_bounds__(VG_WARPS * 32) k_vg_select(int n, const long long* __restrict__ cnt, const long long* __restrict__ off,
                                                             long long lo, long long hi, int last, const double* __restrict__ seg,
                                                             double thr, uint8_t* __restrict__ keep, double* __restrict__ agg,
                                                             int* __restrict__ flags) {
  __shared__ int s_hist[VG_WARPS][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, e = blockIdx.x * VG_WARPS + warp;
  if (e >= n) return;
  if (last && lane == 0 && cnt[e] > 0 && off[e] >= hi) atomicOr(flags, VG_FLAG_OVERFLOW);  // cannot happen: see the plan
  if (!vg_in_chunk(cnt, off, e, lo, hi)) return;
  const int m = (int)cnt[e];
  const double* s = seg + (off[e] - lo);
  bool nan = false;
  for (int i = lane; i < m; i += 32) nan |= isnan(s[i]);
  double v;
  if (__any_sync(FULL, nan)) {
    v = NAN;
  } else if (m <= 32) {
    const double x = lane < m ? s[lane] : 0.0;
    v = vg_rank_select(x, m, m / 2);
    if (m % 2 == 0) v = (vg_rank_select(x, m, m / 2 - 1) + v) / 2.0;  // np.median: the mean of the two middle values
  } else {
    v = vg_radix_select(s, m, m / 2, s_hist[warp]);
    if (m % 2 == 0) v = (vg_radix_select(s, m, m / 2 - 1, s_hist[warp]) + v) / 2.0;
  }
  if (lane == 0) agg[e] = v, keep[e] = v < thr;
}

// test-only: every triplet once, from its edge (i0, i1)
__global__ void __launch_bounds__(VG_WARPS * 32) k_vg_list(VgGraph g, long long cap, int* __restrict__ nodes, double* __restrict__ err,
                                                           unsigned long long* __restrict__ count) {
  const int e = blockIdx.x * VG_WARPS + (threadIdx.x >> 5);
  if (e >= g.n) return;
  const int a = g.edges[2 * e], b = g.edges[2 * e + 1];
  vg_for_common(g, a, b, [&](bool hit, int c, int e_ac, int e_bc) {
    if (hit && c > b) {
      const unsigned long long slot = atomicAdd(count, 1ull);
      if ((long long)slot < cap) {
        nodes[3 * slot] = a, nodes[3 * slot + 1] = b, nodes[3 * slot + 2] = c;
        err[slot] = vg_triplet_error(g.R, a, b, c, e, e_ac, e_bc);
      }
    }
  });
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct ViewGraphState {
  DevBuf in, keys[2], vals[2], scan, tiles, cnt, off, seg, keep, agg, ncyc, flags, list_nodes, list_err;
  HostBuf hin, hout;
};

void vg_destroy(b2_context* ctx) {
  delete ctx->vg;
  ctx->vg = nullptr;
}

static int vg_check(b2_context* ctx, const int32_t* edges, const double* R, int n, int* max_node) {
  if (n < 0) return b2_fail(ctx, B2_ERR_ARG, "view graph: n < 0");
  if (n > 0 && (!edges || !R)) return b2_fail(ctx, B2_ERR_ARG, "view graph: edges / R is NULL");
  if (n > (1 << 29)) return b2_fail(ctx, B2_ERR_ARG, "view graph: more than 2^29 edges");
  int mx = 0;
  for (int e = 0; e < n; ++e) {
    const int a = edges[2 * e], b = edges[2 * e + 1];
    if (a < 0 || b < 0 || a >= b)
      return b2_fail(ctx, B2_ERR_ARG, "view graph edge " + std::to_string(e) + " (" + std::to_string(a) + ", " + std::to_string(b) +
                                          "): indices must satisfy 0 <= i1 < i2");
    mx = b > mx ? b : mx;
  }
  *max_node = mx;
  return B2_OK;
}

// exclusive scan of n int64 in -> out (may alias); the total lands in s->tiles[cdiv(n, 1024)]
static int vg_scan(b2_context* ctx, ViewGraphState* s, const long long* in, long long* out, long long n, cudaStream_t st) {
  const int ntiles = (int)((n + VG_SCAN_THREADS - 1) / VG_SCAN_THREADS);
  B2_CUDA(ctx, s->tiles.ensure(((size_t)ntiles + 1) * sizeof(long long)));
  long long* tiles = s->tiles.as<long long>();
  if (ntiles > 0) {
    B2_LAUNCH(ctx, k_vg_scan_tiles, ntiles, VG_SCAN_THREADS, 0, st, in, out, n, tiles);
  }
  B2_LAUNCH(ctx, k_vg_scan_top, 1, VG_SCAN_THREADS, 0, st, tiles, ntiles);
  if (ntiles > 0) {
    B2_LAUNCH(ctx, k_vg_scan_add, ntiles, VG_SCAN_THREADS, 0, st, out, n, tiles);
  }
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// upload edges and rotations, build the sorted adjacency; *g describes it
static int vg_adjacency(b2_context* ctx, const int32_t* edges, const double* R, int n, int max_node, cudaStream_t st, VgGraph* g) {
  if (!ctx->vg) ctx->vg = new ViewGraphState();
  ViewGraphState* s = ctx->vg;
  int B = 1;
  while ((1ll << B) <= (long long)max_node + 1) ++B;  // node + 1 must fit too: a row ends at key (node + 1) << B
  const int n2 = 2 * n, nblk = cdiv(n2, VG_TILE), passes = (2 * B + 7) / 8;
  const size_t eb = (size_t)n * 2 * sizeof(int), rb = (size_t)n * 9 * sizeof(double);
  B2_CUDA(ctx, s->hin.ensure(eb + rb));
  B2_CUDA(ctx, s->in.ensure(eb + rb));
  memcpy(s->hin.p, edges, eb);
  memcpy((char*)s->hin.p + eb, R, rb);
  B2_CUDA(ctx, cudaMemcpyAsync(s->in.p, s->hin.p, eb + rb, cudaMemcpyHostToDevice, st));
  for (int i = 0; i < 2; ++i) {
    B2_CUDA(ctx, s->keys[i].ensure((size_t)n2 * sizeof(u64)));
    B2_CUDA(ctx, s->vals[i].ensure((size_t)n2 * sizeof(int)));
  }
  B2_CUDA(ctx, s->scan.ensure((size_t)256 * nblk * sizeof(long long)));
  const int* d_edges = s->in.as<int>();
  B2_LAUNCH(ctx, k_vg_halfedges, cdiv(n, 256), 256, 0, st, d_edges, n, B, s->keys[0].as<u64>(), s->vals[0].as<int>());
  B2_CHECK_LAUNCH(ctx);
  for (int p = 0; p < passes; ++p) {
    const int src = p & 1, shift = 8 * p;
    B2_LAUNCH(ctx, k_vg_hist, nblk, VG_SORT_THREADS, 0, st, s->keys[src].as<u64>(), n2, shift, s->scan.as<long long>(), nblk);
    B2_CHECK_LAUNCH(ctx);
    if (int rc = vg_scan(ctx, s, s->scan.as<long long>(), s->scan.as<long long>(), (long long)256 * nblk, st)) return rc;
    B2_LAUNCH(ctx, k_vg_scatter, nblk, VG_SORT_THREADS, 0, st, s->keys[src].as<u64>(), s->vals[src].as<int>(), s->keys[src ^ 1].as<u64>(),
              s->vals[src ^ 1].as<int>(), n2, shift, s->scan.as<long long>(), nblk);
    B2_CHECK_LAUNCH(ctx);
  }
  *g = VgGraph{d_edges, (const double*)((const char*)s->in.p + eb), s->keys[passes & 1].as<u64>(), s->vals[passes & 1].as<int>(), n, n2, B};
  return B2_OK;
}

// segment entries any graph with n edges can have: 3 T, T <= (sqrt(2) / 3) n^1.5
static long long vg_max_entries(int n) { return 3 * (long long)(sqrt(2.0) / 3.0 * pow((double)n, 1.5)) + 3; }

extern "C" int b2_viewgraph_cycle_filter_host(b2_context* ctx, const int32_t* edges, const double* R, int n,
                                              const b2_viewgraph_params* params, uint8_t* keep, double* aggregate, int32_t* num_cycles,
                                              void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (!params) return b2_fail(ctx, B2_ERR_ARG, "view graph: params is NULL");
  if (params->criterion != B2_VG_MEDIAN && params->criterion != B2_VG_MIN)
    return b2_fail(ctx, B2_ERR_ARG, "view graph: criterion must be B2_VG_MEDIAN or B2_VG_MIN");
  if (isnan(params->error_threshold_deg)) return b2_fail(ctx, B2_ERR_ARG, "view graph: error_threshold_deg is NaN");
  int max_node = 0;
  if (int rc = vg_check(ctx, edges, R, n, &max_node)) return rc;
  if (n > 0 && (!keep || !aggregate || !num_cycles)) return b2_fail(ctx, B2_ERR_ARG, "view graph: an output is NULL");
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  VgGraph g;
  if (int rc = vg_adjacency(ctx, edges, R, n, max_node, st, &g)) return rc;
  ViewGraphState* s = ctx->vg;
  B2_CUDA(ctx, s->keep.ensure((size_t)n));
  B2_CUDA(ctx, s->agg.ensure((size_t)n * sizeof(double)));
  B2_CUDA(ctx, s->ncyc.ensure((size_t)n * sizeof(int)));
  B2_CUDA(ctx, s->flags.ensure(sizeof(int)));
  B2_CUDA(ctx, cudaMemsetAsync(s->flags.p, 0, sizeof(int), st));
  const double thr = params->error_threshold_deg;
  uint8_t* d_keep = s->keep.as<uint8_t>();
  double* d_agg = s->agg.as<double>();
  int* d_ncyc = s->ncyc.as<int>();
  int* d_flags = s->flags.as<int>();
  const int grid = cdiv(n, VG_WARPS);
  if (params->criterion == B2_VG_MIN) {
    B2_LAUNCH(ctx, k_vg_count<true>, grid, VG_WARPS * 32, 0, st, g, thr, nullptr, d_ncyc, d_keep, d_agg, d_flags);
    B2_CHECK_LAUNCH(ctx);
  } else {
    B2_CUDA(ctx, s->cnt.ensure((size_t)n * sizeof(long long)));
    B2_CUDA(ctx, s->off.ensure((size_t)n * sizeof(long long)));
    long long* d_cnt = s->cnt.as<long long>();
    long long* d_off = s->off.as<long long>();
    B2_LAUNCH(ctx, k_vg_count<false>, grid, VG_WARPS * 32, 0, st, g, thr, d_cnt, d_ncyc, d_keep, d_agg, d_flags);
    B2_CHECK_LAUNCH(ctx);
    if (int rc = vg_scan(ctx, s, d_cnt, d_off, n, st)) return rc;
    // a window of the segment space per chunk; an edge's segment starts in its window and has at most n - 1 entries
    const long long window = (long long)ctx->vg_workspace_mb * (1ll << 20) / (long long)sizeof(double);
    const long long chunks = (vg_max_entries(n) + window - 1) / window;
    B2_CUDA(ctx, s->seg.ensure((size_t)(window + n) * sizeof(double)));
    for (long long j = 0; j < chunks; ++j) {
      const long long lo = j * window, hi = lo + window;
      B2_LAUNCH(ctx, k_vg_fill, grid, VG_WARPS * 32, 0, st, g, d_cnt, d_off, lo, hi, s->seg.as<double>());
      B2_LAUNCH(ctx, k_vg_select, grid, VG_WARPS * 32, 0, st, n, d_cnt, d_off, lo, hi, (int)(j == chunks - 1), s->seg.as<double>(), thr,
                d_keep, d_agg, d_flags);
      B2_CHECK_LAUNCH(ctx);
    }
  }
  const size_t ob = (size_t)n * (sizeof(double) + sizeof(int) + 1) + sizeof(int);
  B2_CUDA(ctx, s->hout.ensure(ob));
  char* h = (char*)s->hout.p;
  B2_CUDA(ctx, cudaMemcpyAsync(h, d_agg, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h + (size_t)n * 8, d_ncyc, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h + (size_t)n * 12, d_flags, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h + (size_t)n * 12 + 4, d_keep, (size_t)n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  int flags;
  memcpy(&flags, h + (size_t)n * 12, sizeof(int));
  if (flags & VG_FLAG_DUP) return b2_fail(ctx, B2_ERR_ARG, "view graph: an edge (i1, i2) appears more than once");
  if (flags & VG_FLAG_OVERFLOW) return b2_fail(ctx, B2_ERR_STATE, "view graph: more triplets than the chunk plan covers");
  memcpy(aggregate, h, (size_t)n * sizeof(double));
  memcpy(num_cycles, h + (size_t)n * 8, (size_t)n * sizeof(int));
  memcpy(keep, h + (size_t)n * 12 + 4, (size_t)n);
  return B2_OK;
}

extern "C" int b2_debug_viewgraph_triplets_host(b2_context* ctx, const int32_t* edges, const double* R, int n, int64_t capacity,
                                                int32_t* out_nodes, double* out_error, int64_t* out_count, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (capacity < 0 || !out_count || (capacity > 0 && (!out_nodes || !out_error)))
    return b2_fail(ctx, B2_ERR_ARG, "view graph triplets: bad capacity / outputs");
  int max_node = 0;
  if (int rc = vg_check(ctx, edges, R, n, &max_node)) return rc;
  *out_count = 0;
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  VgGraph g;
  if (int rc = vg_adjacency(ctx, edges, R, n, max_node, st, &g)) return rc;
  ViewGraphState* s = ctx->vg;
  const size_t cap = (size_t)capacity;
  B2_CUDA(ctx, s->list_nodes.ensure(cap * 3 * sizeof(int) + 16));
  B2_CUDA(ctx, s->list_err.ensure(cap * sizeof(double) + 16));
  B2_CUDA(ctx, s->flags.ensure(sizeof(unsigned long long)));
  B2_CUDA(ctx, cudaMemsetAsync(s->flags.p, 0, sizeof(unsigned long long), st));
  B2_LAUNCH(ctx, k_vg_list, cdiv(n, VG_WARPS), VG_WARPS * 32, 0, st, g, capacity, s->list_nodes.as<int>(), s->list_err.as<double>(),
            s->flags.as<unsigned long long>());
  B2_CHECK_LAUNCH(ctx);
  unsigned long long count = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&count, s->flags.p, sizeof(count), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  const size_t m = count < cap ? (size_t)count : cap;
  if (m > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(out_nodes, s->list_nodes.p, m * 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(out_error, s->list_err.p, m * sizeof(double), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  *out_count = (int64_t)count;
  return B2_OK;
}
