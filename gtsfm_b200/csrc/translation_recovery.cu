// 1DSfM's translation recovery for sm_90a: gtsam's TranslationRecovery::run(measurements, scale) as
// averaging_1dsfm.py:__run_averaging calls it, i.e. Levenberg-Marquardt with LevenbergMarquardtParams() defaults over one
// Point3 per camera and per landmark, fp64 throughout.  translation_math.cuh holds the factor maths and
// oracle/translation_recovery_ref.py states the same solve in NumPy.  One LM trial is:
//   k_tr_lin      one thread per edge: the whitened, Huber-reweighted residual sqrt(w) r and Jacobian M = sqrt(w) N / sigma
//                 (the Jacobian in b; -M in a); once per linearisation point, not per trial
//   k_tr_lmk      one thread per landmark: its damped 3 x 3 block (edges, priors, lambda), the Cholesky factor L,
//                 z = L^-1 g_l and W_e = L^-1 H_lc for each of its edges
//   k_tr_blocks   one CTA per camera pair (a >= b): the 3 x 3 block of the reduced camera system, summed over the pair's
//                 (edge, edge) list in its fixed order: landmark pairs (-W^T W), a camera's own edges (M^T M) and the
//                 off-diagonal block of a camera-camera edge (-M^T M)
//   k_tr_diag     the priors and the damping on the diagonal; k_tr_rhs the reduced right-hand side
//   dense_chol_solve  the blocked Cholesky of the dense reduced system and its two solves (dense_chol.cu)
//   k_tr_nodes    one thread per node: the camera steps, the landmarks' back-substitution, the candidate
//   k_tr_edges    one thread per edge: its cost at the candidate, its linearised decrease and old linearised cost
//   k_tr_reduce   one CTA: the fixed-order sums, plus the two priors
// The host reads the reduced scalars back once per trial and applies twoview_math.cuh's lm_trial / lm_continue.
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "common.cuh"
#include "dense_chol.cuh"
#include "translation_math.cuh"
#include "../../include/gtsfm_b200.h"

using namespace tvmath;

namespace {
constexpr int TR_THREADS = 128;
constexpr int RED_THREADS = 256;
constexpr int EQ = 9 + 3 + 9;  // per edge: M [3][3], sqrt(w) r [3], W [3][3] (landmark edges)

struct Tr {
  int C, np, L, E;
  double inv_sigma, huber_k;
  trmath::Priors pr;
  const int *ea, *eb;        // [E]
  const double* meas;        // [E][3]
  const int *loff, *ledge;   // landmark l's edges: ledge[loff[l] .. loff[l + 1]), ascending
  const int *coff, *cedge;   // camera a's edges, ascending (a camera-camera edge is in both lists)
  const int2* pairs;         // (x, y) by block, then in the list's fixed order; y < 0: the off-diagonal of edge x
  const int64_t* poff;       // [nblk + 1]
  const int2* blk;           // [nblk] (a, b), a >= b
  double *cur, *cand, *dx;   // [C + L][3]
  double* eq;                // [E][EQ]
  double *Lf, *z;            // [L][9], [L][3]
  double *S, *b, *y, *dc;    // [np][np], [np] x 3
  double *elin, *eold, *ecost;
  double* scal;              // [4]: lin, old, cost, flag
  int* flag;
};

// (M^T M)[r][c] of an edge
__device__ __forceinline__ double mtm(const double* q, int r, int c) { return q[r] * q[c] + q[3 + r] * q[3 + c] + q[6 + r] * q[6 + c]; }
// (M^T sqrt(w) r)[i]
__device__ __forceinline__ double mtr(const double* q, int i) { return q[i] * q[9] + q[3 + i] * q[10] + q[6 + i] * q[11]; }
}  // namespace

__global__ void __launch_bounds__(TR_THREADS) k_tr_lin(Tr t) {
  const int e = blockIdx.x * TR_THREADS + threadIdx.x;
  if (e >= t.E) return;
  double err[3], M[9];
  trmath::edge_error(t.cur + 3 * (int64_t)t.ea[e], t.cur + 3 * (int64_t)t.eb[e], t.meas + 3 * (int64_t)e, t.inv_sigma, err, M);
  const double sw = sqrt(trmath::weight(trmath::norm3(err), t.huber_k));
  double* q = t.eq + (int64_t)e * EQ;
  for (int i = 0; i < 9; ++i) q[i] = sw * M[i];
  for (int i = 0; i < 3; ++i) q[9 + i] = sw * err[i];
}

__global__ void __launch_bounds__(TR_THREADS) k_tr_lmk(Tr t, double lam) {
  const int l = blockIdx.x * TR_THREADS + threadIdx.x;
  if (l >= t.L) return;
  const int n = t.C + l;
  double H[9] = {0}, gl[3] = {0};
  for (int k = t.loff[l]; k < t.loff[l + 1]; ++k) {
    const int e = t.ledge[k];
    const double* q = t.eq + (int64_t)e * EQ;
    const double sgn = t.eb[e] == n ? 1.0 : -1.0;
    for (int i = 0; i < 3; ++i) {
      for (int c = 0; c < 3; ++c) H[i * 3 + c] += mtm(q, i, c);
      gl[i] += sgn * mtr(q, i);
    }
  }
  double h = 0.0;
  trmath::prior_hg(t.pr, n, t.cur + 3 * (int64_t)n, h, gl);
  for (int i = 0; i < 3; ++i) H[i * 4] += h, H[i * 4] += lam;
  if (!chol(H, 3, 3)) *t.flag = 1;
  chol_fwd(H, 3, 3, gl);
  for (int i = 0; i < 9; ++i) t.Lf[9 * (int64_t)l + i] = H[i];
  for (int i = 0; i < 3; ++i) t.z[3 * (int64_t)l + i] = gl[i];
  for (int k = t.loff[l]; k < t.loff[l + 1]; ++k) {
    double* q = t.eq + (int64_t)t.ledge[k] * EQ;
    for (int c = 0; c < 3; ++c) {  // column c of W = L^-1 H_lc, H_lc = -M^T M
      double w[3];
      for (int i = 0; i < 3; ++i) w[i] = -mtm(q, i, c);
      chol_fwd(H, 3, 3, w);
      for (int i = 0; i < 3; ++i) q[12 + 3 * i + c] = w[i];
    }
  }
}

// one CTA per block (a, b), a >= b, threads 0..8 its entries: the sum over the block's list in order
__global__ void __launch_bounds__(32) k_tr_blocks(Tr t) {
  if (*t.flag) return;
  const int e = threadIdx.x;
  if (e >= 9) return;
  const int r = e / 3, c = e % 3;
  const int2 ab = t.blk[blockIdx.x];
  double acc = 0.0;
  for (int64_t p = t.poff[blockIdx.x]; p < t.poff[blockIdx.x + 1]; ++p) {
    const int2 xy = t.pairs[p];
    const double* qa = t.eq + (int64_t)xy.x * EQ;
    double v;
    if (xy.y < 0) {
      v = -mtm(qa, r, c);
    } else {
      v = xy.x == xy.y ? mtm(qa, r, c) : 0.0;
      if (t.ea[xy.x] >= t.C || t.eb[xy.x] >= t.C) {
        const double* qb = t.eq + (int64_t)xy.y * EQ;
        v -= qa[12 + r] * qb[12 + c] + qa[15 + r] * qb[15 + c] + qa[18 + r] * qb[18 + c];
      }
    }
    acc += v;
  }
  t.S[(int64_t)(3 * ab.x + r) * t.np + 3 * ab.y + c] = acc;
}

// the diagonal: the priors on cameras and the damping lam; identity on the padding
__global__ void k_tr_diag(Tr t, double lam) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (*t.flag || u >= t.np) return;
  double* d = t.S + (int64_t)u * t.np + u;
  if (u >= 3 * t.C) {
    *d = 1.0;
    return;
  }
  const int a = u / 3;
  double h = 0.0, g[3] = {0, 0, 0};
  trmath::prior_hg(t.pr, a, t.cur + 3 * a, h, g);
  *d += h;
  *d += lam;
}

// the reduced right-hand side: -(g_c - W^T z) over each camera's edges in order, with the priors' gradients
__global__ void k_tr_rhs(Tr t) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (*t.flag || u >= t.np) return;
  if (u >= 3 * t.C) {
    t.b[u] = 0.0;
    return;
  }
  const int a = u / 3, i = u % 3;
  double acc = 0.0;
  for (int k = t.coff[a]; k < t.coff[a + 1]; ++k) {
    const int e = t.cedge[k];
    const double* q = t.eq + (int64_t)e * EQ;
    const int other = t.eb[e] == a ? t.ea[e] : t.eb[e];
    acc += (t.eb[e] == a ? 1.0 : -1.0) * mtr(q, i);
    if (other >= t.C) {
      const double* zl = t.z + 3 * (int64_t)(other - t.C);
      acc -= q[12 + i] * zl[0] + q[15 + i] * zl[1] + q[18 + i] * zl[2];
    }
  }
  double h = 0.0, g[3] = {0, 0, 0};
  trmath::prior_hg(t.pr, a, t.cur + 3 * a, h, g);
  acc += i == 0 ? g[0] : i == 1 ? g[1] : g[2];  // static indices: g stays in registers
  t.b[u] = -acc;
}

// one thread per node: its step (a camera's from the solve, a landmark's dl = -L^-T (z + sum_e W_e dc_cam(e))) and the
// candidate
__global__ void __launch_bounds__(TR_THREADS) k_tr_nodes(Tr t) {
  const int n = blockIdx.x * TR_THREADS + threadIdx.x;
  if (*t.flag || n >= t.C + t.L) return;
  double d[3];
  if (n < t.C) {
    for (int i = 0; i < 3; ++i) d[i] = t.dc[3 * n + i];
  } else {
    const int l = n - t.C;
    double yv[3] = {t.z[3 * (int64_t)l], t.z[3 * (int64_t)l + 1], t.z[3 * (int64_t)l + 2]};
    for (int k = t.loff[l]; k < t.loff[l + 1]; ++k) {
      const int e = t.ledge[k];
      const double* q = t.eq + (int64_t)e * EQ;
      const double* dca = t.dc + 3 * (t.ea[e] == n ? t.eb[e] : t.ea[e]);
      for (int i = 0; i < 3; ++i) yv[i] += q[12 + 3 * i] * dca[0] + q[13 + 3 * i] * dca[1] + q[14 + 3 * i] * dca[2];
    }
    const double* L = t.Lf + 9 * (int64_t)l;
    for (int i = 2; i >= 0; --i) {  // L^T d' = y, d = -d'
      double s = yv[i];
      for (int m = i + 1; m < 3; ++m) s -= L[m * 3 + i] * yv[m];
      yv[i] = s / L[i * 3 + i];
    }
    for (int i = 0; i < 3; ++i) d[i] = -yv[i];
  }
  for (int i = 0; i < 3; ++i) {
    t.dx[3 * (int64_t)n + i] = d[i];
    t.cand[3 * (int64_t)n + i] = t.cur[3 * (int64_t)n + i] + d[i];
  }
}

// one thread per edge: its cost at the candidate (cost_only: at the current state), and for a trial its share of the
// linearised decrease -(r . Jd + |Jd|^2 / 2), Jd = M (d_b - d_a), and of the old linearised cost
__global__ void __launch_bounds__(TR_THREADS) k_tr_edges(Tr t, int cost_only) {
  const int e = blockIdx.x * TR_THREADS + threadIdx.x;
  if (e >= t.E || (!cost_only && *t.flag)) return;
  const double* X = cost_only ? t.cur : t.cand;
  const int a = t.ea[e], b = t.eb[e];
  double err[3];
  trmath::edge_error(X + 3 * (int64_t)a, X + 3 * (int64_t)b, t.meas + 3 * (int64_t)e, t.inv_sigma, err, nullptr);
  t.ecost[e] = trmath::loss(trmath::norm3(err), t.huber_k);
  if (cost_only) return;
  const double* q = t.eq + (int64_t)e * EQ;
  double dd[3];
  for (int i = 0; i < 3; ++i) dd[i] = t.dx[3 * (int64_t)b + i] - t.dx[3 * (int64_t)a + i];
  double lin = 0.0, old = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double jd = q[3 * i] * dd[0] + q[3 * i + 1] * dd[1] + q[3 * i + 2] * dd[2], r = q[9 + i];
    lin -= r * jd + 0.5 * jd * jd, old += 0.5 * r * r;
  }
  t.elin[e] = lin, t.eold[e] = old;
}

__device__ double tr_block_sum(double v, double* red) {
  const int tid = threadIdx.x;
  red[tid] = v;
  __syncthreads();
  for (int s = RED_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// fixed-order sums over the edges, then the two priors: scal = {lin, old, cost at the candidate (or at the current state:
// cost_only), failed}
__global__ void __launch_bounds__(RED_THREADS) k_tr_reduce(Tr t, int cost_only) {
  __shared__ double red[RED_THREADS];
  const int tid = threadIdx.x;
  double l = 0.0, o = 0.0, c = 0.0;
  const bool go = cost_only || !*t.flag;
  if (go)
    for (int e = tid; e < t.E; e += RED_THREADS) {
      c += t.ecost[e];
      if (!cost_only) l += t.elin[e], o += t.eold[e];
    }
  l = tr_block_sum(l, red);
  o = tr_block_sum(o, red);
  c = tr_block_sum(c, red);
  if (tid == 0) {
    if (go) {
      const double* X = cost_only ? t.cur : t.cand;
      for (int k = 0; k < 2; ++k) {
        const int64_t n = k == 0 ? t.pr.n0 : t.pr.n1;
        c += trmath::prior_cost(t.pr, k, X + 3 * n);
        if (!cost_only) trmath::prior_lin(t.pr, k, t.cur + 3 * n, t.dx + 3 * n, l, o);
      }
    }
    t.scal[0] = l, t.scal[1] = o, t.scal[2] = c, t.scal[3] = cost_only ? 0.0 : (double)*t.flag;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct TranslationRecoveryState {
  DevBuf ws;
};

void tr_destroy(b2_context* ctx) {
  delete ctx->tr;
  ctx->tr = nullptr;
}

namespace {
struct Layout {
  size_t off[24];
  size_t total;
};

int padded(int C) { return (3 * C + CHOL_NB - 1) / CHOL_NB * CHOL_NB; }

// byte offsets of every device array of a call (256-byte aligned)
Layout layout(int C, int L, int E, int64_t P, int64_t nblk) {
  const int np = padded(C);
  const int64_t V = (int64_t)C + L;
  const size_t sizes[] = {
      (size_t)np * np * 8,                             // 0 S
      (size_t)np * 8, (size_t)np * 8, (size_t)np * 8,  // 1-3 b, y, dc
      (size_t)E * EQ * 8,                              // 4 eq
      (size_t)L * 72, (size_t)L * 24,                  // 5-6 Lf, z
      (size_t)V * 24 * 3,                              // 7 cur, cand, dx
      (size_t)E * 24,                                  // 8 elin, eold, ecost
      (size_t)E * 4, (size_t)E * 4, (size_t)E * 24,    // 9-11 ea, eb, meas
      (size_t)(L + 1) * 4, (size_t)E * 4,              // 12-13 loff, ledge
      (size_t)(C + 1) * 4, (size_t)E * 8,              // 14-15 coff, cedge
      (size_t)P * 8, (size_t)(nblk + 1) * 8, (size_t)nblk * 8,  // 16-18 pairs, poff, blk
      64,                                              // 19 scal + flag
  };
  Layout l{};
  size_t o = 0;
  for (size_t i = 0; i < sizeof(sizes) / sizeof(sizes[0]); ++i) l.off[i] = o, o += (sizes[i] + 255) / 256 * 256;
  l.total = o;
  return l;
}

// the landmark endpoint of edge e, or -1 for a camera-camera edge
int lmk_of(int C, int a, int b) { return a >= C ? a - C : b >= C ? b - C : -1; }
int cam_of(int C, int a, int b) { return a >= C ? b : a; }

// the (edge, edge) list's length: every landmark's pairs (x, y) with cam(x) >= cam(y), three per camera-camera edge
int64_t pair_count(int C, int L, int E, const int32_t* ea, const int32_t* eb, std::vector<int>& loff, std::vector<int>& ledge) {
  loff.assign(L + 1, 0);
  for (int e = 0; e < E; ++e) {
    const int l = lmk_of(C, ea[e], eb[e]);
    if (l >= 0) ++loff[l + 1];
  }
  for (int l = 0; l < L; ++l) loff[l + 1] += loff[l];
  ledge.assign(loff[L], 0);
  std::vector<int> fill(loff.begin(), loff.end() - 1);
  int64_t P = 0;
  for (int e = 0; e < E; ++e) {
    const int l = lmk_of(C, ea[e], eb[e]);
    if (l >= 0) ledge[fill[l]++] = e;
    else P += 3;
  }
  for (int l = 0; l < L; ++l)
    for (int x = loff[l]; x < loff[l + 1]; ++x)
      for (int y = loff[l]; y < loff[l + 1]; ++y)
        if (cam_of(C, ea[ledge[x]], eb[ledge[x]]) >= cam_of(C, ea[ledge[y]], eb[ledge[y]])) ++P;
  return P;
}

bool edges_in_range(int C, int L, int E, const int32_t* ea, const int32_t* eb) {
  const int64_t V = (int64_t)C + L;
  for (int e = 0; e < E; ++e)
    if (ea[e] < 0 || ea[e] >= V || eb[e] < 0 || eb[e] >= V) return false;
  return true;
}
}  // namespace

extern "C" size_t b2_translation_recovery_workspace_bytes(int C, int L, int E, const int32_t* edge_a, const int32_t* edge_b) {
  if (C < 1 || L < 0 || E < 1 || C > 1000000 || L > (1 << 30) || !edge_a || !edge_b || !edges_in_range(C, L, E, edge_a, edge_b))
    return 0;
  std::vector<int> loff, ledge;
  const int64_t P = pair_count(C, L, E, edge_a, edge_b, loff, ledge);
  return layout(C, L, E, P, std::min<int64_t>(P, (int64_t)C * (C + 1) / 2)).total;
}

extern "C" int b2_translation_recovery_host(b2_context* ctx, int C, int L, int E, const int32_t* edge_a, const int32_t* edge_b,
                                            const double* meas, const double* init, const b2_tr_params* prm, double* out,
                                            b2_ba_result* result, double* trace, int32_t* trial_out, int trial_cap, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (!prm) return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: params is NULL");
  if (C < 1 || L < 0 || E < 1 || C > 1000000 || L > (1 << 30))
    return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: needs 1..10^6 cameras, 0..2^30 landmarks and at least one edge");
  if (!edge_a || !edge_b || !meas || !init || !out || !result)
    return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: a required array is NULL");
  if (trial_cap < 0 || (trial_cap > 0 && !trial_out))
    return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: bad trial_out / trial_cap");
  if (!(prm->sigma > 0.0) || !std::isfinite(prm->sigma) || !(prm->huber_k >= 0.0) || !std::isfinite(prm->huber_k) ||
      !(prm->prior_sigma > 0.0) || !std::isfinite(prm->prior_sigma) || !std::isfinite(prm->scale) || prm->max_iters < 0 ||
      prm->max_iters > 100000)
    return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: bad params");
  if (!edges_in_range(C, L, E, edge_a, edge_b)) return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: node index out of range");
  const int64_t V = (int64_t)C + L;
  std::vector<char> seen(V, 0);
  for (int e = 0; e < E; ++e) {
    const int a = edge_a[e], b = edge_b[e];
    if (a == b) return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: edge " + std::to_string(e) + " joins a node to itself");
    if (a >= C && b >= C) return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: edge " + std::to_string(e) + " joins two landmarks");
    const double* m = meas + 3 * (int64_t)e;
    if (!std::isfinite(m[0]) || !std::isfinite(m[1]) || !std::isfinite(m[2]) || (m[0] == 0.0 && m[1] == 0.0 && m[2] == 0.0))
      return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: edge " + std::to_string(e) + " has a zero or non-finite measurement");
    seen[a] = seen[b] = 1;
  }
  for (int64_t n = 0; n < V; ++n) {
    if (!seen[n]) return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: node " + std::to_string(n) + " has no edge");
    if (!std::isfinite(init[3 * n]) || !std::isfinite(init[3 * n + 1]) || !std::isfinite(init[3 * n + 2]))
      return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: non-finite initial value");
  }
  std::vector<int> loff, ledge;
  const int64_t P = pair_count(C, L, E, edge_a, edge_b, loff, ledge);
  const int64_t nb_all = (int64_t)C * (C + 1) / 2;
  if (layout(C, L, E, P, std::min(P, nb_all)).total > ((size_t)ctx->ba_workspace_mb << 20))
    return b2_fail(ctx, B2_ERR_ARG, "translation_recovery: the problem needs more than ba_workspace_mb of device workspace");

  // the reduced system's structure, fixed for the call: a counting sort of the (edge, edge) list by block (a, b), a >= b;
  // within a block, camera-camera edges in edge order, then landmarks in order, each landmark's pairs (x, y) row-major
  auto bkey = [](int a, int b) { return (int64_t)a * (a + 1) / 2 + b; };
  std::vector<int64_t> slot(nb_all, 0);
  auto each_pair = [&](auto&& f) {
    for (int e = 0; e < E; ++e) {
      const int a = edge_a[e], b = edge_b[e];
      if (a >= C || b >= C) continue;
      f(bkey(a, a), e, e);
      f(bkey(b, b), e, e);
      f(bkey(std::max(a, b), std::min(a, b)), e, ~e);
    }
    for (int l = 0; l < L; ++l)
      for (int x = loff[l]; x < loff[l + 1]; ++x)
        for (int y = loff[l]; y < loff[l + 1]; ++y) {
          const int ex = ledge[x], ey = ledge[y];
          const int cx = cam_of(C, edge_a[ex], edge_b[ex]), cy = cam_of(C, edge_a[ey], edge_b[ey]);
          if (cx >= cy) f(bkey(cx, cy), ex, ey);
        }
  };
  each_pair([&](int64_t k, int, int) { ++slot[k]; });
  std::vector<int64_t> poff{0};
  std::vector<int2> blk;
  for (int a = 0; a < C; ++a)
    for (int b = 0; b <= a; ++b) {
      const int64_t k = bkey(a, b), n = slot[k];
      if (!n) continue;
      slot[k] = poff.back();
      blk.push_back(make_int2(a, b));
      poff.push_back(poff.back() + n);
    }
  const int64_t nblk = (int64_t)blk.size();
  std::vector<int2> pairs(P);
  each_pair([&](int64_t k, int x, int y) { pairs[slot[k]++] = make_int2(x, y); });
  std::vector<int> coff(C + 1, 0), cedge;
  for (int e = 0; e < E; ++e)
    for (int n : {edge_a[e], edge_b[e]})
      if (n < C) ++coff[n + 1];
  for (int a = 0; a < C; ++a) coff[a + 1] += coff[a];
  cedge.resize(coff[C]);
  {
    std::vector<int> fill(coff.begin(), coff.end() - 1);
    for (int e = 0; e < E; ++e)
      for (int n : {edge_a[e], edge_b[e]})
        if (n < C) cedge[fill[n]++] = e;
  }

  const Layout l = layout(C, L, E, P, nblk);
  const int np = padded(C);
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  if (!ctx->tr) ctx->tr = new TranslationRecoveryState();
  TranslationRecoveryState* s = ctx->tr;
  B2_CUDA(ctx, s->ws.ensure(l.total));
  char* base = s->ws.as<char>();
  auto at = [&](int i) { return base + l.off[i]; };
  Tr t{};
  t.C = C, t.np = np, t.L = L, t.E = E;
  t.inv_sigma = 1.0 / prm->sigma, t.huber_k = prm->huber_k;
  t.pr.n0 = edge_a[0], t.pr.n1 = edge_b[0];
  t.pr.inv_p = 1.0 / prm->prior_sigma, t.pr.inv_s = t.inv_sigma, t.pr.huber_k = prm->huber_k;
  for (int i = 0; i < 3; ++i) t.pr.t1[i] = prm->scale * meas[i];
  t.S = (double*)at(0), t.b = (double*)at(1), t.y = (double*)at(2), t.dc = (double*)at(3);
  t.eq = (double*)at(4), t.Lf = (double*)at(5), t.z = (double*)at(6);
  t.cur = (double*)at(7), t.cand = t.cur + 3 * V, t.dx = t.cur + 6 * V;
  t.elin = (double*)at(8), t.eold = t.elin + E, t.ecost = t.elin + 2 * (int64_t)E;
  t.ea = (const int*)at(9), t.eb = (const int*)at(10), t.meas = (const double*)at(11);
  t.loff = (const int*)at(12), t.ledge = (const int*)at(13), t.coff = (const int*)at(14), t.cedge = (const int*)at(15);
  t.pairs = (const int2*)at(16), t.poff = (const int64_t*)at(17), t.blk = (const int2*)at(18);
  t.scal = (double*)at(19), t.flag = (int*)(t.scal + 4);
  B2_CUDA(ctx, cudaMemcpyAsync(t.cur, init, (size_t)V * 24, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)t.ea, edge_a, (size_t)E * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)t.eb, edge_b, (size_t)E * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)t.meas, meas, (size_t)E * 24, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)t.loff, loff.data(), (size_t)(L + 1) * 4, cudaMemcpyHostToDevice, st));
  if (!ledge.empty()) B2_CUDA(ctx, cudaMemcpyAsync((void*)t.ledge, ledge.data(), ledge.size() * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)t.coff, coff.data(), (size_t)(C + 1) * 4, cudaMemcpyHostToDevice, st));
  if (!cedge.empty()) B2_CUDA(ctx, cudaMemcpyAsync((void*)t.cedge, cedge.data(), cedge.size() * 4, cudaMemcpyHostToDevice, st));
  if (P) B2_CUDA(ctx, cudaMemcpyAsync((void*)t.pairs, pairs.data(), (size_t)P * 8, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((void*)t.poff, poff.data(), (size_t)(nblk + 1) * 8, cudaMemcpyHostToDevice, st));
  if (nblk) B2_CUDA(ctx, cudaMemcpyAsync((void*)t.blk, blk.data(), (size_t)nblk * 8, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(t.scal, 0, 64, st));
  ctx->h2d_bytes += (uint64_t)(V * 24 + (int64_t)E * 32 + (L + 1) * 4 + ledge.size() * 4 + (C + 1) * 4 + cedge.size() * 4 + P * 8 +
                               (nblk + 1) * 8 + nblk * 8);

  const unsigned ge = (unsigned)cdiv(E, TR_THREADS), gl = (unsigned)std::max(1, cdiv(L, TR_THREADS));
  const unsigned gv = (unsigned)((V + TR_THREADS - 1) / TR_THREADS);
  double hs[4];
  auto read_scal = [&]() -> int {
    B2_CUDA(ctx, cudaMemcpyAsync(hs, t.scal, 32, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    return B2_OK;
  };

  // the initial error
  B2_LAUNCH(ctx, k_tr_edges, ge, TR_THREADS, 0, st, t, 1);
  B2_LAUNCH(ctx, k_tr_reduce, 1, RED_THREADS, 0, st, t, 1);
  B2_CHECK_LAUNCH(ctx);
  if (int rc = read_scal()) return rc;
  double nw = hs[2], lam = LM_LAMBDA0;
  int its = 0, ntrace = 0, trials = 0;
  if (trace) trace[ntrace] = nw;
  ++ntrace;
  if (nw > 0.0) {
    bool linearise = true;
    for (;;) {
      const double cur = nw;
      if (linearise) {
        B2_LAUNCH(ctx, k_tr_lin, ge, TR_THREADS, 0, st, t);
        B2_CHECK_LAUNCH(ctx);
        linearise = false;
      }
      for (;;) {  // tryLambda
        B2_CUDA(ctx, cudaMemsetAsync(t.flag, 0, 4, st));
        B2_CUDA(ctx, cudaMemsetAsync(t.S, 0, (size_t)np * np * 8, st));
        if (L) B2_LAUNCH(ctx, k_tr_lmk, gl, TR_THREADS, 0, st, t, lam);
        if (nblk) B2_LAUNCH(ctx, k_tr_blocks, (unsigned)nblk, 32, 0, st, t);
        B2_LAUNCH(ctx, k_tr_diag, (unsigned)cdiv(np, 256), 256, 0, st, t, lam);
        B2_LAUNCH(ctx, k_tr_rhs, (unsigned)cdiv(np, TR_THREADS), TR_THREADS, 0, st, t);
        B2_CHECK_LAUNCH(ctx);
        if (int rc = dense_chol_solve(ctx, t.S, np, t.b, t.y, t.dc, t.flag, st)) return rc;
        B2_LAUNCH(ctx, k_tr_nodes, gv, TR_THREADS, 0, st, t);
        B2_LAUNCH(ctx, k_tr_edges, ge, TR_THREADS, 0, st, t, 0);
        B2_LAUNCH(ctx, k_tr_reduce, 1, RED_THREADS, 0, st, t, 0);
        B2_CHECK_LAUNCH(ctx);
        if (int rc = read_scal()) return rc;
        bool success = false, stop = false;
        const bool failed = hs[3] != 0.0;
        if (!failed) lm_trial(hs[0], hs[1], cur, hs[2], success, stop);
        if (trials < trial_cap) trial_out[trials] = failed ? -1 : success ? 1 : stop ? 2 : 0;
        ++trials;
        if (success) {
          std::swap(t.cur, t.cand);
          lam /= LM_FACTOR, ++its, nw = hs[2];
          linearise = true;
          break;
        }
        if (stop) break;
        lam *= LM_FACTOR;
        if (lam >= LM_LAMBDA_MAX) break;
      }
      if (trace) trace[ntrace] = nw;
      ++ntrace;
      if (!lm_continue(its, prm->max_iters, cur, nw, LM_ABS_TOL)) break;
    }
  }
  B2_CUDA(ctx, cudaMemcpyAsync(out, t.cur, (size_t)V * 24, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memset(result, 0, sizeof(*result));
  result->iterations = its, result->trace_len = ntrace, result->trials = trials, result->final_error = nw;
  return B2_OK;
}
