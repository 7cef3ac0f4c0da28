// Shared host-side dispatch for the matcher networks: one "linear" / attention call site expressed for both execution
// paths (wgmma split-fp16 planes, or the exact-fp32 SIMT kernels under b2_set_option("force_simt", 1)), over a BATCH
// of problems (the images of up to 8 pairs) per launch.
#pragma once
#include "attn_ps.cuh"
#include "common.cuh"
#include "gemm.cuh"
#include "gemm_ws.cuh"

struct TcWeights {  // a model's weight blob in fp32 and as split-fp16 planes (same element offsets in all three)
  const float* f;
  const __half* h;
  const __half* l;
  int* err;     // device flag raised by a timed-out mbarrier wait
  bool use_tc;
  DevBuf* attn_part = nullptr;  // scratch for key-split attention partials (O) ...
  DevBuf* attn_ml = nullptr;    // ... (m, l) ...
  DevBuf* attn_cnt = nullptr;   // ... and the arrival counters of the in-kernel merge
  int sm_count = 132;
};

struct Pl {  // split-fp16 planes of an activation
  __half* hi;
  __half* lo;
};
static inline Pl planes_of(const DevBuf& b, size_t elems) { return {b.as<__half>(), b.as<__half>() + elems}; }

// The packers (weights.fold_message_projection) fold each attention output projection into the feed-forward linear that
// reads the message and leave the identity in its place; a blob whose projection is anything else was not folded, and
// running it without that projection would compute another network.
static inline bool folded_projection(const float* w /*[d][d]*/, const float* b /*[d]*/, int d) {
  for (int r = 0; r < d; ++r) {
    if (b[r] != 0.f) return false;
    for (int c = 0; c < d; ++c)
      if (w[(size_t)r * d + c] != (r == c ? 1.f : 0.f)) return false;
  }
  return true;
}

// One linear / GEMM call site of ONE problem, expressed for both execution paths: fp32 views feed the exact-fp32 SIMT
// kernel, split-fp16 plane views feed the wgmma kernel.
struct LinArgs {
  const float* a1f = nullptr;
  Pl a1p{nullptr, nullptr};
  int lda1 = 0, K1 = 0;
  const float* a2f = nullptr;
  Pl a2p{nullptr, nullptr};
  int lda2 = 0, K2 = 0;
  const float* w = nullptr;   // weight inside the blob (B operand), or
  const float* bf = nullptr;  // an fp32 activation B operand with
  Pl bp{nullptr, nullptr};    // its planes
  int ldb = 0;
  const float* bias = nullptr;
  float scale = 1.f;
  const float* resid = nullptr;
  int ldr = 0;
  float* cf = nullptr;  // fp32 output (always written on the SIMT path; on the wgmma path only if tc_want_f32)
  int ldc = 0;
  Pl cp{nullptr, nullptr};  // plane output (wgmma path)
  int ldch = 0;
  int head_major = 0;
  bool tc_want_f32 = false;
  int relu = 0;  // max(., 0) after bias / scale, before the residual
  int gelu = 0;  // exact GELU after bias / scale, before the residual (wgmma path only)
  int lo_unscaled = 0;  // plane output with an unscaled lo plane (attention operands)
  int M = 0, N = 0;
  // Column segments (seg_n > 0, N = seg_n x segments, head_major): columns s seg_n .. (s + 1) seg_n - 1 go to seg_f[s]
  // (SIMT path) or seg_p[s] (wgmma path) instead of cf / cp.  rot_mask bit s applies rotary (cos / sin [M][32]) to
  // segment s; only the wgmma path has it.
  int seg_n = 0;
  float* seg_f[GW_SEGS] = {};
  Pl seg_p[GW_SEGS] = {};
  int rot_mask = 0;
  const float *cs = nullptr, *sn = nullptr;
};

// `a[0 .. np)`: the same linear applied to np problems.  With a weight operand (a[0].w) every problem shares weights, K,
// N and epilogue, and the wgmma path runs them as ONE persistent launch; with activation B operands (a[i].bf / bp: the
// assignment similarity of each pair) N, ldc and B are per problem, K and the epilogue flags are a[0]'s.
// `site` labels the launch for the profiler: it matches "k_gemm_ws/<site>" (and so the prefix "k_gemm_ws").
static int run_linear(b2_context* ctx, cudaStream_t st, const TcWeights& tw, const LinArgs* a, int np, const char* site = nullptr) {
  if (np <= 0) return B2_OK;
  if (np > GW_MAXP) return b2_fail(ctx, B2_ERR_ARG, "run_linear: too many problems in one launch");
  const LinArgs& a0 = a[0];
  const int nseg = a0.seg_n > 0 ? a0.N / a0.seg_n : 1;
  if (a0.seg_n > 0 && (a0.seg_n % GW_N || a0.N != nseg * a0.seg_n || nseg > GW_SEGS || !a0.head_major || a0.resid || a0.tc_want_f32 ||
                       (a0.rot_mask && (!a0.cs || !a0.sn))))
    return b2_fail(ctx, B2_ERR_ARG, "run_linear: column segments need N = seg_n x (<= 3), seg_n % 128 == 0, head-major planes, "
                                    "no residual or fp32 output, and a rotary table when rotary is on");
  if (!tw.use_tc) {
    if (a0.rot_mask) return b2_fail(ctx, B2_ERR_ARG, "run_linear: the rotary epilogue exists on the wgmma path only");
    for (int i = 0; i < np; ++i) {
      const LinArgs& x = a[i];
      if (x.M <= 0 || x.N <= 0) continue;
      if (x.gelu) return b2_fail(ctx, B2_ERR_ARG, "run_linear: the GELU epilogue exists on the wgmma path only");
      // k_gemm_nt loads float4 operands in K steps of GB_K: a ragged K would read past the end of a row
      if (x.K1 % GB_K || x.K2 % GB_K || x.lda1 % 4 || x.lda2 % 4 || x.ldb % 4)
        return b2_fail(ctx, B2_ERR_ARG, "run_linear: the SIMT GEMM needs K1, K2 multiples of 16 and lda1, lda2, ldb multiples of 4");
    }
    for (int i = 0; i < np; ++i) {
      const LinArgs& x = a[i];
      if (x.M <= 0 || x.N <= 0) continue;
      for (int s = 0; s < nseg; ++s) {  // a segmented linear runs one launch per segment here
        const int c0 = s * x.seg_n;
        GemmArgs g{};
        g.A1 = x.a1f, g.lda1 = x.lda1, g.K1 = x.K1, g.A2 = x.a2f, g.lda2 = x.lda2, g.K2 = x.K2;
        g.B = (x.w ? x.w : x.bf) + (size_t)c0 * x.ldb, g.ldb = x.ldb, g.C = x.seg_n ? x.seg_f[s] : x.cf, g.ldc = x.ldc, g.M = x.M;
        g.N = x.seg_n ? x.seg_n : x.N;
        g.bias = x.bias ? x.bias + c0 : nullptr, g.resid = x.resid, g.ldr = x.ldr, g.scale = x.scale, g.head_major = x.head_major;
        g.relu = x.relu;
        int rc = launch_gemm(ctx, st, g);
        if (rc) return rc;
      }
    }
    return B2_OK;
  }
  // k_gemm_ws walks (K1 + K2) / GW_K whole chunks and switches to A2 at a chunk boundary: a ragged K would be dropped
  if (a0.K1 % GW_K || a0.K2 % GW_K) return b2_fail(ctx, B2_ERR_ARG, "run_linear: the wgmma GEMM needs K1 and K2 multiples of 64");
  if (!tma_encoder()) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled is not available (driver too old?)");
  const bool per_b = a0.w == nullptr;
  static thread_local GemmWsMaps maps;  // 12 KB: keep it off the stack of deep call chains
  GemmWsArgs q{};
  double work = 0.0;
  bool ok = true;
  int nz = 0, tiles = 0;
  for (int i = 0; i < np; ++i) {
    const LinArgs& x = a[i];
    if (x.M <= 0 || x.N <= 0) continue;
    ok = ok && tma_map_2d(&maps.a1h[nz], x.a1p.hi, x.M, x.K1, x.lda1, GW_M) && tma_map_2d(&maps.a1l[nz], x.a1p.lo, x.M, x.K1, x.lda1, GW_M);
    if (x.K2 > 0)
      ok = ok && tma_map_2d(&maps.a2h[nz], x.a2p.hi, x.M, x.K2, x.lda2, GW_M) && tma_map_2d(&maps.a2l[nz], x.a2p.lo, x.M, x.K2, x.lda2, GW_M);
    if (per_b || nz == 0) {
      const __half *bh, *bl;
      if (x.w) {
        const size_t off = (size_t)(x.w - tw.f);
        bh = tw.h + off, bl = tw.l + off;
      } else {
        bh = x.bp.hi, bl = x.bp.lo;
      }
      ok = ok && tma_map_2d(&maps.bh[nz], bh, x.N, x.K1 + x.K2, x.ldb, GW_N) && tma_map_2d(&maps.bl[nz], bl, x.N, x.K1 + x.K2, x.ldb, GW_N);
    }
    GemmProblem& pr = q.p[nz];
    pr.resid = x.resid, pr.C = x.tc_want_f32 ? x.cf : nullptr, pr.M = x.M, pr.N = x.N, pr.ldc = x.ldc;
    for (int s = 0; s < GW_SEGS; ++s) {
      const Pl p = x.seg_n ? (s < nseg ? x.seg_p[s] : Pl{nullptr, nullptr}) : (s == 0 ? x.cp : Pl{nullptr, nullptr});
      pr.Ch[s] = p.hi, pr.Cl[s] = p.lo;
    }
    pr.cs = x.cs, pr.sn = x.sn;
    {  // 16-byte accesses in the epilogue need aligned bases and leading dimensions
      auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
      auto al8 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 7) == 0; };
      const bool hm = x.head_major != 0;
      bool v = al16(pr.resid) && (x.ldr % 4 == 0 || !pr.resid) && al16(pr.C) && (hm || x.ldc % 4 == 0 || !pr.C);
      v = v && (hm || x.ldch % 4 == 0 || !pr.Ch[0]);
      for (int s = 0; s < GW_SEGS; ++s) v = v && al8(pr.Ch[s]) && al8(pr.Cl[s]);
      v = v && al8(pr.cs) && al8(pr.sn);
      pr.vec4 = v ? 1 : 0;
      // segments are written 4 columns at a time only (a rotary pair must not be split across the per-element path)
      if (x.seg_n && !v) return b2_fail(ctx, B2_ERR_ARG, "run_linear: column segments need 8-byte aligned planes and rotary tables");
    }
    pr.tiles_n = cdiv(x.N, GW_N);
    tiles += cdiv(x.M, GW_M) * pr.tiles_n;
    pr.tile_end = tiles;
    work += 2.0 * x.M * x.N * (x.K1 + x.K2);
    ++nz;
  }
  if (nz == 0) return B2_OK;
  if (!ok) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled failed");
  q.nprob = nz, q.tiles = tiles, q.K1 = a0.K1, q.K2 = a0.K2, q.b_per_problem = per_b ? 1 : 0;
  q.bias = a0.bias, q.ldr = a0.ldr, q.scale = a0.scale, q.ldch = a0.ldch;
  q.head_major = a0.head_major, q.relu = a0.relu, q.gelu = a0.gelu, q.lo_unscaled = a0.lo_unscaled, q.err_flag = tw.err;
  q.seg_n = a0.seg_n, q.rot_mask = a0.rot_mask;
  const std::string name = site ? std::string("k_gemm_ws/") + site : std::string("k_gemm_ws");
  b2_prof_work(ctx, name.c_str(), work);
  B2_LAUNCH_NAMED(ctx, name.c_str(), k_gemm_ws, tiles < tw.sm_count ? tiles : tw.sm_count, GW_THREADS, GW_SMEM, st, maps, q);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// One attention problem of a batched launch, as plane views (wgmma path only): q / k / v head-major [heads][n][64] with
// unscaled lo planes, o row-major [nq][ldo] (head h in columns 64 h .. 64 h + 63).
struct FlashPlanes {
  Pl q, k, v, o;
  int nq, nk;
  int heads, ldo;
};
static int run_flash_planes(b2_context* ctx, cudaStream_t st, const TcWeights& tw, const FlashPlanes* jobs, int np, float scale,
                            bool fp16_single = false) {
  if (np <= 0) return B2_OK;
  if (np > AP_MAXP) return b2_fail(ctx, B2_ERR_ARG, "run_flash: too many problems in one launch");
  if (!tma_encoder() || !tw.attn_part) return b2_fail(ctx, B2_ERR_CUDA, "wgmma attention needs cuTensorMapEncodeTiled and its scratch buffers");
  static thread_local AttnPsMaps tmaps;
  AttnPsArgs pa{};
  bool okm = true;
  int items = 0, nz = 0, W = 0, tmax = 0;
  double work = 0.0;
  for (int i = 0; i < np; ++i) {
    const FlashPlanes& j = jobs[i];
    if (j.nq <= 0 || j.nk <= 0) continue;
    AttnPsProblem& p = pa.p[nz];
    p.Qh = j.q.hi, p.Ql = j.q.lo, p.Oh = j.o.hi, p.Ol = j.o.lo, p.Nq = j.nq, p.Nk = j.nk, p.ldo = j.ldo;
    p.qt = cdiv(j.nq, 2 * AW_Q), p.tiles = cdiv(j.nk, AW_KV);
    p.item0 = items;
    items += p.qt * j.heads;
    W += p.qt * j.heads * p.tiles;
    p.w_end = W;
    tmax = p.tiles > tmax ? p.tiles : tmax;
    const uint64_t rows = (uint64_t)j.heads * j.nk;
    okm = okm && tma_map_2d(&tmaps.kh[nz], j.k.hi, rows, 64, 64, AW_KV) && tma_map_2d(&tmaps.kl[nz], j.k.lo, rows, 64, 64, AW_KV);
    okm = okm && tma_map_2d(&tmaps.vh[nz], j.v.hi, rows, 64, 64, AW_KV) && tma_map_2d(&tmaps.vl[nz], j.v.lo, rows, 64, 64, AW_KV);
    work += j.heads * 2.0 * 2.0 * 64 * (double)j.nq * j.nk;  // heads x (QK^T + PV) x 2 FLOP/MAC
    ++nz;
  }
  if (nz == 0) return B2_OK;
  if (!okm) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled failed (attention)");
  pa.nprob = nz, pa.W = W;
  int ncta = W < tw.sm_count ? W : tw.sm_count;
  pa.quota = cdiv(W, ncta);
  ncta = cdiv(W, pa.quota);
  pa.max_splits = cdiv(tmax, pa.quota) + 1;
  B2_CUDA(ctx, tw.attn_part->ensure((size_t)items * pa.max_splits * 256 * 64 * 4));
  B2_CUDA(ctx, tw.attn_ml->ensure((size_t)items * pa.max_splits * 256 * 2 * 4));
  {  // arrival counters: zero once per allocation, the kernel leaves them zero
    DevBuf& cnt = *tw.attn_cnt;
    const size_t need = (size_t)items * 2 * sizeof(int);
    if (cnt.cap < need) {
      B2_CUDA(ctx, cnt.ensure(need * 4));
      B2_CUDA(ctx, cudaMemsetAsync(cnt.p, 0, cnt.cap, st));
    }
    pa.arrivals = cnt.as<int>();
  }
  pa.Opart = tw.attn_part->as<float>(), pa.ml = tw.attn_ml->as<float>();
  pa.scale = scale, pa.err_flag = tw.err;
  b2_prof_work(ctx, "k_flash_ps", work);
  if (fp16_single) B2_LAUNCH(ctx, k_flash_ps<true>, ncta, AS_THREADS, AS_SMEM, st, tmaps, pa);
  else B2_LAUNCH(ctx, k_flash_ps<false>, ncta, AS_THREADS, AS_SMEM, st, tmaps, pa);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// One 4-head attention problem of a batched launch (LightGlue, SuperGlue).  wgmma path: q / k / v / o buffers hold split
// fp16 planes (hi, then lo at + cap * 256 halves); the SIMT path reads them as fp32.
struct FlashJob {
  const DevBuf *q, *k, *v, *o;
  int nq, nk;
  int capq, capk;  // allocated rows of the query-side / key-side buffers (lo plane offset = cap * 256 halves)
};
static int run_flash(b2_context* ctx, cudaStream_t st, const TcWeights& tw, const FlashJob* jobs, int np, float scale, bool fp16_single = false) {
  if (np <= 0) return B2_OK;
  if (np > AP_MAXP) return b2_fail(ctx, B2_ERR_ARG, "run_flash: too many problems in one launch");
  if (!tw.use_tc) {
    for (int i = 0; i < np; ++i) {
      const FlashJob& j = jobs[i];
      int rc = launch_flash(ctx, st, j.q->as<float>(), j.k->as<float>(), j.v->as<float>(), j.o->as<float>(), j.nq, j.nk, scale);
      if (rc) return rc;
    }
    return B2_OK;
  }
  FlashPlanes fp[AP_MAXP];
  for (int i = 0; i < np; ++i) {
    const FlashJob& j = jobs[i];
    fp[i] = {planes_of(*j.q, (size_t)j.capq * 256), planes_of(*j.k, (size_t)j.capk * 256), planes_of(*j.v, (size_t)j.capk * 256),
             planes_of(*j.o, (size_t)j.capq * 256), j.nq, j.nk, 4, 256};
  }
  return run_flash_planes(ctx, st, tw, fp, np, scale, fp16_single);
}
