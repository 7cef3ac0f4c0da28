// LightGlue matcher for sm_90a, as GTSfM drives it (features = "superpoint").
//
// Reference semantics restated (paths relative to the reference repo):
//   thirdparty/LightGlue/lightglue/lightglue.py:31-43 (bbox keypoint normalisation), :68-81 (rotary table),
//   :140-172 (SelfBlock), :175-230 (CrossBlock, shared-sim branch), :84-94 + :645-656 (confidence / early exit),
//   :636-643 + :551-566 (pruning), :265-318 (assignment + filter), :474-629 (_forward); wrapper
//   gtsfm/frontend/matcher/lightglue_matcher.py:43-112.
//
// HBM layout: residual streams [N][256] fp32 row-major; attention operands head-major [4][N][64]; rotary table
// cos/sin [N][32]; the (N0 x N1) similarity of the final assignment is materialised once in fp32.
#include <stdlib.h>

#include "common.cuh"
#include "linear.cuh"
#include "assign_ps.cuh"

namespace {
constexpr int LG_LAYERS = 9;
constexpr size_t LG_NFLOATS = 11851601;
constexpr int D = 256;

// w0 / b0: ffn.0 with the attention output projection folded in (weights.pack_lightglue), so it reads cat[x, ctx]
struct SelfW {
  float *wqkv, *bqkv, *w0, *b0, *lng, *lnb, *w3, *b3;  // wqkv / bqkv rows in b2_lightglue_qkv_rows order
};
struct CrossW {
  float *wqv, *bqv, *w0, *b0, *lng, *lnb, *w3, *b3;  // wqv [512][256] = [to_qk; to_v], bqv [512] likewise
};
struct AssignW {
  float *wm, *bm, *wf, *bf;
};
struct ConfW {
  float *w, *b;
};
}  // namespace

constexpr int LG_MAX_PAIRS = 8;               // pairs walked in lock-step by one batch (b2_lightglue_match_batched_*)
constexpr int LG_MAX_SIDES = 2 * LG_MAX_PAIRS;  // = GW_MAXP = AP_MAXP problems per launch
static_assert(LG_MAX_SIDES <= GW_MAXP && LG_MAX_SIDES <= AP_MAXP, "batch does not fit one launch");

struct LgSide {  // per-image workspace
  DevBuf x[2], xs[2], qkv, q, k, v, ctx, h, hs, cs[2], sn[2], ind[2], conf, mat, src, md, rmax, rlog, ls, lsg, amax, aidx;
  int cur = 0;  // which of x / xs / cs / sn / ind is live
  int n = 0;
  int cap = 0;  // rows allocated; split-plane buffers keep their lo plane at +cap * width halves whatever n shrinks to
};

struct LgPair {  // one pair of the running batch: sides 2 * slot, 2 * slot + 1
  bool active = false;  // still walking the layers
  int n0 = 0, n1 = 0;   // keypoints handed in
  int stop = 0;         // 0-based layer whose assignment head is used (lightglue.py:590-592)
  long long* out_matches = nullptr;
  float* out_scores = nullptr;
};

// One side's state after one layer, recorded when b2_set_option("lightglue_trace", 1) is set (b2_lightglue_trace_get).
struct LgTraceRec {
  int pair = 0, side = 0, layer = 0, n = 0;  // pair = index in the b2_lightglue_match_* call; n = rows going into the heads
  int heads = 0;                             // conf / mat / unconf / kept / keep are filled (pruning or early exit on, not the last layer)
  int unconf = 0, kept = 0, stop = 0;        // stop: the pair's early exit fired after this layer
  std::vector<float> x, conf, mat;
  std::vector<int> ind, keep;  // ind: original index of each row; keep: rows that survive pruning (src map, `kept` entries)
};

struct LightGlueState {
  bool loaded = false;
  int persist_ctas = 132;  // CTAs of the persistent kernels = SMs of the device minus the context's reserve_sms
  DevBuf wblob, wblob_h, wblob_l, errflag;  // fp32 weights + their split-fp16 (hi, lo * 2^11) copies for wgmma
  bool use_tc = true;                          // force_simt keeps every GEMM on the exact-fp32 SIMT kernel
  float* wr = nullptr;
  SelfW sw[LG_LAYERS];
  CrossW cw[LG_LAYERS];
  AssignW aw[LG_LAYERS];
  ConfW tw[LG_LAYERS - 1];
  float thr[LG_LAYERS];
  LgSide side[LG_MAX_SIDES];
  LgPair pair[LG_MAX_PAIRS];
  DevBuf sim[LG_MAX_PAIRS], counters, attn_part, attn_ml, attn_cnt, as_part, as_bar;
  HostBuf hread;
  std::vector<LgTraceRec> trace;
};

template <typename J>
struct JobList {  // per-problem arguments of one batched launch; blockIdx.y (or .z) selects, n == 0 entries exit at once
  J j[LG_MAX_SIDES];
};

void lg_destroy(b2_context* ctx) {
  delete ctx->lg;
  ctx->lg = nullptr;
}

// ------------------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------------------

// normalize_keypoints with size=None (lightglue.py:31-43) + LearnableFourierPositionalEncoding (:68-81).  Every block
// re-derives the bounding box (40 KB of keypoints, L2-resident) and then takes a grid-stride share of the n x 32
// (cos, sin) table.  Also initialises ind[n] = n.
struct PosJob {
  const float* kp;
  int n;
  float *cs, *sn;
  int* ind;
};
__global__ void __launch_bounds__(1024) k_lg_posenc(const __grid_constant__ JobList<PosJob> jobs, const float* __restrict__ wr /*[32][2]*/) {
  const PosJob& jb = jobs.j[blockIdx.y];
  const float* __restrict__ kp = jb.kp;
  const int n = jb.n;
  float* __restrict__ cs = jb.cs;
  float* __restrict__ sn = jb.sn;
  int* __restrict__ ind = jb.ind;
  if (n <= 0 || blockIdx.x * 1024 >= n * 32) return;  // (uniform per block)
  __shared__ float red[4][32];
  __shared__ float bb[4];
  float mnx = INFINITY, mny = INFINITY, mxx = -INFINITY, mxy = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float x = kp[2 * i], y = kp[2 * i + 1];
    mnx = fminf(mnx, x), mny = fminf(mny, y), mxx = fmaxf(mxx, x), mxy = fmaxf(mxy, y);
  }
  mnx = -warp_max(-mnx), mny = -warp_max(-mny), mxx = warp_max(mxx), mxy = warp_max(mxy);
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[0][warp] = mnx, red[1][warp] = mny, red[2][warp] = mxx, red[3][warp] = mxy;
  __syncthreads();
  if (warp == 0) {
    float a = -warp_max(-red[0][lane]), b = -warp_max(-red[1][lane]), c = warp_max(red[2][lane]), d = warp_max(red[3][lane]);
    if (lane == 0) bb[0] = a, bb[1] = b, bb[2] = c, bb[3] = d;
  }
  __syncthreads();
  // size = 1 + max - min ; shift = size / 2 ; scale = max(size) / 2
  const float sx = 1.0f + bb[2] - bb[0], sy = 1.0f + bb[3] - bb[1];
  const float shx = sx / 2.0f, shy = sy / 2.0f, sc = fmaxf(sx, sy) / 2.0f;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  for (int i = gtid; i < n * 32; i += gsz) {
    int p = i >> 5, f = i & 31;
    float x = (kp[2 * p] - shx) / sc, y = (kp[2 * p + 1] - shy) / sc;
    float pr = x * wr[2 * f] + y * wr[2 * f + 1];
    cs[i] = cosf(pr);
    sn[i] = sinf(pr);
  }
  for (int i = gtid; i < n; i += gsz) ind[i] = i;
}

// network input: x = desc (fp32 copy that the residual updates in place) + its split planes
struct LoadJob {
  const float* desc;
  int n;
  float* x;
  __half *hi, *lo;  // null on the SIMT path
};
__global__ void __launch_bounds__(256) k_lg_load_desc(const __grid_constant__ JobList<LoadJob> jobs) {
  const LoadJob& jb = jobs.j[blockIdx.y];
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= (size_t)jb.n * 256) return;
  const float4 v = *reinterpret_cast<const float4*>(jb.desc + i);
  *reinterpret_cast<float4*>(jb.x + i) = v;
  if (jb.hi) {
    uint32_t h01, l01, h23, l23;
    tc::split2(v.x, v.y, h01, l01);
    tc::split2(v.z, v.w, h23, l23);
    *reinterpret_cast<uint2*>(jb.hi + i) = make_uint2(h01, h23);
    *reinterpret_cast<uint2*>(jb.lo + i) = make_uint2(l01, l23);
  }
}

// An image's encoding (b2_lightglue_encode_batched_dev): its state after the layer-0 self block, packed row-count-major as
// x fp32 [n][256] | x hi [n][256] | x lo [n][256] (split planes, wgmma path only) | cos [n][32] | sin [n][32].
constexpr size_t LG_ENC_ROW_BYTES = 256 * 4 + 2 * 256 * 2 + 2 * 32 * 4;
struct EncJob {
  float4* blob;
  int n;
  float* x;
  __half *hi, *lo;  // null on the SIMT path: the blob's plane segments are neither written nor read
  float *cs, *sn;
  int* ind;
};
// to_blob = 1: side workspace -> blob.  0: blob -> side workspace, and ind[n] = n.
__global__ void __launch_bounds__(256) k_lg_enc_copy(const __grid_constant__ JobList<EncJob> jobs, int to_blob) {
  const EncJob& jb = jobs.j[blockIdx.y];
  const size_t n = (size_t)jb.n, g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // float4 index into the blob
  if (!to_blob && g < n) jb.ind[g] = (int)g;
  size_t i = g;
  float4* side;
  if (i < n * 64) side = reinterpret_cast<float4*>(jb.x);
  else if ((i -= n * 64) < n * 32) side = reinterpret_cast<float4*>(jb.hi);
  else if ((i -= n * 32) < n * 32) side = reinterpret_cast<float4*>(jb.lo);
  else if ((i -= n * 32) < n * 8) side = reinterpret_cast<float4*>(jb.cs);
  else if ((i -= n * 8) < n * 8) side = reinterpret_cast<float4*>(jb.sn);
  else return;
  if (!side) return;
  if (to_blob) jb.blob[g] = side[i];
  else side[i] = jb.blob[g];
}

// SIMT path: qkv [N][768] as [q | k | v] (b2_lightglue_qkv_rows) -> rotary on q,k (lightglue.py:58-65) -> fp32 [4][N][64].
// The wgmma path does the same in the projection's epilogue (gemm_ws.cuh, column segments).
struct RotJob {  // one image's share of a two-image launch (blockIdx.y)
  const float *qkv, *cs, *sn;
  int n;
  float *qo, *ko, *vo;
};
__global__ void __launch_bounds__(256) k_lg_split_rotary(const __grid_constant__ JobList<RotJob> jobs) {
  const RotJob& jb = jobs.j[blockIdx.y];
  const float* __restrict__ qkv = jb.qkv;
  const float* __restrict__ cs = jb.cs;
  const float* __restrict__ sn = jb.sn;
  const int n = jb.n;
  float* __restrict__ q = jb.qo;
  float* __restrict__ k = jb.ko;
  float* __restrict__ v = jb.vo;
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // over n * 4 * 32 pairs
  if (i >= n * 128) return;
  int p = i & 31, h = (i >> 5) & 3, r = i >> 7;
  const float* src = qkv + (size_t)r * 768 + h * 64 + 2 * p;
  float q0 = src[0], q1 = src[1], k0 = src[256], k1 = src[257], v0 = src[512], v1 = src[513];
  float c = cs[r * 32 + p], s = sn[r * 32 + p];
  size_t o = ((size_t)h * n + r) * 64 + 2 * p;
  // (t * cos) + (rotate_half(t) * sin), rotate_half: (x1, x2) -> (-x2, x1)
  const float qa = __fadd_rn(__fmul_rn(q0, c), __fmul_rn(-q1, s)), qb = __fadd_rn(__fmul_rn(q1, c), __fmul_rn(q0, s));
  const float ka = __fadd_rn(__fmul_rn(k0, c), __fmul_rn(-k1, s)), kb = __fadd_rn(__fmul_rn(k1, c), __fmul_rn(k0, s));
  q[o] = qa, q[o + 1] = qb, k[o] = ka, k[o + 1] = kb, v[o] = v0, v[o + 1] = v1;
}

// LayerNorm(512, eps 1e-5, affine) + exact GELU in place (lightglue.py:152-157). one warp per row.
// When `hi` is given the result is written as split fp16 planes (the next GEMM's A operand) instead of in place.
struct LnJob {  // one image's share of a two-image launch (blockIdx.y)
  float* h;
  int n;
  __half *hi, *lo;
};
__global__ void __launch_bounds__(256) k_lg_ln_gelu(const __grid_constant__ JobList<LnJob> jobs, const float* __restrict__ g, const float* __restrict__ b) {
  const LnJob& jb = jobs.j[blockIdx.y];
  float* __restrict__ h = jb.h;
  __half* __restrict__ hi = jb.hi;
  __half* __restrict__ lo = jb.lo;
  const int n = jb.n;
  int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n) return;
  float4* row = reinterpret_cast<float4*>(h + (size_t)r * 512);
  float4 v[4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = row[lane + 32 * i];
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  float mean = warp_sum(s) / 512.0f;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + bq * bq + c * c + d * d;
  }
  float rstd = 1.0f / sqrtf(warp_sum(q) / 512.0f + 1e-5f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int c0 = (lane + 32 * i) * 4;
    float4 gg = *reinterpret_cast<const float4*>(g + c0), bb = *reinterpret_cast<const float4*>(b + c0);
    float e[4] = {(v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y,
                  (v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) e[j] = 0.5f * e[j] * (1.0f + erff(e[j] * 0.70710678118654752440f));
    if (hi) {
      uint32_t h01, l01, h23, l23;
      tc::split2(e[0], e[1], h01, l01);
      tc::split2(e[2], e[3], h23, l23);
      *reinterpret_cast<uint2*>(hi + (size_t)r * 512 + c0) = make_uint2(h01, h23);
      *reinterpret_cast<uint2*>(lo + (size_t)r * 512 + c0) = make_uint2(l01, l23);
    } else {
      row[lane + 32 * i] = make_float4(e[0], e[1], e[2], e[3]);
    }
  }
}

// two per-row heads in one pass: sigmoid(w1.x + b1) and sigmoid(w2.x + b2) (token confidence :84-94, matchability
// :298-299).  Also raw logit of head 2 when zraw != null.  one warp per row.
struct HeadJob {  // one image's share of a two-image launch (blockIdx.y)
  const float* x;
  int n;
  const float *w2, *b2;  // head 2 may be off for one image only (pruning threshold on the keypoint count)
  float *o1, *o2, *zraw;
};
__global__ void __launch_bounds__(256) k_lg_rowheads(const __grid_constant__ JobList<HeadJob> jobs, const float* __restrict__ w1,
                                                      const float* __restrict__ b1) {
  const HeadJob& jb = jobs.j[blockIdx.y];
  const float* __restrict__ x = jb.x;
  const float* __restrict__ w2 = jb.w2;
  const float* __restrict__ b2 = jb.b2;
  float* __restrict__ o1 = jb.o1;
  float* __restrict__ o2 = jb.o2;
  float* __restrict__ zraw = jb.zraw;
  const int n = jb.n;
  int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n) return;
  const float4* row = reinterpret_cast<const float4*>(x + (size_t)r * 256);
  float4 a = row[lane], b = row[lane + 32];
  float s1 = 0.f, s2 = 0.f;
  if (w1) {
    float4 wa = reinterpret_cast<const float4*>(w1)[lane], wb = reinterpret_cast<const float4*>(w1)[lane + 32];
    s1 = a.x * wa.x + a.y * wa.y + a.z * wa.z + a.w * wa.w + b.x * wb.x + b.y * wb.y + b.z * wb.z + b.w * wb.w;
  }
  if (w2) {
    float4 wa = reinterpret_cast<const float4*>(w2)[lane], wb = reinterpret_cast<const float4*>(w2)[lane + 32];
    s2 = a.x * wa.x + a.y * wa.y + a.z * wa.z + a.w * wa.w + b.x * wb.x + b.y * wb.y + b.z * wb.z + b.w * wb.w;
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  if (lane == 0) {
    if (w1) o1[r] = 1.0f / (1.0f + expf(-(s1 + b1[0])));
    if (w2) {
      float z = s2 + b2[0];
      if (o2) o2[r] = 1.0f / (1.0f + expf(-z));
      if (zraw) zraw[r] = z;
    }
  }
}

// pruning decision + ordered compaction map for one image (single block):
//   counters[0 + side] += #(conf < thr)            (check_if_stop numerator, lightglue.py:653-655)
//   keep = matchability > (1 - width_conf) | conf <= thr   (:636-643); src[pos] = old index; counters[2 + side] = #kept
struct PruneJob {  // one image's share of a batched launch (blockIdx.y)
  const float *conf, *mat;
  int n;
  int* src;
  int* counters;  // this image's pair: [0 + side] unconfident, [2 + side] kept
  int side;
};
__global__ void __launch_bounds__(1024) k_lg_prune_plan(const __grid_constant__ JobList<PruneJob> jobs, float thr, float keep_thr) {
  const PruneJob& jb = jobs.j[blockIdx.y];
  const int side = jb.side;
  int* __restrict__ counters = jb.counters;
  if (jb.n <= 0) return;
  const float* __restrict__ conf = jb.conf;
  const float* __restrict__ mat = jb.mat;
  int* __restrict__ src = jb.src;
  const int n = jb.n;
  __shared__ int wtot[32];
  __shared__ int carry, unconf;
  if (threadIdx.x == 0) carry = 0, unconf = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    int i = base + threadIdx.x;
    bool keep = false, unc = false;
    if (i < n) {
      float c = conf[i];
      unc = c < thr;
      keep = (mat[i] > keep_thr) || (c <= thr);
    }
    unsigned km = __ballot_sync(0xffffffffu, keep), um = __ballot_sync(0xffffffffu, unc);
    if (lane == 0) wtot[warp] = __popc(km);
    if (lane == 0 && um) atomicAdd(&unconf, __popc(um));
    __syncthreads();
    if (warp == 0) {
      int w = wtot[lane], ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int u = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += u;
      }
      wtot[lane] = ws - w;
    }
    __syncthreads();
    int pos = carry + wtot[warp] + __popc(km & ((1u << lane) - 1));
    if (keep) src[pos] = i;
    __syncthreads();
    if (threadIdx.x == 1023) carry = pos + (keep ? 1 : 0);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counters[side] = unconf;
    counters[2 + side] = carry;
  }
}

// gather rows by src map: x [n][256], cos/sin [n][32], ind [n]  (lightglue.py:556-566)
struct GatherJob {
  const int *src, *cnt;
  int n;  // rows before pruning (launch bound); *cnt rows are written
  const float *x, *cs, *sn;
  const int* ind;
  float *x2, *cs2, *sn2;
  int* ind2;
  const __half* ph;  // split planes of x travel with it (null on the SIMT path)
  size_t pstride;
  __half* ph2;
  size_t pstride2;
};
__global__ void __launch_bounds__(256) k_lg_gather(const __grid_constant__ JobList<GatherJob> jobs) {
  const GatherJob& jb = jobs.j[blockIdx.y];
  int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (jb.n <= 0 || r >= *jb.cnt) return;
  int s = jb.src[r];
  const float4* a = reinterpret_cast<const float4*>(jb.x + (size_t)s * 256);
  float4* o = reinterpret_cast<float4*>(jb.x2 + (size_t)r * 256);
  o[lane] = a[lane];
  o[lane + 32] = a[lane + 32];
  jb.cs2[r * 32 + lane] = jb.cs[s * 32 + lane];
  jb.sn2[r * 32 + lane] = jb.sn[s * 32 + lane];
  if (lane == 0) jb.ind2[r] = jb.ind[s];
  if (jb.ph) {  // 256 halves = 32 lanes x 16 bytes per plane
    reinterpret_cast<uint4*>(jb.ph2 + (size_t)r * 256)[lane] = reinterpret_cast<const uint4*>(jb.ph + (size_t)s * 256)[lane];
    reinterpret_cast<uint4*>(jb.ph2 + jb.pstride2 + (size_t)r * 256)[lane] = reinterpret_cast<const uint4*>(jb.ph + jb.pstride + (size_t)s * 256)[lane];
  }
}

// log-softmax statistics of sim rows: max and log(sum(exp(x - max)))  (F.log_softmax, lightglue.py:271). warp per row.
__device__ __forceinline__ float logsigmoid(float z) {  // F.logsigmoid: min(z, 0) - log1p(exp(-|z|))
  return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
}

// Row statistics of log_softmax(sim, dim 2) (:271): warp per row.  Also tabulates logsigmoid(z) of the row's
// matchability logit so the arg-max passes do not re-evaluate it per matrix element.
__global__ void __launch_bounds__(256) k_lg_row_stats(const float* __restrict__ sim, int m, int n, float* __restrict__ rmax,
                                                       float* __restrict__ rlog, const float* __restrict__ z,
                                                       float* __restrict__ lsg) {
  int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= m) return;
  const float* row = sim + (size_t)r * n;
  float mx = -INFINITY;
  for (int j = lane; j < n; j += 32) mx = fmaxf(mx, row[j]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int j = lane; j < n; j += 32) s += expf(row[j] - mx);
  s = warp_sum(s);
  if (lane == 0) rmax[r] = mx, rlog[r] = logf(s), lsg[r] = logsigmoid(z[r]);
}
// same along columns (log_softmax of sim^T, :272): a block owns 32 columns; its 32 warps stride over the rows (each row
// access is one coalesced 128-byte line, four independent loads in flight per warp - the pass is load-latency bound),
// keeping an online (max, sum) pair that is merged across warps at the end.
constexpr int LG_COL_WARPS = 32, LG_COL_UNROLL = 4;
__global__ void __launch_bounds__(1024) k_lg_col_stats(const float* __restrict__ sim, int m, int n, float* __restrict__ cmax,
                                                        float* __restrict__ clog, const float* __restrict__ z,
                                                        float* __restrict__ lsg) {
  __shared__ float sm[LG_COL_WARPS][32], ss[LG_COL_WARPS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  float mx = -INFINITY, s = 0.f;
  if (j < n) {
    for (int i0 = warp; i0 < m; i0 += LG_COL_WARPS * LG_COL_UNROLL) {
      float x[LG_COL_UNROLL];
#pragma unroll
      for (int u = 0; u < LG_COL_UNROLL; ++u) {
        const int i = i0 + u * LG_COL_WARPS;
        x[u] = i < m ? sim[(size_t)i * n + j] : -INFINITY;
      }
#pragma unroll
      for (int u = 0; u < LG_COL_UNROLL; ++u) {
        if (x[u] > mx) {
          s = s * expf(mx - x[u]) + 1.0f;
          mx = x[u];
        } else if (x[u] > -INFINITY) {
          s += expf(x[u] - mx);
        }
      }
    }
  }
  sm[warp][lane] = mx, ss[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && j < n) {
    float M = sm[0][lane];
    for (int w = 1; w < LG_COL_WARPS; ++w) M = fmaxf(M, sm[w][lane]);
    float S = 0.f;
    for (int w = 0; w < LG_COL_WARPS; ++w)
      if (ss[w][lane] > 0.f) S += ss[w][lane] * expf(sm[w][lane] - M);
    cmax[j] = M, clog[j] = logf(S), lsg[j] = logsigmoid(z[j]);
  }
}

// scores[i][j] = (log_softmax_rows + log_softmax_cols) + (logsigmoid(z0_i) + logsigmoid(z1_j))  (:269-274);
// row arg-max (first maximum) per i. warp per row.  l0 / l1 = the tabulated logsigmoid terms.
__global__ void __launch_bounds__(256) k_lg_row_argmax(const float* __restrict__ sim, int m, int n,
                                                        const float* __restrict__ rmax, const float* __restrict__ rlog,
                                                        const float* __restrict__ cmax, const float* __restrict__ clog,
                                                        const float* __restrict__ l0g, const float* __restrict__ l1g,
                                                        float* __restrict__ best, int* __restrict__ arg) {
  int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= m) return;
  const float* row = sim + (size_t)r * n;
  const float rm = rmax[r], rl = rlog[r], l0 = l0g[r];
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < n; j += 32) {
    float x = row[j];
    float sc = (((x - rm) - rl) + ((x - cmax[j]) - clog[j])) + (l0 + l1g[j]);
    if (sc > bv) bv = sc, bi = j;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
  }
  if (lane == 0) best[r] = bv, arg[r] = bi == 0x7fffffff ? 0 : bi;  // no score beat -inf (a NaN row): best -inf, never a match
}
__global__ void __launch_bounds__(1024) k_lg_col_argmax(const float* __restrict__ sim, int m, int n,
                                                         const float* __restrict__ rmax, const float* __restrict__ rlog,
                                                         const float* __restrict__ cmax, const float* __restrict__ clog,
                                                         const float* __restrict__ l0g, const float* __restrict__ l1g,
                                                         int* __restrict__ arg) {
  __shared__ float sv[LG_COL_WARPS][32];
  __shared__ int si[LG_COL_WARPS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  if (j < n) {
    const float cm = cmax[j], cl = clog[j], l1 = l1g[j];
    for (int i0 = warp; i0 < m; i0 += LG_COL_WARPS * LG_COL_UNROLL) {
      float x[LG_COL_UNROLL], rm[LG_COL_UNROLL], rl[LG_COL_UNROLL], l0[LG_COL_UNROLL];
#pragma unroll
      for (int u = 0; u < LG_COL_UNROLL; ++u) {
        const int i = i0 + u * LG_COL_WARPS;
        const bool in = i < m;
        x[u] = in ? sim[(size_t)i * n + j] : 0.f;
        rm[u] = in ? rmax[i] : 0.f, rl[u] = in ? rlog[i] : 0.f, l0[u] = in ? l0g[i] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < LG_COL_UNROLL; ++u) {
        const int i = i0 + u * LG_COL_WARPS;
        if (i < m) {
          const float sc = (((x[u] - rm[u]) - rl[u]) + ((x[u] - cm) - cl)) + (l0[u] + l1);
          if (sc > bv) bv = sc, bi = i;  // rows ascend within a warp: first maximum kept
        }
      }
    }
  }
  sv[warp][lane] = bv, si[warp][lane] = bi;
  __syncthreads();
  if (warp == 0 && j < n) {
    for (int w = 1; w < LG_COL_WARPS; ++w) {
      float ov = sv[w][lane];
      int oi = si[w][lane];
      if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
    }
    arg[j] = bi == 0x7fffffff ? 0 : bi;
  }
}

// filter_matches (:302-318) + index mapping through ind0 / ind1 (:598-602) + ordered compaction (single block).
__global__ void __launch_bounds__(1024) k_lg_filter(const float* __restrict__ best0, const int* __restrict__ a0,
                                                     const int* __restrict__ a1, int m, float th, const int* __restrict__ ind0,
                                                     const int* __restrict__ ind1, long long* __restrict__ out,
                                                     float* __restrict__ outs, int* __restrict__ count) {
  __shared__ int wtot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < m; base += 1024) {
    int i = base + threadIdx.x;
    bool valid = false;
    float ms = 0.f;
    int j = 0;
    if (i < m) {
      j = a0[i];
      bool mutual = a1[j] == i;
      ms = mutual ? expf(best0[i]) : 0.f;
      valid = mutual && best0[i] > -INFINITY && ms > th;  // a row without an arg-max (best -inf) never matches, whatever th is
    }
    unsigned vm = __ballot_sync(0xffffffffu, valid);
    if (lane == 0) wtot[warp] = __popc(vm);
    __syncthreads();
    if (warp == 0) {
      int w = wtot[lane], ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int u = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += u;
      }
      wtot[lane] = ws - w;
    }
    __syncthreads();
    int pos = carry + wtot[warp] + __popc(vm & ((1u << lane) - 1));
    if (valid) {
      out[2 * (size_t)pos] = ind0[i];
      out[2 * (size_t)pos + 1] = ind1[j];
      if (outs) outs[pos] = ms;
    }
    __syncthreads();
    if (threadIdx.x == 1023) carry = pos + (valid ? 1 : 0);
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = carry;
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------

// The assignment step on the similarity sim [M][N]: the row / column log-softmax statistics and logsigmoid terms of
// sigmoid_log_double_softmax (lightglue.py:265-277), the mutual arg-max and threshold of filter_matches (:302-318), and
// the match list mapped through ind0 / ind1 (:598-602).
struct LgStats {
  float *max, *log, *lsg;  // per row (or column): max, log of the sum of exp(x - max), logsigmoid of the matchability logit
};
struct LgAssign {
  const float* sim;
  int M, N;
  const float *z0, *z1;  // matchability logits [M], [N]
  const int *ind0, *ind1;
  float thr;
  LgStats r, c;
  float* best0;
  int *arg0, *arg1;
  DevBuf *part, *bar;  // scratch of the persistent kernel
  int* err_flag;
  long long* out_matches;
  float* out_scores;
  int* count;
};

// The statistics and the mutual arg-max (everything before the filter).  path 0 runs the persistent kernel when it fits
// (what the matcher does), 1 forces it, 2 forces the multi-launch passes; G is the persistent kernel's CTA count.  *ran
// (when given) receives the path that ran, 1 or 2.
static int lg_assign_argmax(b2_context* ctx, cudaStream_t st, const LgAssign& p, int path, int G, int* ran) {
  const float* sim = p.sim;
  const int M = p.M, N = p.N;
  const bool persistent = path == 0 ? assign_ps_fits(1, N) : path == 1;
  if (persistent && !assign_ps_fits(1, N)) return b2_fail(ctx, B2_ERR_ARG, "the persistent assignment kernel holds at most 6240 columns");
  if (ran) *ran = persistent ? 1 : 2;
  int rc;
  if (persistent) {
    // persistent cooperative kernel (assign_ps.cuh, KIND 1): row / column log-softmax statistics in one sweep of the
    // similarity, mutual arg-max in a second one - 2 reads and 1 launch instead of 4 and 4
    B2_CUDA(ctx, p.part->ensure((size_t)G * 2 * N * sizeof(float)));
    B2_CUDA(ctx, p.bar->ensure(16));
    B2_CUDA(ctx, cudaMemsetAsync(p.bar->p, 0, 16, st));
    SinkArgs sa{};
    sa.Z = sim, sa.M = M, sa.N = N, sa.iters = 1, sa.u = p.r.max, sa.v = p.c.max;
    sa.rlog = p.r.log, sa.clog = p.c.log, sa.z0 = p.z0, sa.z1 = p.z1;
    sa.lsg0 = p.r.lsg, sa.lsg1 = p.c.lsg, sa.part = p.part->as<float>(), sa.bar = p.bar->as<unsigned>();
    sa.best0 = p.best0, sa.arg0 = p.arg0, sa.arg1 = p.arg1, sa.err_flag = p.err_flag;
    if ((rc = launch_assign_ps<1>(ctx, st, sa, G, "k_lg_assign"))) return rc;
  } else {
    B2_LAUNCH(ctx, k_lg_row_stats, cdiv(M, 8), 256, 0, st, sim, M, N, p.r.max, p.r.log, p.z0, p.r.lsg);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_lg_col_stats, cdiv(N, 32), 1024, 0, st, sim, M, N, p.c.max, p.c.log, p.z1, p.c.lsg);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_lg_row_argmax, cdiv(M, 8), 256, 0, st, sim, M, N, p.r.max, p.r.log, p.c.max, p.c.log, p.r.lsg, p.c.lsg, p.best0,
              p.arg0);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_lg_col_argmax, cdiv(N, 32), 1024, 0, st, sim, M, N, p.r.max, p.r.log, p.c.max, p.c.log, p.r.lsg, p.c.lsg, p.arg1);
    B2_CHECK_LAUNCH(ctx);
  }
  return B2_OK;
}

static int lg_assign(b2_context* ctx, cudaStream_t st, const LgAssign& p, int path, int G, int* ran) {
  const int M = p.M;
  int rc;
  if ((rc = lg_assign_argmax(ctx, st, p, path, G, ran))) return rc;
  B2_LAUNCH(ctx, k_lg_filter, 1, 1024, 0, st, p.best0, p.arg0, p.arg1, M, p.thr, p.ind0, p.ind1, p.out_matches, p.out_scores, p.count);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// Row r of the device copy of a self block's QKV projection (weight and bias) is row out[r] of the checkpoint's.  The
// checkpoint interleaves q, k, v per feature, (h * 64 + j) * 3 + {q, k, v} (lightglue.py:166-167); the device copy is
// [q | k | v], each 256 rows in head-major order h * 64 + j, so the rotary pair (2p, 2p + 1) of a head is two adjacent
// output columns and each of q, k, v is one column segment of the GEMM.  Every output is the same dot product as before.
extern "C" int b2_lightglue_qkv_rows(int* out) {
  if (!out) return B2_ERR_ARG;
  for (int r = 0; r < 3 * D; ++r) out[r] = (r % D) * 3 + r / D;
  return B2_OK;
}

extern "C" int b2_lightglue_set_weights(b2_context* ctx, const float* blob, size_t n_floats) {
  if (!ctx || !blob) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (n_floats != LG_NFLOATS)
    return b2_fail(ctx, B2_ERR_ARG, "lightglue blob must hold 11851601 floats, got " + std::to_string(n_floats));
  cudaSetDevice(ctx->device);
  if (!ctx->lg) ctx->lg = new LightGlueState();
  LightGlueState* s = ctx->lg;
  // device copy with every tensor 256-byte aligned
  std::vector<size_t> sizes;
  sizes.push_back(64);  // posenc.Wr
  for (int i = 0; i < LG_LAYERS; ++i) {
    const size_t self_sz[] = {768 * 256, 768, 256 * 256, 256, 512 * 512, 512, 512, 512, 256 * 512, 256};
    const size_t cross_sz[] = {256 * 256, 256, 256 * 256, 256, 256 * 256, 256, 512 * 512, 512, 512, 512, 256 * 512, 256};
    for (size_t z : self_sz) sizes.push_back(z);
    for (size_t z : cross_sz) sizes.push_back(z);
  }
  for (int i = 0; i < LG_LAYERS; ++i) {
    const size_t asz[] = {256, 1, 256 * 256, 256};
    for (size_t z : asz) sizes.push_back(z);
  }
  for (int i = 0; i < LG_LAYERS - 1; ++i) sizes.push_back(256), sizes.push_back(1);
  // device placement: the blob order, except that each cross block's to_v weight goes right after its to_qk weight (and
  // the biases likewise), so that [to_qk; to_v] is one [512][256] operand (a 256 x 256 tensor fills whole 64-float slots)
  constexpr int SELF_T = 10, LAYER_T = 22;  // tensors per self block, per layer (self + cross)
  std::vector<size_t> order(sizes.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  for (int i = 0; i < LG_LAYERS; ++i) std::swap(order[1 + LAYER_T * i + SELF_T + 1], order[1 + LAYER_T * i + SELF_T + 2]);
  size_t total = 0, src_total = 0;
  std::vector<size_t> doff(sizes.size()), soff(sizes.size());
  for (size_t k : order) {
    doff[k] = total;
    total += (sizes[k] + 63) / 64 * 64;
  }
  for (size_t i = 0; i < sizes.size(); ++i) soff[i] = src_total, src_total += sizes[i];
  if (src_total != LG_NFLOATS) return b2_fail(ctx, B2_ERR_STATE, "internal lightglue layout mismatch");
  for (int i = 0; i < LG_LAYERS; ++i)  // out_proj, to_out
    for (size_t t : {1 + LAYER_T * i + 2, 1 + LAYER_T * i + SELF_T + 4})
      if (!folded_projection(blob + soff[t], blob + soff[t + 1], D))
        return b2_fail(ctx, B2_ERR_ARG, "lightglue blob: layer " + std::to_string(i) + "'s attention output projections are not folded "
                                        "into ffn.0 (pack the checkpoint with weights.pack_lightglue)");
  std::vector<float> host(total, 0.f);
  for (size_t i = 0; i < sizes.size(); ++i) memcpy(host.data() + doff[i], blob + soff[i], sizes[i] * sizeof(float));
  int qkv_rows[3 * D];
  b2_lightglue_qkv_rows(qkv_rows);
  for (int i = 0; i < LG_LAYERS; ++i) {  // self QKV weight and bias rows -> [q | k | v]
    const size_t tw = 1 + LAYER_T * i, tb = tw + 1;
    for (int r = 0; r < 3 * D; ++r) {
      memcpy(host.data() + doff[tw] + (size_t)r * D, blob + soff[tw] + (size_t)qkv_rows[r] * D, D * sizeof(float));
      host[doff[tb] + r] = blob[soff[tb] + qkv_rows[r]];
    }
  }
  B2_CUDA(ctx, s->wblob.ensure(total * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->wblob.p, host.data(), total * sizeof(float), cudaMemcpyHostToDevice));
  float* base = s->wblob.as<float>();
  size_t ti = 0;
  auto next = [&]() { return base + doff[ti++]; };
  s->wr = next();
  for (int i = 0; i < LG_LAYERS; ++i) {
    SelfW& a = s->sw[i];
    a.wqkv = next(), a.bqkv = next(), next(), next();  // out_proj: the identity (folded)
    a.w0 = next(), a.b0 = next(), a.lng = next(), a.lnb = next(), a.w3 = next(), a.b3 = next();
    CrossW& c = s->cw[i];
    c.wqv = next(), c.bqv = next(), next(), next();  // to_v's weight and bias sit right behind to_qk's
    next(), next();                                  // to_out: the identity (folded)
    c.w0 = next(), c.b0 = next(), c.lng = next(), c.lnb = next(), c.w3 = next(), c.b3 = next();
  }
  for (int i = 0; i < LG_LAYERS; ++i) {
    AssignW& a = s->aw[i];
    a.wm = next(), a.bm = next(), a.wf = next(), a.bf = next();
  }
  for (int i = 0; i < LG_LAYERS - 1; ++i) s->tw[i].w = next(), s->tw[i].b = next();
  // confidence_threshold buffer (lightglue.py:631-634) evaluated in double then stored as float32 like torch.Tensor([...])
  for (int i = 0; i < LG_LAYERS; ++i) {
    double t = 0.8 + 0.1 * exp(-4.0 * i / LG_LAYERS);
    t = t < 0 ? 0 : (t > 1 ? 1 : t);
    s->thr[i] = (float)t;
  }
  B2_CUDA(ctx, s->wblob_h.ensure(total * sizeof(__half)));
  B2_CUDA(ctx, s->wblob_l.ensure(total * sizeof(__half)));
  B2_CUDA(ctx, s->errflag.ensure(16));
  B2_CUDA(ctx, cudaMemset(s->errflag.p, 0, 16));
  B2_LAUNCH(ctx, k_split_f32, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)0, s->wblob.as<float>(), total,
            s->wblob_h.as<__half>(), s->wblob_l.as<__half>());
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaDeviceSynchronize());
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  s->use_tc = !b2_force_simt(ctx);
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_attn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FA_SMEM));
  B2_CUDA(ctx, s->hread.ensure(8 * LG_MAX_PAIRS * sizeof(int)));
  B2_CUDA(ctx, s->counters.ensure(8 * LG_MAX_PAIRS * sizeof(int)));
  B2_CUDA(ctx, cudaMemset(s->counters.p, 0, 8 * LG_MAX_PAIRS * sizeof(int)));
  s->loaded = true;
  return B2_OK;
}

static inline TcWeights lg_tw(LightGlueState* s) {
  TcWeights t{s->wblob.as<float>(), s->wblob_h.as<__half>(), s->wblob_l.as<__half>(), s->errflag.as<int>(), s->use_tc};
  t.attn_part = &s->attn_part, t.attn_ml = &s->attn_ml, t.attn_cnt = &s->attn_cnt, t.sm_count = s->persist_ctas;
  return t;
}

static int lg_side_alloc(b2_context* ctx, LgSide& sd, int n, bool use_tc) {
  const size_t N = (size_t)(n > 0 ? n : 1);
  for (int i = 0; i < 2; ++i) {
    B2_CUDA(ctx, sd.x[i].ensure(N * 256 * 4));
    B2_CUDA(ctx, sd.xs[i].ensure(N * 256 * 4));
    B2_CUDA(ctx, sd.cs[i].ensure(N * 32 * 4));
    B2_CUDA(ctx, sd.sn[i].ensure(N * 32 * 4));
    B2_CUDA(ctx, sd.ind[i].ensure(N * 4));
  }
  if (!use_tc) B2_CUDA(ctx, sd.qkv.ensure(N * 768 * 4));  // the wgmma path writes q / k / v from the projection directly
  B2_CUDA(ctx, sd.q.ensure(N * 256 * 4));
  B2_CUDA(ctx, sd.k.ensure(N * 256 * 4));
  B2_CUDA(ctx, sd.v.ensure(N * 256 * 4));
  B2_CUDA(ctx, sd.ctx.ensure(N * 256 * 4));
  B2_CUDA(ctx, sd.h.ensure(N * 512 * 4));
  B2_CUDA(ctx, sd.hs.ensure(N * 512 * 4));
  B2_CUDA(ctx, sd.md.ensure(N * 256 * 4));
  DevBuf* small[] = {&sd.conf, &sd.mat, &sd.src, &sd.rmax, &sd.rlog, &sd.ls, &sd.lsg, &sd.amax, &sd.aidx};
  for (DevBuf* b : small) B2_CUDA(ctx, b->ensure(N * 4));
  sd.cur = 0;
  sd.n = n;
  sd.cap = n;
  return B2_OK;
}

// The sides (images) of the pairs that are still walking the layers, in launch order.
struct LgActive {
  int side[LG_MAX_SIDES];
  int n = 0;
};
static LgActive lg_active_sides(const LightGlueState* s, int np) {
  LgActive a;
  for (int p = 0; p < np; ++p)
    if (s->pair[p].active) a.side[a.n++] = 2 * p, a.side[a.n++] = 2 * p + 1;
  return a;
}
static int lg_max_n(const LightGlueState* s, const LgActive& act) {
  int mx = 0;
  for (int i = 0; i < act.n; ++i) mx = s->side[act.side[i]].n > mx ? s->side[act.side[i]].n : mx;
  return mx;
}

// x + ffn(cat[x, msg]) with msg = out(ctx)  (lightglue.py:152-157,172,228-229): Linear(512,512) -> LN -> GELU ->
// Linear(512,256) + x.  The message projection (out_proj / to_out) is folded into the first linear on the host
// (weights.fold_message_projection), so that linear reads cat[x, ctx] straight from the attention output; every image of
// the batch goes through each GEMM together.  `blk` ("lg_self" / "lg_cross") prefixes the profiler labels of the two GEMM
// call sites.
static int lg_ffn(b2_context* ctx, cudaStream_t st, LightGlueState* s, const LgActive& act, const char* blk, const float* w0,
                  const float* b0, const float* lng, const float* lnb, const float* w3, const float* b3) {
  int rc;
  const TcWeights tw = lg_tw(s);
  LinArgs f0[LG_MAX_SIDES], f3[LG_MAX_SIDES];
  for (int i = 0; i < act.n; ++i) {
    LgSide& sd = s->side[act.side[i]];
    const size_t e = (size_t)sd.cap * 256;
    float* x = sd.x[sd.cur].as<float>();
    LinArgs& f = f0[i];
    f.a1f = x, f.a1p = planes_of(sd.xs[sd.cur], e), f.lda1 = 256, f.K1 = 256;
    f.a2f = sd.ctx.as<float>(), f.a2p = planes_of(sd.ctx, e), f.lda2 = 256, f.K2 = 256;
    f.w = w0, f.ldb = 512, f.bias = b0, f.cf = sd.h.as<float>(), f.ldc = 512, f.tc_want_f32 = true, f.M = sd.n, f.N = 512;
    LinArgs& c = f3[i];
    c.a1f = sd.h.as<float>(), c.a1p = planes_of(sd.hs, (size_t)sd.cap * 512), c.lda1 = 512, c.K1 = 512, c.w = w3, c.ldb = 512, c.bias = b3;
    c.resid = x, c.ldr = 256;  // in place: every element is read (as residual) and written by the same thread
    c.cf = x, c.ldc = 256, c.tc_want_f32 = true, c.cp = planes_of(sd.xs[sd.cur], e), c.ldch = 256, c.M = sd.n, c.N = 256;
  }
  const std::string site(blk);
  if ((rc = run_linear(ctx, st, tw, f0, act.n, (site + "_ffn0").c_str()))) return rc;
  {
    JobList<LnJob> lj{};
    for (int i = 0; i < act.n; ++i) {
      LgSide& sd = s->side[act.side[i]];
      const Pl hs = planes_of(sd.hs, (size_t)sd.cap * 512);
      lj.j[i] = {sd.h.as<float>(), sd.n, s->use_tc ? hs.hi : (__half*)nullptr, s->use_tc ? hs.lo : (__half*)nullptr};
    }
    const int mx = lg_max_n(s, act);
    if (mx > 0) {
      B2_LAUNCH(ctx, k_lg_ln_gelu, dim3(cdiv(mx, 8), act.n), 256, 0, st, lj, lng, lnb);
      B2_CHECK_LAUNCH(ctx);
    }
  }
  return run_linear(ctx, st, tw, f3, act.n, (site + "_ffn3").c_str());
}

static int lg_self_layer(b2_context* ctx, cudaStream_t st, LightGlueState* s, const LgActive& act, int layer, bool fp16_attn) {
  const SelfW& w = s->sw[layer];
  const TcWeights tw = lg_tw(s);
  int rc;
  // wgmma path: one launch writes rotated q, k and unrotated v as head-major planes with unscaled lo (attention operands);
  // SIMT path: qkv fp32 [N][768], then the rotary kernel
  LinArgs q[LG_MAX_SIDES];
  for (int i = 0; i < act.n; ++i) {
    LgSide& sd = s->side[act.side[i]];
    const size_t e = (size_t)sd.cap * 256;
    LinArgs& a = q[i];
    a.a1f = sd.x[sd.cur].as<float>(), a.a1p = planes_of(sd.xs[sd.cur], e), a.lda1 = 256, a.K1 = 256;
    a.w = w.wqkv, a.ldb = 256, a.bias = w.bqkv, a.M = sd.n, a.N = 768;
    if (s->use_tc) {
      a.seg_n = 256, a.seg_p[0] = planes_of(sd.q, e), a.seg_p[1] = planes_of(sd.k, e), a.seg_p[2] = planes_of(sd.v, e);
      a.rot_mask = 3, a.cs = sd.cs[sd.cur].as<float>(), a.sn = sd.sn[sd.cur].as<float>();
      a.head_major = 1, a.lo_unscaled = 1;
    } else {
      a.cf = sd.qkv.as<float>(), a.ldc = 768;
    }
  }
  if ((rc = run_linear(ctx, st, tw, q, act.n, "lg_self_qkv"))) return rc;
  const int mx = lg_max_n(s, act);
  if (!s->use_tc && mx > 0) {
    JobList<RotJob> rj{};
    for (int i = 0; i < act.n; ++i) {
      LgSide& sd = s->side[act.side[i]];
      rj.j[i] = {sd.qkv.as<float>(), sd.cs[sd.cur].as<float>(), sd.sn[sd.cur].as<float>(), sd.n, sd.q.as<float>(), sd.k.as<float>(), sd.v.as<float>()};
    }
    B2_LAUNCH(ctx, k_lg_split_rotary, dim3(cdiv(mx * 128, 256), act.n), 256, 0, st, rj);
    B2_CHECK_LAUNCH(ctx);
  }
  FlashJob fj[LG_MAX_SIDES];
  for (int i = 0; i < act.n; ++i) {
    LgSide& a = s->side[act.side[i]];
    fj[i] = {&a.q, &a.k, &a.v, &a.ctx, a.n, a.n, a.cap, a.cap};
  }
  if ((rc = run_flash(ctx, st, tw, fj, act.n, 0.125f, fp16_attn))) return rc;
  return lg_ffn(ctx, st, s, act, "lg_self", w.w0, w.b0, w.lng, w.lnb, w.w3, w.b3);
}

static int lg_cross_block(b2_context* ctx, cudaStream_t st, LightGlueState* s, const LgActive& act, int layer, bool fp16_attn) {
  const CrossW& w = s->cw[layer];
  const TcWeights tw = lg_tw(s);
  int rc;
  LinArgs p[LG_MAX_SIDES];  // [to_qk; to_v] in one launch: columns 0-255 -> sd.q, 256-511 -> sd.v, both head-major [4][n][64]
  for (int i = 0; i < act.n; ++i) {
    LgSide& sd = s->side[act.side[i]];
    const size_t e = (size_t)sd.cap * 256;
    LinArgs& a = p[i];
    a.a1f = sd.x[sd.cur].as<float>(), a.a1p = planes_of(sd.xs[sd.cur], e), a.lda1 = 256, a.K1 = 256;
    a.w = w.wqv, a.ldb = 256, a.bias = w.bqv, a.head_major = 1, a.M = sd.n, a.N = 512;
    a.seg_n = 256, a.seg_f[0] = sd.q.as<float>(), a.seg_f[1] = sd.v.as<float>(), a.seg_p[0] = planes_of(sd.q, e), a.seg_p[1] = planes_of(sd.v, e);
    a.lo_unscaled = s->use_tc ? 1 : 0;  // attention operands
  }
  if ((rc = run_linear(ctx, st, tw, p, act.n, "lg_cross_qv"))) return rc;
  // m0 = softmax(s * qk0 qk1^T) v1 ; m1 = softmax(s * qk1 qk0^T) v0 with s = 64^-0.5 (the reference scales each
  // operand by 64^-0.25, lightglue.py:216-221); both directions of every pair in one launch
  FlashJob fj[LG_MAX_SIDES];
  for (int i = 0; i < act.n; ++i) {
    LgSide &a = s->side[act.side[i]], &b = s->side[act.side[i] ^ 1];
    fj[i] = {&a.q, &b.q, &b.v, &a.ctx, a.n, b.n, a.cap, b.cap};
  }
  if ((rc = run_flash(ctx, st, tw, fj, act.n, 0.125f, fp16_attn))) return rc;
  return lg_ffn(ctx, st, s, act, "lg_cross", w.w0, w.b0, w.lng, w.lnb, w.w3, w.b3);
}

// Network input of the sides in `act` (kp[i], desc[i] belong to act.side[i]): x = desc and its split planes, the rotary
// table of the keypoints, ind = identity.
static int lg_load_sides(b2_context* ctx, cudaStream_t st, LightGlueState* s, const LgActive& act, const float* const* kp,
                         const float* const* desc) {
  if (act.n == 0) return B2_OK;
  JobList<LoadJob> lj{};
  JobList<PosJob> pj{};
  for (int i = 0; i < act.n; ++i) {
    LgSide& sd = s->side[act.side[i]];
    const Pl xp = planes_of(sd.xs[0], (size_t)sd.cap * 256);
    lj.j[i] = {desc[i], sd.n, sd.x[0].as<float>(), s->use_tc ? xp.hi : (__half*)nullptr, s->use_tc ? xp.lo : (__half*)nullptr};
    pj.j[i] = {kp[i], sd.n, sd.cs[0].as<float>(), sd.sn[0].as<float>(), sd.ind[0].as<int>()};
  }
  const int mx = lg_max_n(s, act);
  B2_LAUNCH(ctx, k_lg_load_desc, dim3(cdiv(mx * 64, 256), act.n), 256, 0, st, lj);
  B2_CHECK_LAUNCH(ctx);
  const int pb = cdiv(mx * 32, 1024);
  B2_LAUNCH(ctx, k_lg_posenc, dim3(pb < 16 ? pb : 16, act.n), 1024, 0, st, pj, s->wr);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// Copies the live layer-0 state (x / xs / cs / sn [0]) of the sides in `act` to the encoding blob[i] of act.side[i]
// (to_blob), or back from it, setting ind[0] to the identity.
static int lg_enc_copy(b2_context* ctx, cudaStream_t st, LightGlueState* s, const LgActive& act, void* const* blob, bool to_blob) {
  if (act.n == 0) return B2_OK;
  JobList<EncJob> ej{};
  for (int i = 0; i < act.n; ++i) {
    LgSide& sd = s->side[act.side[i]];
    const Pl xp = planes_of(sd.xs[0], (size_t)sd.cap * 256);
    ej.j[i] = {static_cast<float4*>(blob[i]), sd.n, sd.x[0].as<float>(), s->use_tc ? xp.hi : (__half*)nullptr,
               s->use_tc ? xp.lo : (__half*)nullptr, sd.cs[0].as<float>(), sd.sn[0].as<float>(), sd.ind[0].as<int>()};
  }
  const int mx = lg_max_n(s, act);
  B2_LAUNCH(ctx, k_lg_enc_copy, dim3(cdiv(mx * (int)(LG_ENC_ROW_BYTES / 16), 256), act.n), 256, 0, st, ej, to_blob ? 1 : 0);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// Appends the state of the sides in `act` after `layer` to the trace (synchronises the stream); with `heads` also their
// confidence, matchability, counters and keep maps.  p0: index of the batch's first pair in the call.
static int lg_trace_layer(b2_context* ctx, cudaStream_t st, LightGlueState* s, const LgActive& act, int layer, int p0, bool heads) {
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  const int* hc = s->hread.as<int>();
  for (int i = 0; i < act.n; ++i) {
    const int sdi = act.side[i];
    const LgSide& sd = s->side[sdi];
    LgTraceRec r;
    r.pair = p0 + (sdi >> 1), r.side = sdi & 1, r.layer = layer, r.n = sd.n, r.heads = heads ? 1 : 0;
    r.x.resize((size_t)sd.n * 256), r.ind.resize(sd.n);
    B2_CUDA(ctx, cudaMemcpy(r.x.data(), sd.x[sd.cur].p, r.x.size() * 4, cudaMemcpyDeviceToHost));
    B2_CUDA(ctx, cudaMemcpy(r.ind.data(), sd.ind[sd.cur].p, r.ind.size() * 4, cudaMemcpyDeviceToHost));
    if (heads) {
      r.unconf = hc[4 * (sdi >> 1) + r.side], r.kept = hc[4 * (sdi >> 1) + 2 + r.side];
      r.conf.resize(sd.n), r.mat.resize(sd.n), r.keep.resize(r.kept);
      B2_CUDA(ctx, cudaMemcpy(r.conf.data(), sd.conf.p, (size_t)sd.n * 4, cudaMemcpyDeviceToHost));
      B2_CUDA(ctx, cudaMemcpy(r.mat.data(), sd.mat.p, (size_t)sd.n * 4, cudaMemcpyDeviceToHost));
      B2_CUDA(ctx, cudaMemcpy(r.keep.data(), sd.src.p, (size_t)r.kept * 4, cudaMemcpyDeviceToHost));
    }
    s->trace.push_back(std::move(r));
  }
  return B2_OK;
}

// One batch of up to LG_MAX_PAIRS pairs walked in lock-step (lightglue.py:474-629 for each of them).  p0: index of its first
// pair in the call (trace records only).
static int lg_match_batch(b2_context* ctx, b2_lightglue_pair* pairs, int np, const b2_lightglue_params* prm, cudaStream_t st, int p0) {
  LightGlueState* s = ctx->lg;
  int rc;
  for (int p = 0; p < np; ++p) {
    b2_lightglue_pair& pr = pairs[p];
    pr.out_k = 0, pr.out_stop_layer = 1;
    LgPair& lp = s->pair[p];
    lp.n0 = pr.n0, lp.n1 = pr.n1, lp.stop = 0, lp.out_matches = (long long*)pr.out_matches, lp.out_scores = pr.out_scores;
    lp.active = pr.n0 > 0 && pr.n1 > 0;  // lightglue.py:568-588 (no keypoints -> empty matches)
    if (!lp.active) {
      s->side[2 * p].n = s->side[2 * p + 1].n = 0;
      continue;
    }
    if ((rc = lg_side_alloc(ctx, s->side[2 * p], pr.n0, s->use_tc))) return rc;
    if ((rc = lg_side_alloc(ctx, s->side[2 * p + 1], pr.n1, s->use_tc))) return rc;
  }
  LgActive act = lg_active_sides(s, np);
  if (act.n == 0) return B2_OK;
  LgActive fresh, encoded;  // sides handed in as features / as encodings (which have been through layer 0's self block)
  const float *kp[LG_MAX_SIDES], *desc[LG_MAX_SIDES];
  void* blob[LG_MAX_SIDES];
  for (int i = 0; i < act.n; ++i) {
    const int sdi = act.side[i];
    const b2_lightglue_pair& pr = pairs[sdi >> 1];
    const void* enc = (sdi & 1) ? pr.enc1 : pr.enc0;
    if (enc) {
      blob[encoded.n] = const_cast<void*>(enc);
      encoded.side[encoded.n++] = sdi;
    } else {
      kp[fresh.n] = (sdi & 1) ? pr.kp1 : pr.kp0, desc[fresh.n] = (sdi & 1) ? pr.desc1 : pr.desc0;
      fresh.side[fresh.n++] = sdi;
    }
  }
  if ((rc = lg_load_sides(ctx, st, s, fresh, kp, desc))) return rc;
  if ((rc = lg_enc_copy(ctx, st, s, encoded, blob, false))) return rc;
  const bool do_stop = prm->depth_confidence > 0.0, do_prune = prm->width_confidence > 0.0;
  const float keep_thr = (float)(1.0 - prm->width_confidence);  // scores > float32(1 - width_confidence)
  int* counters = s->counters.as<int>();
  int* hread = s->hread.as<int>();
  for (int layer = 0; layer < LG_LAYERS && act.n > 0; ++layer) {
    const bool fp16_attn = prm->fp16_attention != 0 && s->use_tc;
    if ((rc = lg_self_layer(ctx, st, s, layer == 0 ? fresh : act, layer, fp16_attn))) return rc;
    if ((rc = lg_cross_block(ctx, st, s, act, layer, fp16_attn))) return rc;
    for (int p = 0; p < np; ++p)
      if (s->pair[p].active) s->pair[p].stop = layer;
    if (layer == LG_LAYERS - 1 || (!do_stop && !do_prune)) {
      if (ctx->lg_trace && (rc = lg_trace_layer(ctx, st, s, act, layer, p0, false))) return rc;
      if (layer == LG_LAYERS - 1) break;
      continue;
    }
    bool prune_side[LG_MAX_SIDES];
    JobList<HeadJob> hj{};
    JobList<PruneJob> pj{};
    for (int i = 0; i < act.n; ++i) {
      const int sdi = act.side[i];
      LgSide& sd = s->side[sdi];
      prune_side[i] = do_prune && sd.n > prm->prune_min_kpts;
      hj.j[i] = {sd.x[sd.cur].as<float>(), sd.n, prune_side[i] ? s->aw[layer].wm : nullptr, prune_side[i] ? s->aw[layer].bm : nullptr,
                 sd.conf.as<float>(), sd.mat.as<float>(), nullptr};
      pj.j[i] = {sd.conf.as<float>(), sd.mat.as<float>(), sd.n, sd.src.as<int>(), counters + 4 * (sdi >> 1), sdi & 1};
    }
    const int mxn = lg_max_n(s, act);
    B2_LAUNCH(ctx, k_lg_rowheads, dim3(cdiv(mxn, 8), act.n), 256, 0, st, hj, do_stop ? s->tw[layer].w : nullptr,
              do_stop ? s->tw[layer].b : nullptr);
    B2_CHECK_LAUNCH(ctx);
    for (int i = 0; i < act.n; ++i) {
      LgSide& sd = s->side[act.side[i]];
      if (!do_stop) B2_CUDA(ctx, cudaMemsetAsync(sd.conf.p, 0, (size_t)sd.n * 4, st));  // confidences None -> never "<= thr"
      if (!prune_side[i]) B2_CUDA(ctx, cudaMemsetAsync(sd.mat.p, 0x7f, (size_t)sd.n * 4, st));  // huge positive: keep all
    }
    B2_LAUNCH(ctx, k_lg_prune_plan, dim3(1, act.n), 1024, 0, st, pj, do_stop ? s->thr[layer] : -1.0f, keep_thr);
    B2_CHECK_LAUNCH(ctx);
    B2_CUDA(ctx, cudaMemcpyAsync(hread, counters, 4 * LG_MAX_PAIRS * sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    const size_t trace0 = s->trace.size();
    if (ctx->lg_trace && (rc = lg_trace_layer(ctx, st, s, act, layer, p0, true))) return rc;
    JobList<GatherJob> gj{};
    int ng = 0, gmax = 0;
    for (int p = 0; p < np; ++p) {
      LgPair& lp = s->pair[p];
      if (!lp.active) continue;
      const int* hc = hread + 4 * p;
      if (do_stop) {
        // check_if_stop (lightglue.py:645-656) in float32: 1 - (#unconfident / (m + n)) > depth_confidence
        const float ratio = 1.0f - (float)(hc[0] + hc[1]) / (float)(lp.n0 + lp.n1);
        if (ratio > (float)prm->depth_confidence) {
          lp.active = false;
          for (size_t t = trace0; t < s->trace.size(); ++t) s->trace[t].stop |= s->trace[t].pair == p0 + p;
          continue;
        }
      }
      for (int side = 0; side < 2; ++side) {
        LgSide& sd = s->side[2 * p + side];
        const bool pruned = do_prune && sd.n > prm->prune_min_kpts;
        if (!pruned || hc[2 + side] == sd.n) continue;  // nothing pruned: the buffers stay as they are
        const int nxt = sd.cur ^ 1;
        gj.j[ng++] = {sd.src.as<int>(), counters + 4 * p + 2 + side, sd.n, sd.x[sd.cur].as<float>(), sd.cs[sd.cur].as<float>(),
                      sd.sn[sd.cur].as<float>(), sd.ind[sd.cur].as<int>(), sd.x[nxt].as<float>(), sd.cs[nxt].as<float>(), sd.sn[nxt].as<float>(),
                      sd.ind[nxt].as<int>(), s->use_tc ? sd.xs[sd.cur].as<__half>() : (const __half*)nullptr, (size_t)sd.cap * 256,
                      sd.xs[nxt].as<__half>(), (size_t)sd.cap * 256};
        gmax = sd.n > gmax ? sd.n : gmax;
        sd.cur = nxt;
        sd.n = hc[2 + side];
      }
      if (s->side[2 * p].n == 0 || s->side[2 * p + 1].n == 0) {  // everything pruned away: no matches
        lp.active = false;
        lp.stop = layer + 1;  // the reference's loop stops at the top of the next layer (lightglue.py:580-592: stop = i + 1)
      }
    }
    if (ng > 0) {
      B2_LAUNCH(ctx, k_lg_gather, dim3(cdiv(gmax, 8), ng), 256, 0, st, gj);
      B2_CHECK_LAUNCH(ctx);
    }
    act = lg_active_sides(s, np);
  }
  // ---- MatchAssignment (lightglue.py:280-296) of every pair at its stopping layer -------------------------------------
  const TcWeights tw = lg_tw(s);
  int live[LG_MAX_PAIRS], nlive = 0;
  for (int p = 0; p < np; ++p) {
    pairs[p].out_stop_layer = s->pair[p].stop + 1;
    if (s->pair[p].n0 > 0 && s->pair[p].n1 > 0 && s->side[2 * p].n > 0 && s->side[2 * p + 1].n > 0) live[nlive++] = p;
  }
  if (nlive == 0) return B2_OK;
  for (int layer = 0; layer < LG_LAYERS; ++layer) {  // final_proj + matchability logits, grouped by stopping layer
    LinArgs g[LG_MAX_SIDES];
    JobList<HeadJob> hj{};
    int ns = 0, mx = 0;
    for (int li = 0; li < nlive; ++li) {
      if (s->pair[live[li]].stop != layer) continue;
      for (int side = 0; side < 2; ++side) {
        LgSide& sd = s->side[2 * live[li] + side];
        const float* x = sd.x[sd.cur].as<float>();
        LinArgs& a = g[ns];
        a.a1f = x, a.a1p = planes_of(sd.xs[sd.cur], (size_t)sd.cap * 256), a.lda1 = 256, a.K1 = 256, a.w = s->aw[layer].wf, a.ldb = 256;
        a.bias = s->aw[layer].bf, a.scale = 0.25f;  // / 256 ** 0.25
        a.cf = sd.md.as<float>(), a.ldc = 256, a.cp = planes_of(sd.md, (size_t)sd.cap * 256), a.ldch = 256, a.M = sd.n, a.N = 256;
        hj.j[ns] = {x, sd.n, s->aw[layer].wm, s->aw[layer].bm, nullptr, nullptr, sd.ls.as<float>()};
        mx = sd.n > mx ? sd.n : mx;
        ++ns;
      }
    }
    if (ns == 0) continue;
    if ((rc = run_linear(ctx, st, tw, g, ns, "lg_assign_proj"))) return rc;
    B2_LAUNCH(ctx, k_lg_rowheads, dim3(cdiv(mx, 8), ns), 256, 0, st, hj, (const float*)nullptr, (const float*)nullptr);
    B2_CHECK_LAUNCH(ctx);
  }
  {  // sim = m0 m1^T of every pair: one launch, per-problem B operands
    LinArgs gs[LG_MAX_PAIRS];
    for (int li = 0; li < nlive; ++li) {
      const int p = live[li];
      LgSide &a = s->side[2 * p], &b = s->side[2 * p + 1];
      B2_CUDA(ctx, s->sim[p].ensure((size_t)a.n * b.n * 4));
      LinArgs& g = gs[li];
      g.a1f = a.md.as<float>(), g.a1p = planes_of(a.md, (size_t)a.cap * 256), g.lda1 = 256, g.K1 = 256;
      g.bf = b.md.as<float>(), g.bp = planes_of(b.md, (size_t)b.cap * 256), g.ldb = 256;
      g.cf = s->sim[p].as<float>(), g.ldc = b.n, g.tc_want_f32 = true, g.M = a.n, g.N = b.n;
    }
    if ((rc = run_linear(ctx, st, tw, gs, nlive, "lg_assign_sim"))) return rc;
  }
  for (int li = 0; li < nlive; ++li) {
    const int p = live[li];
    LgSide &a = s->side[2 * p], &b = s->side[2 * p + 1];
    const LgAssign la{s->sim[p].as<float>(), a.n, b.n, a.ls.as<float>(), b.ls.as<float>(), a.ind[a.cur].as<int>(), b.ind[b.cur].as<int>(),
                      (float)prm->filter_threshold, {a.rmax.as<float>(), a.rlog.as<float>(), a.lsg.as<float>()},
                      {b.rmax.as<float>(), b.rlog.as<float>(), b.lsg.as<float>()}, a.amax.as<float>(), a.aidx.as<int>(), b.aidx.as<int>(),
                      &s->as_part, &s->as_bar, s->errflag.as<int>(), s->pair[p].out_matches, s->pair[p].out_scores,
                      counters + 4 * LG_MAX_PAIRS + p};
    if ((rc = lg_assign(ctx, st, la, 0, s->persist_ctas, nullptr))) return rc;
  }
  B2_CUDA(ctx, cudaMemcpyAsync(hread + 4 * LG_MAX_PAIRS, counters + 4 * LG_MAX_PAIRS, LG_MAX_PAIRS * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(hread + 5 * LG_MAX_PAIRS, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (s->use_tc && hread[5 * LG_MAX_PAIRS]) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  for (int li = 0; li < nlive; ++li) pairs[live[li]].out_k = hread[4 * LG_MAX_PAIRS + live[li]];
  ctx->debug["lg_desc0"] = {s->side[0].x[s->side[0].cur].as<float>(), (int64_t)s->side[0].n * 256};
  ctx->debug["lg_desc1"] = {s->side[1].x[s->side[1].cur].as<float>(), (int64_t)s->side[1].n * 256};
  return B2_OK;
}

static int lg_match_pairs(b2_context* ctx, b2_lightglue_pair* pairs, int n_pairs, const b2_lightglue_params* prm, cudaStream_t st) {
  LightGlueState* s = ctx->lg;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "lightglue weights not set");
  s->persist_ctas = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  s->trace.clear();
  const int bmax = ctx->lg_batch > 0 && ctx->lg_batch < LG_MAX_PAIRS ? ctx->lg_batch : LG_MAX_PAIRS;
  for (int p0 = 0; p0 < n_pairs; p0 += bmax) {
    const int np = n_pairs - p0 < bmax ? n_pairs - p0 : bmax;
    int rc = lg_match_batch(ctx, pairs + p0, np, prm, st, p0);
    if (rc) return rc;
  }
  return B2_OK;
}

extern "C" int b2_lightglue_match_batched_dev(b2_context* ctx, b2_lightglue_pair* pairs, int n_pairs, const b2_lightglue_params* params,
                                              void* stream) {
  if (!ctx || !params || n_pairs < 0 || (n_pairs > 0 && !pairs)) return B2_ERR_ARG;
  for (int p = 0; p < n_pairs; ++p) {
    const b2_lightglue_pair& pr = pairs[p];
    if (pr.n0 < 0 || pr.n1 < 0) return B2_ERR_ARG;
    if (pr.n0 > 0 && pr.n1 > 0 && (!pr.kp0 || !pr.desc0 || !pr.kp1 || !pr.desc1 || !pr.out_matches)) return B2_ERR_ARG;
    if (((uintptr_t)pr.enc0 | (uintptr_t)pr.enc1) & 15) return B2_ERR_ARG;  // the blob is copied 16 bytes at a time
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return lg_match_pairs(ctx, pairs, n_pairs, params, (cudaStream_t)stream);
}

extern "C" size_t b2_lightglue_encoded_bytes(int n) { return n > 0 ? (size_t)n * LG_ENC_ROW_BYTES : 0; }

extern "C" int b2_lightglue_encode_batched_dev(b2_context* ctx, const b2_lightglue_image* imgs, int n_imgs, const b2_lightglue_params* params,
                                               void* stream) {
  if (!ctx || !params || n_imgs < 0 || (n_imgs > 0 && !imgs)) return B2_ERR_ARG;
  for (int i = 0; i < n_imgs; ++i) {
    const b2_lightglue_image& im = imgs[i];
    if (im.n < 0 || (im.n > 0 && (!im.kp || !im.desc || !im.out || ((uintptr_t)im.out & 15)))) return B2_ERR_ARG;
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LightGlueState* s = ctx->lg;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "lightglue weights not set");
  s->persist_ctas = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  const cudaStream_t st = (cudaStream_t)stream;
  const bool fp16_attn = params->fp16_attention != 0 && s->use_tc;
  int rc;
  // the images go through layer 0's self block LG_MAX_SIDES at a time on the side workspaces, as the sides of a batch do
  for (int i = 0; i < n_imgs;) {
    LgActive act;
    const float *kp[LG_MAX_SIDES], *desc[LG_MAX_SIDES];
    void* out[LG_MAX_SIDES];
    for (; i < n_imgs && act.n < LG_MAX_SIDES; ++i) {
      const b2_lightglue_image& im = imgs[i];
      if (im.n == 0) continue;
      if ((rc = lg_side_alloc(ctx, s->side[act.n], im.n, s->use_tc))) return rc;
      kp[act.n] = im.kp, desc[act.n] = im.desc, out[act.n] = im.out;
      act.side[act.n] = act.n;
      ++act.n;
    }
    if ((rc = lg_load_sides(ctx, st, s, act, kp, desc))) return rc;
    if ((rc = lg_self_layer(ctx, st, s, act, 0, fp16_attn))) return rc;
    if ((rc = lg_enc_copy(ctx, st, s, act, out, true))) return rc;
  }
  return B2_OK;
}

extern "C" int b2_lightglue_match_dev(b2_context* ctx, const float* kp0, const float* desc0, int n0, const float* kp1,
                                      const float* desc1, int n1, const b2_lightglue_params* params, int64_t* out_matches,
                                      float* out_scores, int* out_k, int* out_stop_layer, void* stream) {
  if (!ctx || !params || !out_k || !out_stop_layer || n0 < 0 || n1 < 0) return B2_ERR_ARG;
  if (n0 > 0 && n1 > 0 && (!kp0 || !desc0 || !kp1 || !desc1 || !out_matches)) return B2_ERR_ARG;
  b2_lightglue_pair pr{kp0, desc0, n0, kp1, desc1, n1, out_matches, out_scores, 0, 1};
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  int rc = lg_match_pairs(ctx, &pr, 1, params, (cudaStream_t)stream);
  *out_k = pr.out_k, *out_stop_layer = pr.out_stop_layer;
  return rc;
}


// Content hash of a host feature array: EVERY byte takes part (four interleaved 64-bit multiply-xorshift lanes over 8-byte
// words, then the tail), so an in-place edit anywhere in the array changes the signature.  ~10 GB/s on one host core.
static uint64_t b2_feat_signature(const void* host, size_t bytes) {
  const unsigned char* p = static_cast<const unsigned char*>(host);
  const uint64_t K0 = 0x9E3779B97F4A7C15ull, K1 = 0xC2B2AE3D27D4EB4Full;
  uint64_t h[4] = {K0 ^ bytes, K1 + bytes, K0 * 3 + bytes, K1 * 5 ^ bytes};
  size_t i = 0;
  for (; i + 32 <= bytes; i += 32) {
    uint64_t w[4];
    memcpy(w, p + i, 32);
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      h[l] = (h[l] ^ w[l]) * K0;
      h[l] ^= h[l] >> 29;
    }
  }
  uint64_t tail = 0;
  for (int sh = 0; i < bytes; ++i, sh += 8) {
    tail ^= (uint64_t)p[i] << (sh & 63);
    if ((sh & 63) == 56) h[0] = (h[0] ^ tail) * K1, h[0] ^= h[0] >> 31, tail = 0;
  }
  h[1] = (h[1] ^ tail) * K1;
  uint64_t r = h[0];
  for (int l = 1; l < 4; ++l) r = (r ^ (h[l] + K0 + (r << 6) + (r >> 2))) * K1, r ^= r >> 32;
  return r;
}
// Device address of a host array: from the cache when the same (pointer, size, signature) was uploaded before, else
// copied (into an LRU cache slot, or into `fallback` when the cache is off).
static int b2_upload_cached(b2_context* ctx, const void* host, size_t bytes, DevBuf* fallback, cudaStream_t st, const void** dev) {
  if (ctx->fcache_on < 0) {  // OFF unless asked for: b2_set_option("feature_cache", 1) or B2_FEATURE_CACHE=1
    const char* e = getenv("B2_FEATURE_CACHE");
    ctx->fcache_on = (e && e[0] == '1') ? 1 : 0;
  }
  if (!ctx->fcache_on || bytes < 4) {
    B2_CUDA(ctx, fallback->ensure(bytes));
    B2_CUDA(ctx, cudaMemcpyAsync(fallback->p, host, bytes, cudaMemcpyHostToDevice, st));
    ctx->h2d_bytes += bytes;
    *dev = fallback->p;
    return B2_OK;
  }
  const uint64_t sig = b2_feat_signature(host, bytes);
  FeatCacheEntry* lru = &ctx->fcache[0];
  for (FeatCacheEntry& e : ctx->fcache) {
    if (e.host == host && e.bytes == bytes && e.sig == sig) {
      e.stamp = ++ctx->fstamp;
      *dev = e.buf.p;
      return B2_OK;
    }
    if (e.stamp < lru->stamp) lru = &e;
  }
  B2_CUDA(ctx, lru->buf.ensure(bytes));  // (cudaFree inside ensure synchronises: no kernel still reads the old block)
  B2_CUDA(ctx, cudaMemcpyAsync(lru->buf.p, host, bytes, cudaMemcpyHostToDevice, st));
  ctx->h2d_bytes += bytes;
  lru->host = host, lru->bytes = bytes, lru->sig = sig, lru->stamp = ++ctx->fstamp;
  *dev = lru->buf.p;
  return B2_OK;
}

extern "C" int b2_lightglue_match_host(b2_context* ctx, const float* kp0, const float* desc0, int n0, const float* kp1,
                                       const float* desc1, int n1, const b2_lightglue_params* params,
                                       int64_t* out_matches, float* out_scores, int* out_k, int* out_stop_layer) {
  if (!ctx || !params || !out_k || !out_stop_layer || n0 < 0 || n1 < 0) return B2_ERR_ARG;
  *out_k = 0;
  *out_stop_layer = 1;
  if (n0 == 0 || n1 == 0) return B2_OK;
  if (!kp0 || !desc0 || !kp1 || !desc1 || !out_matches) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int mk = n0 < n1 ? n0 : n1;
  B2_CUDA(ctx, ctx->stage_d[5].ensure((size_t)mk * 2 * 8));
  B2_CUDA(ctx, ctx->stage_d[6].ensure((size_t)mk * 4));
  const float* dkp[2];
  const float* ddesc[2];
  {
    const float* hk[2] = {kp0, kp1};
    const float* hd[2] = {desc0, desc1};
    const int nn[2] = {n0, n1};
    for (int i = 0; i < 2; ++i) {
      const void *a = nullptr, *b = nullptr;
      int rc2;
      if ((rc2 = b2_upload_cached(ctx, hk[i], (size_t)nn[i] * 2 * 4, &ctx->stage_d[2 * i], st, &a))) return rc2;
      if ((rc2 = b2_upload_cached(ctx, hd[i], (size_t)nn[i] * 256 * 4, &ctx->stage_d[2 * i + 1], st, &b))) return rc2;
      dkp[i] = static_cast<const float*>(a), ddesc[i] = static_cast<const float*>(b);
    }
  }
  b2_lightglue_pair pr{dkp[0], ddesc[0], n0, dkp[1], ddesc[1], n1, ctx->stage_d[5].as<int64_t>(), ctx->stage_d[6].as<float>(), 0, 1};
  int rc = lg_match_pairs(ctx, &pr, 1, params, st);
  *out_k = pr.out_k, *out_stop_layer = pr.out_stop_layer;
  if (rc) return rc;
  if (*out_k > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(out_matches, ctx->stage_d[5].p, (size_t)*out_k * 2 * 8, cudaMemcpyDeviceToHost, st));
    if (out_scores) B2_CUDA(ctx, cudaMemcpyAsync(out_scores, ctx->stage_d[6].p, (size_t)*out_k * 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return B2_OK;
}

// ---- test-only entry point: the assignment step on its own, on a host similarity matrix --------------------------------------

extern "C" int b2_debug_lightglue_assign_host(b2_context* ctx, int path, int ctas, const float* sim, int M, int N, const float* z0,
                                              const float* z1, const int* ind0, const int* ind1, float threshold, float* row_stats,
                                              float* col_stats, float* best0, int* arg0, int* arg1, int64_t* out_matches,
                                              float* out_scores, int* out_k, int* out_path) {
  if (!ctx || !sim || !z0 || !z1 || !row_stats || !col_stats || !best0 || !arg0 || !arg1 || !out_matches || !out_scores || !out_k ||
      !out_path || M <= 0 || N <= 0 || path < 0 || path > 2 || ctas < 0 || ctas > ctx->sm_count)
    return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  DevBuf dsim, dz0, dz1, di0, di1, rs, cs, dbest, da0, da1, part, bar, err, out, outs, cnt;
  B2_CUDA(ctx, dsim.ensure((size_t)M * N * 4));
  B2_CUDA(ctx, dz0.ensure((size_t)M * 4));
  B2_CUDA(ctx, dz1.ensure((size_t)N * 4));
  B2_CUDA(ctx, di0.ensure((size_t)M * 4));
  B2_CUDA(ctx, di1.ensure((size_t)N * 4));
  B2_CUDA(ctx, rs.ensure((size_t)3 * M * 4));
  B2_CUDA(ctx, cs.ensure((size_t)3 * N * 4));
  B2_CUDA(ctx, dbest.ensure((size_t)M * 4));
  B2_CUDA(ctx, da0.ensure((size_t)M * 4));
  B2_CUDA(ctx, da1.ensure((size_t)N * 4));
  B2_CUDA(ctx, err.ensure(16));
  B2_CUDA(ctx, out.ensure((size_t)M * 16));
  B2_CUDA(ctx, outs.ensure((size_t)M * 4));
  B2_CUDA(ctx, cnt.ensure(16));
  std::vector<int> iota((size_t)(M > N ? M : N));
  for (size_t i = 0; i < iota.size(); ++i) iota[i] = (int)i;
  B2_CUDA(ctx, cudaMemcpyAsync(dsim.p, sim, (size_t)M * N * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dz0.p, z0, (size_t)M * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dz1.p, z1, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(di0.p, ind0 ? ind0 : iota.data(), (size_t)M * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(di1.p, ind1 ? ind1 : iota.data(), (size_t)N * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(err.p, 0, 16, st));
  const int G = ctas > 0 ? ctas : (ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1);
  float *r = rs.as<float>(), *c = cs.as<float>();
  const LgAssign p{dsim.as<float>(), M, N, dz0.as<float>(), dz1.as<float>(), di0.as<int>(), di1.as<int>(), threshold, {r, r + M, r + 2 * M},
                   {c, c + N, c + 2 * N}, dbest.as<float>(), da0.as<int>(), da1.as<int>(), &part, &bar, err.as<int>(),
                   out.as<long long>(), outs.as<float>(), cnt.as<int>()};
  const int rc = lg_assign(ctx, st, p, path, G, out_path);
  if (rc) return rc;
  int k = 0, e = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&k, cnt.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&e, err.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(row_stats, rs.p, (size_t)3 * M * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(col_stats, cs.p, (size_t)3 * N * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(best0, dbest.p, (size_t)M * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(arg0, da0.p, (size_t)M * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(arg1, da1.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (k > 0) {
    B2_CUDA(ctx, cudaMemcpy(out_matches, out.p, (size_t)k * 16, cudaMemcpyDeviceToHost));
    B2_CUDA(ctx, cudaMemcpy(out_scores, outs.p, (size_t)k * 4, cudaMemcpyDeviceToHost));
  }
  *out_k = k;
  if (e) return b2_fail(ctx, B2_ERR_STATE, "the persistent assignment kernel timed out in its grid barrier (kernel bug)");
  return B2_OK;
}

// ---- the per-layer trace (b2_set_option "lightglue_trace") ------------------------------------------------------------------

extern "C" int b2_lightglue_trace_count(b2_context* ctx) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return ctx->lg ? (int)ctx->lg->trace.size() : 0;
}

extern "C" int b2_lightglue_trace_get(b2_context* ctx, int i, int* meta, float* x, int* ind, float* conf, float* mat, int* keep) {
  if (!ctx || !meta) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->lg || i < 0 || i >= (int)ctx->lg->trace.size()) return b2_fail(ctx, B2_ERR_ARG, "no such lightglue trace record");
  const LgTraceRec& r = ctx->lg->trace[i];
  const int m[8] = {r.pair, r.side, r.layer, r.n, r.heads, r.unconf, r.kept, r.stop};
  memcpy(meta, m, sizeof(m));
  if (x) memcpy(x, r.x.data(), r.x.size() * 4);
  if (ind) memcpy(ind, r.ind.data(), r.ind.size() * 4);
  if (conf) memcpy(conf, r.conf.data(), r.conf.size() * 4);
  if (mat) memcpy(mat, r.mat.data(), r.mat.size() * 4);
  if (keep) memcpy(keep, r.keep.data(), r.keep.size() * 4);
  return B2_OK;
}

// ---- test-only entry points: one LightGlue kernel on host arrays, launched as lg_match_batch launches it ------------------
// Entry i of a batched launch has n[i] rows (0 allowed); its arrays are concatenated over i on the host and live in buffers
// of their own on the device, each output followed by a 0xFF guard that the kernel must leave alone.

constexpr size_t LG_DBG_GUARD = 4096;

struct LgDbg {
  b2_context* ctx;
  cudaStream_t st;
  std::vector<std::unique_ptr<DevBuf>> bufs;
  struct Out {
    void* host;
    size_t bytes;
    const DevBuf* d;
  };
  std::vector<Out> outs;
  // host -> device; an output (out = true) is copied in too, so what the kernel does not write comes back as it went in
  template <typename T>
  int put(const T* host, size_t n, bool out, T** dev) {
    *dev = nullptr;
    if (!host) return B2_OK;
    bufs.emplace_back(new DevBuf());
    DevBuf& d = *bufs.back();
    int rc;
    if ((rc = dbg_upload(ctx, st, host, n * sizeof(T), out ? LG_DBG_GUARD : 0, d))) return rc;
    if (out) outs.push_back({const_cast<T*>(host), n * sizeof(T), &d});
    *dev = d.as<T>();
    return B2_OK;
  }
  int finish(const char* what) {
    bool guard_ok = true;
    int rc;
    for (const Out& o : outs)
      if ((rc = dbg_download(ctx, st, o.host, o.bytes, LG_DBG_GUARD, *o.d, guard_ok))) return rc;
    if (!guard_ok) return b2_fail(ctx, B2_ERR_STATE, std::string(what) + ": the kernel wrote past the end of an output");
    return B2_OK;
  }
};

static int lg_dbg_sizes(const int* n, int np, int* mx) {
  if (!n || np <= 0 || np > LG_MAX_SIDES) return B2_ERR_ARG;
  *mx = 0;
  for (int i = 0; i < np; ++i) {
    if (n[i] < 0) return B2_ERR_ARG;
    *mx = n[i] > *mx ? n[i] : *mx;
  }
  return B2_OK;
}

extern "C" int b2_debug_lightglue_posenc_host(b2_context* ctx, int np, const int* n, const float* kp, const float* wr, float* cs,
                                              float* sn, int* ind) {
  int mx, rc;
  if (!ctx || !kp || !wr || !cs || !sn || !ind || lg_dbg_sizes(n, np, &mx)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  JobList<PosJob> pj{};
  float* dwr;
  if ((rc = d.put(wr, 64, false, &dwr))) return rc;
  for (int i = 0, o = 0; i < np; o += n[i++]) {
    PosJob& j = pj.j[i];
    j.n = n[i];
    float* k;
    if ((rc = d.put(kp + 2 * o, 2 * (size_t)n[i], false, &k)) || (rc = d.put(cs + 32 * (size_t)o, 32 * (size_t)n[i], true, &j.cs)) ||
        (rc = d.put(sn + 32 * (size_t)o, 32 * (size_t)n[i], true, &j.sn)) || (rc = d.put(ind + o, (size_t)n[i], true, &j.ind)))
      return rc;
    j.kp = k;
  }
  if (mx > 0) {
    const int pb = cdiv(mx * 32, 1024);
    B2_LAUNCH(ctx, k_lg_posenc, dim3(pb < 16 ? pb : 16, np), 1024, 0, d.st, pj, dwr);
    B2_CHECK_LAUNCH(ctx);
  }
  return d.finish("b2_debug_lightglue_posenc_host");
}

extern "C" int b2_debug_lightglue_ln_gelu_host(b2_context* ctx, int np, const int* n, const float* g, const float* b, float* h,
                                               uint16_t* hi, uint16_t* lo) {
  int mx, rc;
  if (!ctx || !g || !b || !h || !hi != !lo || lg_dbg_sizes(n, np, &mx)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  JobList<LnJob> lj{};
  float *dg, *db;
  if ((rc = d.put(g, 512, false, &dg)) || (rc = d.put(b, 512, false, &db))) return rc;
  for (int i = 0, o = 0; i < np; o += n[i++]) {
    LnJob& j = lj.j[i];
    const size_t e = 512 * (size_t)o, ne = 512 * (size_t)n[i];
    j.n = n[i];
    uint16_t *dh = nullptr, *dl = nullptr;
    if ((rc = d.put(h + e, ne, true, &j.h)) || (hi && ((rc = d.put(hi + e, ne, true, &dh)) || (rc = d.put(lo + e, ne, true, &dl)))))
      return rc;
    j.hi = reinterpret_cast<__half*>(dh), j.lo = reinterpret_cast<__half*>(dl);
  }
  if (mx > 0) {
    B2_LAUNCH(ctx, k_lg_ln_gelu, dim3(cdiv(mx, 8), np), 256, 0, d.st, lj, dg, db);
    B2_CHECK_LAUNCH(ctx);
  }
  return d.finish("b2_debug_lightglue_ln_gelu_host");
}

extern "C" int b2_debug_lightglue_rowheads_host(b2_context* ctx, int np, const int* n, const int* mode, const float* x, const float* w1,
                                                const float* b1, const float* w2, const float* b2, float* o1, float* o2, float* zraw) {
  int mx, rc;
  if (!ctx || !mode || !x || !o1 || !o2 || !zraw || !w1 != !b1 || !w2 != !b2 || lg_dbg_sizes(n, np, &mx)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  JobList<HeadJob> hj{};
  float *dw1, *db1, *dw2, *db2;
  if ((rc = d.put(w1, 256, false, &dw1)) || (rc = d.put(b1, 1, false, &db1)) || (rc = d.put(w2, 256, false, &dw2)) ||
      (rc = d.put(b2, 1, false, &db2)))
    return rc;
  for (int i = 0, o = 0; i < np; o += n[i++]) {
    HeadJob& j = hj.j[i];
    float *dx, *d1, *d2, *dz;
    if ((rc = d.put(x + 256 * (size_t)o, 256 * (size_t)n[i], false, &dx)) || (rc = d.put(o1 + o, (size_t)n[i], true, &d1)) ||
        (rc = d.put(o2 + o, (size_t)n[i], true, &d2)) || (rc = d.put(zraw + o, (size_t)n[i], true, &dz)))
      return rc;
    // mode bit 0: head 2 on for this entry; bit 1: its sigmoid is written (o2); bit 2: its raw logit is written (zraw)
    const bool h2 = (mode[i] & 1) && dw2;
    j = {dx, n[i], h2 ? dw2 : nullptr, h2 ? db2 : nullptr, d1, (mode[i] & 2) ? d2 : nullptr, (mode[i] & 4) ? dz : nullptr};
  }
  if (mx > 0) {
    B2_LAUNCH(ctx, k_lg_rowheads, dim3(cdiv(mx, 8), np), 256, 0, d.st, hj, dw1, db1);
    B2_CHECK_LAUNCH(ctx);
  }
  return d.finish("b2_debug_lightglue_rowheads_host");
}

extern "C" int b2_debug_lightglue_prune_host(b2_context* ctx, int np, const int* n, const float* conf, const float* mat, float thr,
                                             float keep_thr, int* src, int* counters) {
  int mx, rc;
  if (!ctx || !conf || !mat || !src || !counters || lg_dbg_sizes(n, np, &mx)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  JobList<PruneJob> pj{};
  int* dc;  // entries 2p and 2p + 1 are the two sides of pair p: [unconf0, unconf1, kept0, kept1]
  if ((rc = d.put(counters, 4 * (size_t)((np + 1) / 2), true, &dc))) return rc;
  for (int i = 0, o = 0; i < np; o += n[i++]) {
    PruneJob& j = pj.j[i];
    float *dcf, *dm;
    if ((rc = d.put(conf + o, (size_t)n[i], false, &dcf)) || (rc = d.put(mat + o, (size_t)n[i], false, &dm)) ||
        (rc = d.put(src + o, (size_t)n[i], true, &j.src)))
      return rc;
    j.conf = dcf, j.mat = dm, j.n = n[i], j.counters = dc + 4 * (i >> 1), j.side = i & 1;
  }
  B2_LAUNCH(ctx, k_lg_prune_plan, dim3(1, np), 1024, 0, d.st, pj, thr, keep_thr);
  B2_CHECK_LAUNCH(ctx);
  return d.finish("b2_debug_lightglue_prune_host");
}

extern "C" int b2_debug_lightglue_gather_host(b2_context* ctx, int np, const int* n, const int* cnt, const int* src, const float* x,
                                              const float* cs, const float* sn, const int* ind, const uint16_t* planes, float* x2,
                                              float* cs2, float* sn2, int* ind2, uint16_t* planes2) {
  int mx, rc;
  if (!ctx || !cnt || !src || !x || !cs || !sn || !ind || !x2 || !cs2 || !sn2 || !ind2 || !planes != !planes2 || lg_dbg_sizes(n, np, &mx))
    return B2_ERR_ARG;
  for (int i = 0, o = 0; i < np; o += n[i++]) {  // the kernel trusts the plan: cnt <= n rows, each src entry a row
    if (cnt[i] < 0 || cnt[i] > n[i]) return B2_ERR_ARG;
    for (int r = 0; r < cnt[i]; ++r)
      if (src[o + r] < 0 || src[o + r] >= n[i]) return B2_ERR_ARG;
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  JobList<GatherJob> gj{};
  int* dcnt;
  if ((rc = d.put(cnt, (size_t)np, false, &dcnt))) return rc;
  for (int i = 0, o = 0; i < np; o += n[i++]) {
    GatherJob& j = gj.j[i];
    const size_t m = (size_t)n[i];
    int *ds, *di;
    float *dx, *dcs, *dsn;
    uint16_t *dp = nullptr, *dp2 = nullptr;  // per entry: hi [n][256] then lo [n][256]
    if ((rc = d.put(src + o, m, false, &ds)) || (rc = d.put(x + 256 * (size_t)o, 256 * m, false, &dx)) ||
        (rc = d.put(cs + 32 * (size_t)o, 32 * m, false, &dcs)) || (rc = d.put(sn + 32 * (size_t)o, 32 * m, false, &dsn)) ||
        (rc = d.put(ind + o, m, false, &di)) || (rc = d.put(x2 + 256 * (size_t)o, 256 * m, true, &j.x2)) ||
        (rc = d.put(cs2 + 32 * (size_t)o, 32 * m, true, &j.cs2)) || (rc = d.put(sn2 + 32 * (size_t)o, 32 * m, true, &j.sn2)) ||
        (rc = d.put(ind2 + o, m, true, &j.ind2)) ||
        (planes && ((rc = d.put(planes + 512 * (size_t)o, 512 * m, false, &dp)) || (rc = d.put(planes2 + 512 * (size_t)o, 512 * m, true, &dp2)))))
      return rc;
    j.src = ds, j.cnt = dcnt + i, j.n = n[i], j.x = dx, j.cs = dcs, j.sn = dsn, j.ind = di;
    j.ph = reinterpret_cast<const __half*>(dp), j.pstride = 256 * m, j.ph2 = reinterpret_cast<__half*>(dp2), j.pstride2 = 256 * m;
  }
  if (mx > 0) {
    B2_LAUNCH(ctx, k_lg_gather, dim3(cdiv(mx, 8), np), 256, 0, d.st, gj);
    B2_CHECK_LAUNCH(ctx);
  }
  return d.finish("b2_debug_lightglue_gather_host");
}

extern "C" int b2_debug_lightglue_filter_host(b2_context* ctx, int m, int n, const float* best0, const int* a0, const int* a1, float th,
                                              const int* ind0, const int* ind1, int64_t* out_matches, float* out_scores, int* out_k) {
  if (!ctx || m <= 0 || n <= 0 || !best0 || !a0 || !a1 || !ind0 || !ind1 || !out_matches || !out_scores || !out_k) return B2_ERR_ARG;
  for (int i = 0; i < m; ++i)  // the kernel reads a1[a0[i]]: the arg-max kernels never hand it anything else
    if (a0[i] < 0 || a0[i] >= n) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_lightglue_filter_host: a0 entry out of range");
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  float *db, *dos;
  int *da0, *da1, *di0, *di1, *dk;
  int64_t* dom;
  int rc;
  if ((rc = d.put(best0, (size_t)m, false, &db)) || (rc = d.put(a0, (size_t)m, false, &da0)) || (rc = d.put(a1, (size_t)n, false, &da1)) ||
      (rc = d.put(ind0, (size_t)m, false, &di0)) || (rc = d.put(ind1, (size_t)n, false, &di1)) ||
      (rc = d.put(out_matches, 2 * (size_t)m, true, &dom)) || (rc = d.put(out_scores, (size_t)m, true, &dos)) ||
      (rc = d.put(out_k, 1, true, &dk)))
    return rc;
  B2_LAUNCH(ctx, k_lg_filter, 1, 1024, 0, d.st, db, da0, da1, m, th, di0, di1, reinterpret_cast<long long*>(dom), dos, dk);
  B2_CHECK_LAUNCH(ctx);
  return d.finish("b2_debug_lightglue_filter_host");
}

extern "C" int b2_debug_lightglue_argmax_host(b2_context* ctx, int path, const float* sim, int M, int N, const float* z0, const float* z1,
                                              float* best0, int* arg0, int* arg1, int* out_path) {
  if (!ctx || !sim || !z0 || !z1 || !best0 || !arg0 || !arg1 || !out_path || M <= 0 || N <= 0 || path < 0 || path > 2) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  LgDbg d{ctx, ctx->stream};
  DevBuf stats, part, bar, err;
  float *dsim, *dz0, *dz1, *db;
  int *da0, *da1;
  int rc;
  if ((rc = d.put(sim, (size_t)M * N, false, &dsim)) || (rc = d.put(z0, (size_t)M, false, &dz0)) || (rc = d.put(z1, (size_t)N, false, &dz1)) ||
      (rc = d.put(best0, (size_t)M, true, &db)) || (rc = d.put(arg0, (size_t)M, true, &da0)) || (rc = d.put(arg1, (size_t)N, true, &da1)))
    return rc;
  B2_CUDA(ctx, stats.ensure((size_t)3 * (M + N) * 4));
  B2_CUDA(ctx, err.ensure(16));
  B2_CUDA(ctx, cudaMemsetAsync(err.p, 0, 16, d.st));
  float *r = stats.as<float>(), *c = r + 3 * M;
  const LgAssign p{dsim, M, N, dz0, dz1, nullptr, nullptr, 0.f, {r, r + M, r + 2 * M}, {c, c + N, c + 2 * N}, db, da0, da1, &part, &bar,
                   err.as<int>(), nullptr, nullptr, nullptr};
  const int G = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  if ((rc = lg_assign_argmax(ctx, d.st, p, path, G, out_path))) return rc;
  if ((rc = d.finish("b2_debug_lightglue_argmax_host"))) return rc;
  int e = 0;
  B2_CUDA(ctx, cudaMemcpy(&e, err.p, 4, cudaMemcpyDeviceToHost));
  if (e) return b2_fail(ctx, B2_ERR_STATE, "the persistent assignment kernel timed out in its grid barrier (kernel bug)");
  return B2_OK;
}
