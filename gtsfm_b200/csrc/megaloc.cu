// MegaLoc global image descriptor: DINOv2 ViT-B/14 backbone + SALAD aggregation + Linear(16640 -> 8448), the retrieval front
// of megaloc_sift_frontend.yaml.  Reference: thirdparty/megaloc/megaloc.py:25-257 (MegaLocModel, SALAD, get_matching_probs,
// log_otp_solver) on DINOv2's DinoVisionTransformer (vit_base, patch 14, 12 blocks, 12 heads x 64, LayerScale), wrapped by
// gtsfm/frontend/global_descriptor/megaloc_global_descriptor.py:18-77.
//
// Per image of H x W (multiples of 14; gh = H / 14, gw = W / 14, n = gh gw patches, T = n + 1 tokens):
//   patch embed   one GEMM per image over an im2col operand [n][640] (K = 3 x 14 x 14 = 588, zero-padded for TMA rows),
//                 bias and the interpolated position table fused as the epilogue's residual; the cls row = cls + pos[0]
//   12 blocks     x += proj'(attn(LN1 x)); x += fc2'(GELU(fc1(LN2 x)))  (LayerScale folded into proj' / fc2' on upload)
//                 QKV: k_gemm_ws with the head-major epilogue, [36][T][64] per image (q heads, then k, then v);
//                 attention: k_flash_ps with 12 heads per problem writing [T][768]
//   final LN      tokens [T][768]: cls = row 0, patches = rows 1 .. n
//   SALAD         cluster_features.0 and score.0 as ONE GEMM (N = 1024, ReLU), then .3 of each; token_features on the cls rows;
//                 Sinkhorn on the 65 x n log matrix (k_ml_sinkhorn, one CTA per image); A = f p^T (k_ml_aggregate);
//                 intra-normalisation, [t | A flattened l-major] and L2 (k_ml_assemble)
//   head          Linear(16640 -> 8448) over every image of the call as ONE GEMM (M = batch; reading the 562 MB weight is
//                 the cost), K walked in chunks whose partial sums the epilogue adds in fp32, then L2.
// Arithmetic: split-fp16 x 3 on the tensor cores (gemm_ws.cuh, attn_ps.cuh), fp32 everywhere else.  There is no SIMT path:
// with force_simt set every b2_megaloc_* call fails with B2_ERR_STATE.
#include <cmath>

#include "common.cuh"
#include "linear.cuh"

constexpr int ML_D = 768, ML_HEADS = 12, ML_QKV = 3 * ML_D, ML_MLP = 3072, ML_BLOCKS = 12, ML_P = 14, ML_KP = 588, ML_KPAD = 640;
constexpr int ML_POS_G = 37;                     // the position table's grid (518 / 14)
constexpr int ML_SMLP = 512, ML_L = 256, ML_M = 64, ML_TOK = 256;
constexpr int ML_AGG = ML_TOK + ML_L * ML_M;     // 16640
constexpr int ML_OUT = 8448;
constexpr int ML_CHUNK = AP_MAXP < GW_MAXP ? AP_MAXP : GW_MAXP;  // images per pass of the backbone (one problem per image)
constexpr int ML_FC2_KC = 1024, ML_HEAD_KC = 640;  // K chunks whose partial products are summed by the fp32 epilogue
constexpr int ML_RS = 322;                       // the plugin's resize target
constexpr float ML_LN_EPS = 1e-6f;

struct MlBlockOff {
  size_t qkv, proj, fc1, fc2;               // planes
  size_t n1w, n1b, qkvb, projb, n2w, n2b, fc1b, fc2b;  // fp32
};
struct MlResizeTab {  // one axis of torch's uint8 antialiased bilinear resize: int16 weights, first tap, tap count, precision
  int in = -1, taps = 0, prec = 0;
  DevBuf w, x0;  // int16 [ML_RS][taps], int32 [ML_RS][2] (first, count)
};

struct MegaLocState {
  bool loaded = false;
  DevBuf wh, wl, small, errflag, attn_part, attn_ml, attn_cnt;
  size_t patch = 0, s0 = 0, c3 = 0, s3 = 0, t0 = 0, t2 = 0, head = 0;  // planes
  size_t cls = 0, pos = 0, patchb = 0, nw = 0, nb = 0, s0b = 0, c3b = 0, s3b = 0, t0b = 0, t2b = 0, headb = 0, dust = 0;  // fp32
  MlBlockOff blk[ML_BLOCKS];
  int pos_gh = -1, pos_gw = -1;
  DevBuf postab;
  MlResizeTab rh, rv;
  DevBuf col, x, lnp, qkv, att, hid, h1, fcl, sco, t1, tfe, vsc, pm, agg, dph, dpl, hout, imgs, rsz, rtmp;
};

void ml_destroy(b2_context* ctx) {
  if (!ctx->ml) return;
  ctx->debug.erase("megaloc_tokens");
  delete ctx->ml;
  ctx->ml = nullptr;
}

// ---- kernels ---------------------------------------------------------------------------------------------------------

// Patch-embed operand: row img * n + (py * gw + px), column c * 196 + ky * 14 + kx (the Conv2d weight's flattening), zero
// past 588.  U8: the resized uint8 [3][H][W] image, normalised here exactly as the plugin's batch transform does it
// ((u / 255 - mean) / std in fp32, IEEE division).
struct MlNorm {
  float mean[3], std[3];
};
template <bool U8>
__global__ void __launch_bounds__(256) k_ml_im2col(const void* __restrict__ images, int B, int H, int W, MlNorm nm, __half* __restrict__ oh,
                                                   __half* __restrict__ ol) {
  const int gw = W / ML_P, n = (H / ML_P) * gw;
  const size_t total = (size_t)B * n * (ML_KPAD / 2);
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = (int)(i % (ML_KPAD / 2)) * 2;
  const size_t row = i / (ML_KPAD / 2);
  const int img = (int)(row / n), p = (int)(row % n), py = p / gw, px = p % gw;
  float v[2] = {0.f, 0.f};
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int kk = k + e;
    if (kk >= ML_KP) break;
    const int c = kk / 196, r = kk % 196, y = py * ML_P + r / ML_P, x = px * ML_P + r % ML_P;
    const size_t off = (((size_t)img * 3 + c) * H + y) * W + x;
    if (U8) v[e] = __fdiv_rn(__fdiv_rn((float)static_cast<const uint8_t*>(images)[off], 255.0f) - nm.mean[c], nm.std[c]);
    else v[e] = static_cast<const float*>(images)[off];
  }
  uint32_t hi, lo;
  tc::split2(v[0], v[1], hi, lo);
  reinterpret_cast<uint32_t*>(oh)[i] = hi;
  reinterpret_cast<uint32_t*>(ol)[i] = lo;
}

// cls rows of the residual stream: x[img * T] = cls_token + pos_embed[0]
__global__ void k_ml_cls(const float* __restrict__ cls, const float* __restrict__ pos0, int T, float* __restrict__ x) {
  const int c = threadIdx.x + blockIdx.x * blockDim.x;
  if (c < ML_D) x[(size_t)blockIdx.y * T * ML_D + c] = cls[c] + pos0[c];
}

// Patch rows of the position table for a gh x gw grid: torch's bicubic upsample (A = -0.75, align_corners False, border taps
// clamped) of the 37 x 37 table with scale_factor ((gh + 0.1) / 37, (gw + 0.1) / 37): source = (dst + 0.5) * inv - 0.5 where inv
// = 1 / scale_factor (interpolate_pos_encoding, vision_transformer.py:180-212).  The first grid axis is the image height.
__device__ __forceinline__ void ml_cubic_coeffs(float t, float* c) {
  const float A = -0.75f;
  const float x1 = t + 1.0f, x2 = 1.0f - t, x3 = x2 + 1.0f;
  c[0] = ((A * x1 - 5.0f * A) * x1 + 8.0f * A) * x1 - 4.0f * A;
  c[1] = ((A + 2.0f) * t - (A + 3.0f)) * t * t + 1.0f;
  c[2] = ((A + 2.0f) * x2 - (A + 3.0f)) * x2 * x2 + 1.0f;
  c[3] = ((A * x3 - 5.0f * A) * x3 + 8.0f * A) * x3 - 4.0f * A;
}
__global__ void __launch_bounds__(256) k_ml_pos(const float* __restrict__ pos /*[1 + 37 * 37][768]*/, int gh, int gw, float inv_h, float inv_w,
                                                float* __restrict__ out /*[gh * gw][768]*/) {
  const int p = blockIdx.x, oy = p / gw, ox = p % gw;
  const float ry = (oy + 0.5f) * inv_h - 0.5f, rx = (ox + 0.5f) * inv_w - 0.5f;
  const float fy = floorf(ry), fx = floorf(rx);
  float cy[4], cx[4];
  ml_cubic_coeffs(ry - fy, cy);
  ml_cubic_coeffs(rx - fx, cx);
  int ys[4], xs[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    ys[i] = min(max((int)fy - 1 + i, 0), ML_POS_G - 1);
    xs[i] = min(max((int)fx - 1 + i, 0), ML_POS_G - 1);
  }
  for (int c = threadIdx.x; c < ML_D; c += blockDim.x) {
    float r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float* row = pos + (size_t)(1 + ys[i] * ML_POS_G) * ML_D + c;
      r[i] = row[(size_t)xs[0] * ML_D] * cx[0] + row[(size_t)xs[1] * ML_D] * cx[1] + row[(size_t)xs[2] * ML_D] * cx[2] + row[(size_t)xs[3] * ML_D] * cx[3];
    }
    out[(size_t)p * ML_D + c] = r[0] * cy[0] + r[1] * cy[1] + r[2] * cy[2] + r[3] * cy[3];
  }
}

// LayerNorm(768, affine) of `rows` rows: one warp per row, two-pass variance; writes fp32 (optional) and split planes
__global__ void __launch_bounds__(256) k_ml_ln(const float* __restrict__ x, int rows, const float* __restrict__ g, const float* __restrict__ b,
                                               float eps, float* __restrict__ of, __half* __restrict__ oh, __half* __restrict__ ol) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float4* row = reinterpret_cast<const float4*>(x + (size_t)r * ML_D);
  float4 v[6];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    v[i] = row[lane + 32 * i];
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float mean = warp_sum(s) / (float)ML_D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + bq * bq + c * c + d * d;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)ML_D + eps);
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    const int c0 = (lane + 32 * i) * 4;
    const float4 gg = *reinterpret_cast<const float4*>(g + c0), bb = *reinterpret_cast<const float4*>(b + c0);
    const float4 e = make_float4((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y, (v[i].z - mean) * rstd * gg.z + bb.z,
                                 (v[i].w - mean) * rstd * gg.w + bb.w);
    const size_t o = (size_t)r * ML_D + c0;
    if (of) *reinterpret_cast<float4*>(of + o) = e;
    uint32_t h0, l0, h1, l1;
    tc::split2(e.x, e.y, h0, l0);
    tc::split2(e.z, e.w, h1, l1);
    *reinterpret_cast<uint2*>(oh + o) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(ol + o) = make_uint2(l0, l1);
  }
}

// Sinkhorn of SALAD (get_matching_probs + log_otp_solver, megaloc.py:155-188) for one image per CTA: S = [score logits (64 x n);
// dust_bin row], log_a = norm (+ log(n - 64) on the dustbin row), log_b = norm, norm = -log(n + 64); 3 x (u = log_a - LSE_j(S + v),
// v = log_b - LSE_i(S + u)); P = exp(S + u + v - norm) without the dustbin row.  sc: the score GEMM's fp32 rows of the image
// (token rows, row 0 = cls skipped), [T][64]; v: scratch [n]; P out: [64][n].
__global__ void __launch_bounds__(512) k_ml_sinkhorn(const float* __restrict__ sc_all, int T, const float* __restrict__ dust_p, float norm,
                                                      float log_a_dust, float* __restrict__ v_all, float* __restrict__ P_all) {
  const int img = blockIdx.x, n = T - 1, t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const float* sc = sc_all + ((size_t)img * T + 1) * ML_M;
  float* v = v_all + (size_t)img * n;
  float* P = P_all + (size_t)img * ML_M * n;
  const float dust = *dust_p;
  __shared__ float u[ML_M + 1];
  for (int j = t; j < n; j += blockDim.x) v[j] = 0.f;
  __syncthreads();
  for (int it = 0; it < 3; ++it) {
    for (int i = warp; i <= ML_M; i += blockDim.x >> 5) {  // u_i = log_a_i - logsumexp_j (S_ij + v_j)
      float mx = -INFINITY;
      for (int j = lane; j < n; j += 32) mx = fmaxf(mx, (i < ML_M ? sc[(size_t)j * ML_M + i] : dust) + v[j]);
      mx = warp_max(mx);
      float s = 0.f;
      for (int j = lane; j < n; j += 32) s += expf((i < ML_M ? sc[(size_t)j * ML_M + i] : dust) + v[j] - mx);
      s = warp_sum(s);
      if (lane == 0) u[i] = (i < ML_M ? norm : log_a_dust) - (mx + logf(s));
    }
    __syncthreads();
    for (int j = t; j < n; j += blockDim.x) {  // v_j = log_b - logsumexp_i (S_ij + u_i)
      const float* r = sc + (size_t)j * ML_M;
      float mx = dust + u[ML_M];
      for (int i = 0; i < ML_M; ++i) mx = fmaxf(mx, r[i] + u[i]);
      float s = expf(dust + u[ML_M] - mx);
      for (int i = 0; i < ML_M; ++i) s += expf(r[i] + u[i] - mx);
      v[j] = norm - (mx + logf(s));
    }
    __syncthreads();
  }
  for (int e = t; e < ML_M * n; e += blockDim.x) {
    const int i = e / n, j = e % n;
    P[e] = expf(sc[(size_t)j * ML_M + i] + u[i] + v[j] - norm);
  }
}

// A[l][m] = sum_j f[j][l] P[m][j] for one image and 16 cluster dims l per block (the reference's repeat / multiply / sum)
__global__ void __launch_bounds__(1024) k_ml_aggregate(const float* __restrict__ f_all, int T, const float* __restrict__ P_all,
                                                       float* __restrict__ agg /*[B][256][64]*/) {
  const int img = blockIdx.y, l0 = blockIdx.x * 16, n = T - 1;
  const int m = threadIdx.x & 63, li = threadIdx.x >> 6;
  const float* f = f_all + ((size_t)img * T + 1) * ML_L;
  const float* P = P_all + (size_t)img * ML_M * n;
  __shared__ float fs[32][17];
  __shared__ float ps[ML_M][33];
  float acc = 0.f;
  for (int j0 = 0; j0 < n; j0 += 32) {
    __syncthreads();
    if (threadIdx.x < 512) {
      const int jj = threadIdx.x >> 4, ll = threadIdx.x & 15;
      fs[jj][ll] = j0 + jj < n ? f[(size_t)(j0 + jj) * ML_L + l0 + ll] : 0.f;
    }
    for (int e = threadIdx.x; e < ML_M * 32; e += 1024) {
      const int mm = e >> 5, jj = e & 31;
      ps[mm][jj] = j0 + jj < n ? P[(size_t)mm * n + j0 + jj] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int jj = 0; jj < 32; ++jj) acc = fmaf(fs[jj][li], ps[m][jj], acc);
  }
  agg[((size_t)img * ML_L + l0 + li) * ML_M + m] = acc;
}

// One image per block: [normalize(t) | normalize(A, over l) flattened l * 64 + m], then L2 over the 16640 values -> split planes
__global__ void __launch_bounds__(1024) k_ml_assemble(const float* __restrict__ tfe /*[B][256]*/, const float* __restrict__ agg, __half* __restrict__ dh,
                                                      __half* __restrict__ dl) {
  const int img = blockIdx.x, t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const float* A = agg + (size_t)img * ML_L * ML_M;
  __shared__ float cn[ML_M];
  __shared__ float red[32];
  __shared__ float tn;
  for (int m = warp; m < ML_M; m += 32) {
    float s = 0.f;
    for (int l = lane; l < ML_L; l += 32) s += A[l * ML_M + m] * A[l * ML_M + m];
    s = warp_sum(s);
    if (lane == 0) cn[m] = fmaxf(sqrtf(s), 1e-12f);
  }
  if (warp == 31) {
    float s = 0.f;
    for (int i = lane; i < ML_TOK; i += 32) s += tfe[(size_t)img * ML_TOK + i] * tfe[(size_t)img * ML_TOK + i];
    s = warp_sum(s);
    if (lane == 0) tn = fmaxf(sqrtf(s), 1e-12f);
  }
  __syncthreads();
  auto val = [&](int i) { return i < ML_TOK ? tfe[(size_t)img * ML_TOK + i] / tn : A[i - ML_TOK] / cn[(i - ML_TOK) & (ML_M - 1)]; };
  float ss = 0.f;
  for (int i = t; i < ML_AGG; i += 1024) {
    const float x = val(i);
    ss += x * x;
  }
  ss = warp_sum(ss);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) tot += red[i];
  const float nrm = fmaxf(sqrtf(tot), 1e-12f);
  for (int i = t; i < ML_AGG; i += 1024) {
    __half h, l;
    tc::split_h(val(i) / nrm, h, l);
    dh[(size_t)img * ML_AGG + i] = h, dl[(size_t)img * ML_AGG + i] = l;
  }
}

// L2 normalisation of one row of `n` floats per block
__global__ void __launch_bounds__(1024) k_ml_rownorm(const float* __restrict__ in, int n, float* __restrict__ out) {
  __shared__ float red[32];
  const float* r = in + (size_t)blockIdx.x * n;
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += 1024) ss += r[i] * r[i];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) tot += red[i];
  const float nrm = fmaxf(sqrtf(tot), 1e-12f);
  for (int i = threadIdx.x; i < n; i += 1024) out[(size_t)blockIdx.x * n + i] = r[i] / nrm;
}

// torch's uint8 antialiased bilinear resize (UpSampleKernelAVXAntialias.h: separable, horizontal pass first, int16 weights of
// `prec` fractional bits, sum + 2^(prec - 1) shifted right and clamped to 0..255 after each pass).  Horizontal: [H][W][3] pitched
// source -> [H][322][3]; vertical: [H][322][3] -> [3][322][322].  An axis that keeps its size runs the identity table (one tap of
// weight 2^prec), which returns its input exactly.
struct MlSrcList {
  const uint8_t* p[ML_CHUNK];
};
__global__ void __launch_bounds__(256) k_ml_resize_h(MlSrcList src, size_t pitch, int H, const short* __restrict__ w, const int* __restrict__ x0,
                                                     int taps, int prec, uint8_t* __restrict__ tmp) {
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (y, ox)
  if (i >= H * ML_RS) return;
  const int y = i / ML_RS, ox = i % ML_RS;
  const uint8_t* row = src.p[img] + (size_t)y * pitch;
  const int first = x0[2 * ox], cnt = x0[2 * ox + 1];
  int s0 = 1 << (prec - 1), s1 = s0, s2 = s0;
  for (int k = 0; k < cnt; ++k) {
    const int wk = w[ox * taps + k];
    const uint8_t* px = row + (size_t)(first + k) * 3;
    s0 += wk * px[0], s1 += wk * px[1], s2 += wk * px[2];
  }
  uint8_t* o = tmp + (((size_t)img * H + y) * ML_RS + ox) * 3;
  o[0] = (uint8_t)min(max(s0 >> prec, 0), 255);
  o[1] = (uint8_t)min(max(s1 >> prec, 0), 255);
  o[2] = (uint8_t)min(max(s2 >> prec, 0), 255);
}
__global__ void __launch_bounds__(256) k_ml_resize_v(const uint8_t* __restrict__ tmp, int H, const short* __restrict__ w, const int* __restrict__ y0,
                                                     int taps, int prec, uint8_t* __restrict__ out /*[B][3][322][322]*/) {
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (oy, x)
  if (i >= ML_RS * ML_RS) return;
  const int oy = i / ML_RS, x = i % ML_RS;
  const int first = y0[2 * oy], cnt = y0[2 * oy + 1];
  int s[3];
  s[0] = s[1] = s[2] = 1 << (prec - 1);
  for (int k = 0; k < cnt; ++k) {
    const int wk = w[oy * taps + k];
    const uint8_t* px = tmp + (((size_t)img * H + first + k) * ML_RS + x) * 3;
    s[0] += wk * px[0], s[1] += wk * px[1], s[2] += wk * px[2];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(((size_t)img * 3 + c) * ML_RS + oy) * ML_RS + x] = (uint8_t)min(max(s[c] >> prec, 0), 255);
}

// ---- host ------------------------------------------------------------------------------------------------------------

// torch's int16 weights of one axis (compute_index_ranges_int16_weights with the bilinear antialias filter), in double as
// there: scale = in / out, support = scale >= 1 ? scale : 1, taps [xmin, xmin + xsize), normalised weights rounded at the
// precision that keeps the largest one below 2^15.
static int ml_resize_table(b2_context* ctx, MlResizeTab& t, int in) {
  if (t.in == in) return B2_OK;
  std::vector<int> x0(2 * ML_RS);
  std::vector<double> wd;
  int taps = 1, prec = 14;
  std::vector<short> wi;
  if (in == ML_RS) {  // identity: torch skips the pass
    wi.assign(ML_RS, (short)(1 << prec));
    for (int i = 0; i < ML_RS; ++i) x0[2 * i] = i, x0[2 * i + 1] = 1;
  } else {
    const double scale = (double)in / ML_RS;
    const double support = scale >= 1.0 ? scale : 1.0;
    const double invscale = scale >= 1.0 ? 1.0 / scale : 1.0;
    taps = (int)std::ceil(support) * 2 + 1;
    wd.assign((size_t)ML_RS * taps, 0.0);
    double wmax = 0.0;
    for (int i = 0; i < ML_RS; ++i) {
      const double center = scale * (i + 0.5);
      const int64_t xmin = std::max((int64_t)(center - support + 0.5), (int64_t)0);
      int64_t xsize = std::min((int64_t)(center + support + 0.5), (int64_t)in) - xmin;
      xsize = std::min(std::max(xsize, (int64_t)0), (int64_t)taps);
      double tot = 0.0;
      double* wr = wd.data() + (size_t)i * taps;
      for (int j = 0; j < xsize; ++j) {
        const double a = std::fabs((j + xmin - center + 0.5) * invscale);
        wr[j] = a < 1.0 ? 1.0 - a : 0.0;
        tot += wr[j];
      }
      if (tot != 0.0)
        for (int j = 0; j < xsize; ++j) wr[j] /= tot, wmax = std::max(wmax, wr[j]);
      x0[2 * i] = (int)xmin, x0[2 * i + 1] = (int)xsize;
    }
    for (prec = 0; prec < 22; ++prec)
      if ((int)(0.5 + wmax * (1 << (prec + 1))) >= (1 << 15)) break;
    wi.resize(wd.size());
    for (size_t k = 0; k < wd.size(); ++k) {
      const double v = wd[k] * (1 << prec);
      wi[k] = (short)(v < 0 ? (int)(-0.5 + v) : (int)(0.5 + v));
    }
  }
  B2_CUDA(ctx, t.w.ensure(wi.size() * sizeof(short)));
  B2_CUDA(ctx, t.x0.ensure(x0.size() * sizeof(int)));
  B2_CUDA(ctx, cudaMemcpy(t.w.p, wi.data(), wi.size() * sizeof(short), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, cudaMemcpy(t.x0.p, x0.data(), x0.size() * sizeof(int), cudaMemcpyHostToDevice));
  t.in = in, t.taps = taps, t.prec = prec;
  return B2_OK;
}

// blob order (weights.MEGALOC_ORDER): cls_token [768], pos_embed [1370][768], patch_embed.proj weight [768][3][14][14] and bias;
// 12 x (norm1 w, b, qkv w [2304][768], b, proj w [768][768], b, ls1 gamma, norm2 w, b, fc1 w [3072][768], b, fc2 w [768][3072],
// b, ls2 gamma); norm w, b; cluster_features.0 w [512][768], b, .3 w [256][512], b; score.0 w [512][768], b, .3 w [64][512], b;
// token_features.0 w [512][768], b, .2 w [256][512], b; dust_bin; aggregator.linear w [8448][16640], b.
static size_t ml_blob_floats() {
  size_t n = ML_D + (size_t)(1 + ML_POS_G * ML_POS_G) * ML_D + (size_t)ML_D * ML_KP + ML_D;
  n += (size_t)ML_BLOCKS * (2 * ML_D + (size_t)ML_QKV * ML_D + ML_QKV + (size_t)ML_D * ML_D + ML_D + ML_D + 2 * ML_D + (size_t)ML_MLP * ML_D +
                            ML_MLP + (size_t)ML_D * ML_MLP + ML_D + ML_D);
  n += 2 * ML_D;
  n += (size_t)ML_SMLP * ML_D + ML_SMLP + (size_t)ML_L * ML_SMLP + ML_L;
  n += (size_t)ML_SMLP * ML_D + ML_SMLP + (size_t)ML_M * ML_SMLP + ML_M;
  n += (size_t)ML_SMLP * ML_D + ML_SMLP + (size_t)ML_TOK * ML_SMLP + ML_TOK;
  n += 1;
  n += (size_t)ML_OUT * ML_AGG + ML_OUT;
  return n;
}

extern "C" size_t b2_megaloc_blob_floats(void) { return ml_blob_floats(); }

extern "C" int b2_megaloc_set_weights(b2_context* ctx, const float* blob, size_t n_floats) {
  if (!ctx || !blob) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (b2_force_simt(ctx)) return b2_fail(ctx, B2_ERR_STATE, "megaloc runs on the wgmma path only (force_simt is set)");
  if (n_floats != ml_blob_floats())
    return b2_fail(ctx, B2_ERR_ARG, "megaloc blob must hold " + std::to_string(ml_blob_floats()) + " floats, got " + std::to_string(n_floats));
  if (!tma_encoder()) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled is not available (driver too old?)");
  cudaSetDevice(ctx->device);
  if (!ctx->ml) ctx->ml = new MegaLocState();
  MegaLocState* s = ctx->ml;
  s->loaded = false;
  s->pos_gh = s->pos_gw = -1;
  // plane arena: matrices as the GEMMs read them ([N][K] row-major)
  size_t pw = 0;
  auto take = [&](size_t n) { const size_t o = pw; pw += n; return o; };
  s->patch = take((size_t)ML_D * ML_KPAD);
  for (int l = 0; l < ML_BLOCKS; ++l) {
    s->blk[l].qkv = take((size_t)ML_QKV * ML_D), s->blk[l].proj = take((size_t)ML_D * ML_D);
    s->blk[l].fc1 = take((size_t)ML_MLP * ML_D), s->blk[l].fc2 = take((size_t)ML_D * ML_MLP);
  }
  s->s0 = take((size_t)2 * ML_SMLP * ML_D), s->c3 = take((size_t)ML_L * ML_SMLP), s->s3 = take((size_t)ML_M * ML_SMLP);
  s->t0 = take((size_t)ML_SMLP * ML_D), s->t2 = take((size_t)ML_TOK * ML_SMLP), s->head = take((size_t)ML_OUT * ML_AGG);
  // fp32 parameters
  size_t pf = 0;
  auto takef = [&](size_t n) { const size_t o = pf; pf += (n + 3) & ~(size_t)3; return o; };  // 16-byte aligned starts
  s->cls = takef(ML_D), s->pos = takef((size_t)(1 + ML_POS_G * ML_POS_G) * ML_D), s->patchb = takef(ML_D);
  for (int l = 0; l < ML_BLOCKS; ++l) {
    MlBlockOff& b = s->blk[l];
    b.n1w = takef(ML_D), b.n1b = takef(ML_D), b.qkvb = takef(ML_QKV), b.projb = takef(ML_D);
    b.n2w = takef(ML_D), b.n2b = takef(ML_D), b.fc1b = takef(ML_MLP), b.fc2b = takef(ML_D);
  }
  s->nw = takef(ML_D), s->nb = takef(ML_D), s->s0b = takef(2 * ML_SMLP), s->c3b = takef(ML_L), s->s3b = takef(ML_M);
  s->t0b = takef(ML_SMLP), s->t2b = takef(ML_TOK), s->headb = takef(ML_OUT), s->dust = takef(1);
  std::vector<float> small(pf, 0.f);

  B2_CUDA(ctx, s->wh.ensure(pw * sizeof(__half)));
  B2_CUDA(ctx, s->wl.ensure(pw * sizeof(__half)));
  DevBuf tmp;
  const size_t piece = (size_t)32 << 20;
  B2_CUDA(ctx, tmp.ensure(piece * sizeof(float)));
  auto put = [&](size_t dst, const float* host, size_t n) -> cudaError_t {  // fp32 host values -> planes at arena offset dst
    cudaError_t e;
    for (size_t o = 0; o < n; o += piece) {
      const size_t m = n - o < piece ? n - o : piece;
      if ((e = cudaMemcpy(tmp.p, host + o, m * sizeof(float), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
      k_split_f32<<<(unsigned)((m + 255) / 256), 256>>>(tmp.as<float>(), m, s->wh.as<__half>() + dst + o, s->wl.as<__half>() + dst + o);
      if ((e = cudaDeviceSynchronize()) != cudaSuccess) return e;
    }
    return cudaSuccess;
  };
  auto cpy = [&](size_t dst, const float* src, size_t n) { std::copy(src, src + n, small.begin() + dst); };
  const float* p = blob;
  cpy(s->cls, p, ML_D), p += ML_D;
  cpy(s->pos, p, (size_t)(1 + ML_POS_G * ML_POS_G) * ML_D), p += (size_t)(1 + ML_POS_G * ML_POS_G) * ML_D;
  {
    std::vector<float> w((size_t)ML_D * ML_KPAD, 0.f);
    for (int o = 0; o < ML_D; ++o) std::copy(p + (size_t)o * ML_KP, p + (size_t)(o + 1) * ML_KP, w.begin() + (size_t)o * ML_KPAD);
    B2_CUDA(ctx, put(s->patch, w.data(), w.size()));
    p += (size_t)ML_D * ML_KP;
  }
  cpy(s->patchb, p, ML_D), p += ML_D;
  std::vector<float> fold((size_t)ML_D * ML_MLP);
  for (int l = 0; l < ML_BLOCKS; ++l) {
    MlBlockOff& b = s->blk[l];
    cpy(b.n1w, p, ML_D), p += ML_D;
    cpy(b.n1b, p, ML_D), p += ML_D;
    B2_CUDA(ctx, put(b.qkv, p, (size_t)ML_QKV * ML_D));
    p += (size_t)ML_QKV * ML_D;
    cpy(b.qkvb, p, ML_QKV), p += ML_QKV;
    const float* projw = p;
    p += (size_t)ML_D * ML_D;
    const float* projb = p;
    p += ML_D;
    const float* ls1 = p;
    p += ML_D;
    for (int o = 0; o < ML_D; ++o) {  // LayerScale folded: ls * (W x + b) = (ls W) x + ls b
      for (int k = 0; k < ML_D; ++k) fold[(size_t)o * ML_D + k] = ls1[o] * projw[(size_t)o * ML_D + k];
      small[b.projb + o] = ls1[o] * projb[o];
    }
    B2_CUDA(ctx, put(b.proj, fold.data(), (size_t)ML_D * ML_D));
    cpy(b.n2w, p, ML_D), p += ML_D;
    cpy(b.n2b, p, ML_D), p += ML_D;
    B2_CUDA(ctx, put(b.fc1, p, (size_t)ML_MLP * ML_D));
    p += (size_t)ML_MLP * ML_D;
    cpy(b.fc1b, p, ML_MLP), p += ML_MLP;
    const float* fc2w = p;
    p += (size_t)ML_D * ML_MLP;
    const float* fc2b = p;
    p += ML_D;
    const float* ls2 = p;
    p += ML_D;
    for (int o = 0; o < ML_D; ++o) {
      for (int k = 0; k < ML_MLP; ++k) fold[(size_t)o * ML_MLP + k] = ls2[o] * fc2w[(size_t)o * ML_MLP + k];
      small[b.fc2b + o] = ls2[o] * fc2b[o];
    }
    B2_CUDA(ctx, put(b.fc2, fold.data(), (size_t)ML_D * ML_MLP));
  }
  cpy(s->nw, p, ML_D), p += ML_D;
  cpy(s->nb, p, ML_D), p += ML_D;
  // SALAD: cluster_features.0 and score.0 stacked into one [1024][768] weight
  B2_CUDA(ctx, put(s->s0, p, (size_t)ML_SMLP * ML_D));
    p += (size_t)ML_SMLP * ML_D;
  cpy(s->s0b, p, ML_SMLP), p += ML_SMLP;
  B2_CUDA(ctx, put(s->c3, p, (size_t)ML_L * ML_SMLP));
    p += (size_t)ML_L * ML_SMLP;
  cpy(s->c3b, p, ML_L), p += ML_L;
  B2_CUDA(ctx, put(s->s0 + (size_t)ML_SMLP * ML_D, p, (size_t)ML_SMLP * ML_D));
    p += (size_t)ML_SMLP * ML_D;
  cpy(s->s0b + ML_SMLP, p, ML_SMLP), p += ML_SMLP;
  B2_CUDA(ctx, put(s->s3, p, (size_t)ML_M * ML_SMLP));
    p += (size_t)ML_M * ML_SMLP;
  cpy(s->s3b, p, ML_M), p += ML_M;
  B2_CUDA(ctx, put(s->t0, p, (size_t)ML_SMLP * ML_D));
    p += (size_t)ML_SMLP * ML_D;
  cpy(s->t0b, p, ML_SMLP), p += ML_SMLP;
  B2_CUDA(ctx, put(s->t2, p, (size_t)ML_TOK * ML_SMLP));
    p += (size_t)ML_TOK * ML_SMLP;
  cpy(s->t2b, p, ML_TOK), p += ML_TOK;
  cpy(s->dust, p, 1), p += 1;
  B2_CUDA(ctx, put(s->head, p, (size_t)ML_OUT * ML_AGG));
    p += (size_t)ML_OUT * ML_AGG;
  cpy(s->headb, p, ML_OUT), p += ML_OUT;
  tmp.release();
  if ((size_t)(p - blob) != n_floats) return b2_fail(ctx, B2_ERR_STATE, "megaloc blob walk does not match its size (library bug)");
  B2_CUDA(ctx, s->small.ensure(pf * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->small.p, small.data(), pf * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, s->errflag.ensure(16));
  B2_CUDA(ctx, cudaMemset(s->errflag.p, 0, 16));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  s->loaded = true;
  return B2_OK;
}

static Pl ml_planes(const MegaLocState* s, size_t off) { return {s->wh.as<__half>() + off, s->wl.as<__half>() + off}; }

// The backbone and SALAD of Bc <= ML_CHUNK images whose patch-embed operand is in s->col; the flattened SALAD descriptors go to
// rows d0 .. d0 + Bc - 1 of the head's operand planes.
static int ml_chunk(b2_context* ctx, cudaStream_t st, int Bc, int gh, int gw, int d0) {
  MegaLocState* s = ctx->ml;
  const int n = gh * gw, T = n + 1, M = Bc * T;
  const float* sm = s->small.as<float>();
  TcWeights tw{nullptr, nullptr, nullptr, s->errflag.as<int>(), true};
  tw.attn_part = &s->attn_part, tw.attn_ml = &s->attn_ml, tw.attn_cnt = &s->attn_cnt;
  tw.sm_count = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  const Pl col = planes_of(s->col, (size_t)Bc * n * ML_KPAD), ln = planes_of(s->lnp, (size_t)M * ML_D);
  const Pl qkv = planes_of(s->qkv, (size_t)M * ML_QKV), att = planes_of(s->att, (size_t)M * ML_D), hid = planes_of(s->hid, (size_t)M * ML_MLP);
  const Pl h1 = planes_of(s->h1, (size_t)M * 2 * ML_SMLP), t1 = planes_of(s->t1, (size_t)Bc * ML_SMLP);
  float* x = s->x.as<float>();
  int rc;
  LinArgs la[ML_CHUNK];
  auto one = [&](const LinArgs& a) { return run_linear(ctx, st, tw, &a, 1); };
  // tokens: cls rows, then patch rows = conv bias + position table + patch embed
  B2_LAUNCH(ctx, k_ml_cls, dim3(cdiv(ML_D, 256), Bc), 256, 0, st, sm + s->cls, sm + s->pos, T, x);
  B2_CHECK_LAUNCH(ctx);
  for (int i = 0; i < Bc; ++i) {
    LinArgs& a = la[i];
    a = LinArgs{};
    a.a1p = {col.hi + (size_t)i * n * ML_KPAD, col.lo + (size_t)i * n * ML_KPAD}, a.lda1 = ML_KPAD, a.K1 = ML_KPAD;
    a.bp = ml_planes(s, s->patch), a.ldb = ML_KPAD, a.bias = sm + s->patchb;
    a.resid = s->postab.as<float>(), a.ldr = ML_D;
    a.cf = x + ((size_t)i * T + 1) * ML_D, a.ldc = ML_D, a.tc_want_f32 = true, a.M = n, a.N = ML_D;
  }
  if ((rc = run_linear(ctx, st, tw, la, Bc))) return rc;
  for (int l = 0; l < ML_BLOCKS; ++l) {
    const MlBlockOff& b = s->blk[l];
    B2_LAUNCH(ctx, k_ml_ln, cdiv(M, 8), 256, 0, st, x, M, sm + b.n1w, sm + b.n1b, ML_LN_EPS, (float*)nullptr, ln.hi, ln.lo);
    B2_CHECK_LAUNCH(ctx);
    for (int i = 0; i < Bc; ++i) {  // q, k, v head-major per image: [36][T][64]
      LinArgs& a = la[i];
      a = LinArgs{};
      a.a1p = {ln.hi + (size_t)i * T * ML_D, ln.lo + (size_t)i * T * ML_D}, a.lda1 = ML_D, a.K1 = ML_D;
      a.bp = ml_planes(s, b.qkv), a.ldb = ML_D, a.bias = sm + b.qkvb;
      a.cp = {qkv.hi + (size_t)i * T * ML_QKV, qkv.lo + (size_t)i * T * ML_QKV}, a.head_major = 1, a.lo_unscaled = 1, a.M = T, a.N = ML_QKV;
    }
    if ((rc = run_linear(ctx, st, tw, la, Bc))) return rc;
    FlashPlanes fp[ML_CHUNK];
    for (int i = 0; i < Bc; ++i) {
      const size_t q0 = (size_t)i * T * ML_QKV, hs = (size_t)ML_HEADS * T * 64;
      fp[i] = {{qkv.hi + q0, qkv.lo + q0}, {qkv.hi + q0 + hs, qkv.lo + q0 + hs}, {qkv.hi + q0 + 2 * hs, qkv.lo + q0 + 2 * hs},
               {att.hi + (size_t)i * T * ML_D, att.lo + (size_t)i * T * ML_D}, T, T, ML_HEADS, ML_D};
    }
    if ((rc = run_flash_planes(ctx, st, tw, fp, Bc, 0.125f))) return rc;
    {
      LinArgs a;
      a.a1p = att, a.lda1 = ML_D, a.K1 = ML_D, a.bp = ml_planes(s, b.proj), a.ldb = ML_D, a.bias = sm + b.projb;
      a.resid = x, a.ldr = ML_D, a.cf = x, a.ldc = ML_D, a.tc_want_f32 = true, a.M = M, a.N = ML_D;
      if ((rc = one(a))) return rc;
    }
    B2_LAUNCH(ctx, k_ml_ln, cdiv(M, 8), 256, 0, st, x, M, sm + b.n2w, sm + b.n2b, ML_LN_EPS, (float*)nullptr, ln.hi, ln.lo);
    B2_CHECK_LAUNCH(ctx);
    {
      LinArgs a;
      a.a1p = ln, a.lda1 = ML_D, a.K1 = ML_D, a.bp = ml_planes(s, b.fc1), a.ldb = ML_D, a.bias = sm + b.fc1b, a.gelu = 1;
      a.cp = hid, a.ldch = ML_MLP, a.M = M, a.N = ML_MLP;
      if ((rc = one(a))) return rc;
    }
    for (int kc = 0; kc < ML_MLP; kc += ML_FC2_KC) {
      LinArgs a;
      const Pl w = ml_planes(s, b.fc2);
      a.a1p = {hid.hi + kc, hid.lo + kc}, a.lda1 = ML_MLP, a.K1 = ML_FC2_KC, a.bp = {w.hi + kc, w.lo + kc}, a.ldb = ML_MLP;
      if (kc == 0) a.bias = sm + b.fc2b;
      a.resid = x, a.ldr = ML_D, a.cf = x, a.ldc = ML_D, a.tc_want_f32 = true, a.M = M, a.N = ML_D;
      if ((rc = one(a))) return rc;
    }
  }
  // final LayerNorm: fp32 tokens (kept for inspection) and planes
  float* tok = s->x.as<float>() + (size_t)M * ML_D;
  B2_LAUNCH(ctx, k_ml_ln, cdiv(M, 8), 256, 0, st, x, M, sm + s->nw, sm + s->nb, ML_LN_EPS, tok, ln.hi, ln.lo);
  B2_CHECK_LAUNCH(ctx);
  ctx->debug["megaloc_tokens"] = DebugView{tok, (int64_t)M * ML_D};
  // SALAD (the cls rows run through the per-token heads too; the Sinkhorn and aggregation kernels skip them)
  {
    LinArgs a;
    a.a1p = ln, a.lda1 = ML_D, a.K1 = ML_D, a.bp = ml_planes(s, s->s0), a.ldb = ML_D, a.bias = sm + s->s0b, a.relu = 1;
    a.cp = h1, a.ldch = 2 * ML_SMLP, a.M = M, a.N = 2 * ML_SMLP;
    if ((rc = one(a))) return rc;
  }
  {
    LinArgs a;
    a.a1p = h1, a.lda1 = 2 * ML_SMLP, a.K1 = ML_SMLP, a.bp = ml_planes(s, s->c3), a.ldb = ML_SMLP, a.bias = sm + s->c3b;
    a.cf = s->fcl.as<float>(), a.ldc = ML_L, a.tc_want_f32 = true, a.M = M, a.N = ML_L;
    if ((rc = one(a))) return rc;
  }
  {
    LinArgs a;
    a.a1p = {h1.hi + ML_SMLP, h1.lo + ML_SMLP}, a.lda1 = 2 * ML_SMLP, a.K1 = ML_SMLP, a.bp = ml_planes(s, s->s3), a.ldb = ML_SMLP;
    a.bias = sm + s->s3b, a.cf = s->sco.as<float>(), a.ldc = ML_M, a.tc_want_f32 = true, a.M = M, a.N = ML_M;
    if ((rc = one(a))) return rc;
  }
  {  // token_features on the cls rows (row pitch T x 768)
    LinArgs a;
    a.a1p = ln, a.lda1 = T * ML_D, a.K1 = ML_D, a.bp = ml_planes(s, s->t0), a.ldb = ML_D, a.bias = sm + s->t0b, a.relu = 1;
    a.cp = t1, a.ldch = ML_SMLP, a.M = Bc, a.N = ML_SMLP;
    if ((rc = one(a))) return rc;
    LinArgs c;
    c.a1p = t1, c.lda1 = ML_SMLP, c.K1 = ML_SMLP, c.bp = ml_planes(s, s->t2), c.ldb = ML_SMLP, c.bias = sm + s->t2b;
    c.cf = s->tfe.as<float>(), c.ldc = ML_TOK, c.tc_want_f32 = true, c.M = Bc, c.N = ML_TOK;
    if ((rc = one(c))) return rc;
  }
  const float norm = -(float)std::log((double)(n + ML_M));
  const float log_a_dust = norm + (float)std::log((double)(n - ML_M));
  B2_LAUNCH(ctx, k_ml_sinkhorn, Bc, 512, 0, st, s->sco.as<float>(), T, sm + s->dust, norm, log_a_dust, s->vsc.as<float>(), s->pm.as<float>());
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_ml_aggregate, dim3(ML_L / 16, Bc), 1024, 0, st, s->fcl.as<float>(), T, s->pm.as<float>(), s->agg.as<float>());
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_ml_assemble, Bc, 1024, 0, st, s->tfe.as<float>(), s->agg.as<float>(), s->dph.as<__half>() + (size_t)d0 * ML_AGG,
            s->dpl.as<__half>() + (size_t)d0 * ML_AGG);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// work buffers for chunks of up to ML_CHUNK images of a gh x gw grid and a call of B images; the position table of the grid
static int ml_prepare(b2_context* ctx, cudaStream_t st, int B, int gh, int gw) {
  MegaLocState* s = ctx->ml;
  const int Bc = B < ML_CHUNK ? B : ML_CHUNK, n = gh * gw, T = n + 1;
  const size_t M = (size_t)Bc * T, h = sizeof(__half), f = sizeof(float);
  B2_CUDA(ctx, s->col.ensure((size_t)Bc * n * ML_KPAD * 2 * h));
  B2_CUDA(ctx, s->x.ensure(M * ML_D * 2 * f));  // residual stream, then the final tokens
  B2_CUDA(ctx, s->lnp.ensure(M * ML_D * 2 * h));
  B2_CUDA(ctx, s->qkv.ensure(M * ML_QKV * 2 * h));
  B2_CUDA(ctx, s->att.ensure(M * ML_D * 2 * h));
  B2_CUDA(ctx, s->hid.ensure(M * ML_MLP * 2 * h));
  B2_CUDA(ctx, s->h1.ensure(M * 2 * ML_SMLP * 2 * h));
  B2_CUDA(ctx, s->fcl.ensure(M * ML_L * f));
  B2_CUDA(ctx, s->sco.ensure(M * ML_M * f));
  B2_CUDA(ctx, s->t1.ensure((size_t)Bc * ML_SMLP * 2 * h));
  B2_CUDA(ctx, s->tfe.ensure((size_t)Bc * ML_TOK * f));
  B2_CUDA(ctx, s->vsc.ensure((size_t)Bc * n * f));
  B2_CUDA(ctx, s->pm.ensure((size_t)Bc * ML_M * n * f));
  B2_CUDA(ctx, s->agg.ensure((size_t)Bc * ML_L * ML_M * f));
  B2_CUDA(ctx, s->dph.ensure((size_t)B * ML_AGG * h));
  B2_CUDA(ctx, s->dpl.ensure((size_t)B * ML_AGG * h));
  B2_CUDA(ctx, s->hout.ensure((size_t)B * ML_OUT * f));
  if (s->pos_gh != gh || s->pos_gw != gw) {
    B2_CUDA(ctx, s->postab.ensure((size_t)n * ML_D * f));
    const float* pos = s->small.as<float>() + s->pos;
    if (gh == ML_POS_G && gw == ML_POS_G) {  // the table as is (interpolate_pos_encoding returns pos_embed unchanged)
      B2_CUDA(ctx, cudaMemcpyAsync(s->postab.p, pos + ML_D, (size_t)n * ML_D * f, cudaMemcpyDeviceToDevice, st));
    } else {
      const float inv_h = (float)(1.0 / ((gh + 0.1) / ML_POS_G)), inv_w = (float)(1.0 / ((gw + 0.1) / ML_POS_G));
      B2_LAUNCH(ctx, k_ml_pos, n, 256, 0, st, pos, gh, gw, inv_h, inv_w, s->postab.as<float>());
      B2_CHECK_LAUNCH(ctx);
    }
    s->pos_gh = gh, s->pos_gw = gw;
  }
  B2_CUDA(ctx, cudaMemsetAsync(s->errflag.p, 0, 16, st));
  return B2_OK;
}

static int ml_check(b2_context* ctx, int B, int H, int W) {
  MegaLocState* s = ctx->ml;
  if (b2_force_simt(ctx)) return b2_fail(ctx, B2_ERR_STATE, "megaloc runs on the wgmma path only (force_simt is set)");
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "megaloc weights not set");
  if (B <= 0 || H <= 0 || W <= 0 || H % ML_P || W % ML_P) return b2_fail(ctx, B2_ERR_ARG, "megaloc needs H and W that are multiples of 14");
  if ((H / ML_P) * (W / ML_P) <= ML_M)
    return b2_fail(ctx, B2_ERR_ARG, "megaloc needs more than 64 patches (SALAD's dustbin weight is log(n - 64))");
  if ((int64_t)(H / ML_P) * (W / ML_P) > 65536) return b2_fail(ctx, B2_ERR_ARG, "megaloc takes at most 65536 patches per image");
  return B2_OK;
}

// the head over all B images of the call, then L2
static int ml_head(b2_context* ctx, cudaStream_t st, int B, float* out) {
  MegaLocState* s = ctx->ml;
  TcWeights tw{nullptr, nullptr, nullptr, s->errflag.as<int>(), true};
  tw.sm_count = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  const Pl w = ml_planes(s, s->head);
  int rc;
  for (int kc = 0; kc < ML_AGG; kc += ML_HEAD_KC) {
    LinArgs a;
    a.a1p = {s->dph.as<__half>() + kc, s->dpl.as<__half>() + kc}, a.lda1 = ML_AGG, a.K1 = ML_HEAD_KC;
    a.bp = {w.hi + kc, w.lo + kc}, a.ldb = ML_AGG;
    a.cf = s->hout.as<float>(), a.ldc = ML_OUT, a.tc_want_f32 = true, a.M = B, a.N = ML_OUT;
    if (kc == 0) a.bias = s->small.as<float>() + s->headb;
    else a.resid = s->hout.as<float>(), a.ldr = ML_OUT;
    if ((rc = run_linear(ctx, st, tw, &a, 1))) return rc;
  }
  B2_LAUNCH(ctx, k_ml_rownorm, B, 1024, 0, st, s->hout.as<float>(), ML_OUT, out);
  B2_CHECK_LAUNCH(ctx);
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&err, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

extern "C" int b2_megaloc_describe_dev(b2_context* ctx, const float* images, int B, int H, int W, float* out, void* stream) {
  if (!ctx || !images || !out) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  int rc;
  if ((rc = ml_check(ctx, B, H, W))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int gh = H / ML_P, gw = W / ML_P, n = gh * gw;
  if ((rc = ml_prepare(ctx, st, B, gh, gw))) return rc;
  MegaLocState* s = ctx->ml;
  const MlNorm nm{};
  for (int b0 = 0; b0 < B; b0 += ML_CHUNK) {
    const int Bc = B - b0 < ML_CHUNK ? B - b0 : ML_CHUNK;
    const size_t units = (size_t)Bc * n * (ML_KPAD / 2);
    __half* ch = s->col.as<__half>();
    B2_LAUNCH(ctx, k_ml_im2col<false>, (unsigned)((units + 255) / 256), 256, 0, st, (const void*)(images + (size_t)b0 * 3 * H * W), Bc, H, W, nm, ch,
              ch + (size_t)Bc * n * ML_KPAD);
    B2_CHECK_LAUNCH(ctx);
    if ((rc = ml_chunk(ctx, st, Bc, gh, gw, b0))) return rc;
  }
  return ml_head(ctx, st, B, out);
}

static int ml_resize(b2_context* ctx, cudaStream_t st, const uint8_t* const* images, int n, int H, int W, size_t pitch, uint8_t* out) {
  MegaLocState* s = ctx->ml;
  int rc;
  if ((rc = ml_resize_table(ctx, s->rh, W)) || (rc = ml_resize_table(ctx, s->rv, H))) return rc;
  B2_CUDA(ctx, s->rtmp.ensure((size_t)n * H * ML_RS * 3));
  MlSrcList src{};
  for (int i = 0; i < n; ++i) src.p[i] = images[i];
  B2_LAUNCH(ctx, k_ml_resize_h, dim3(cdiv(H * ML_RS, 256), n), 256, 0, st, src, pitch, H, s->rh.w.as<short>(), s->rh.x0.as<int>(), s->rh.taps,
            s->rh.prec, s->rtmp.as<uint8_t>());
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_ml_resize_v, dim3(cdiv(ML_RS * ML_RS, 256), n), 256, 0, st, s->rtmp.as<uint8_t>(), H, s->rv.w.as<short>(), s->rv.x0.as<int>(),
            s->rv.taps, s->rv.prec, out);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

static int ml_check_u8(b2_context* ctx, const uint8_t* const* images, int n, int H, int W, size_t pitch) {
  if (!images || n <= 0 || H <= 0 || W <= 0 || pitch < (size_t)W * 3) return b2_fail(ctx, B2_ERR_ARG, "megaloc u8: bad image list or shape");
  if ((int64_t)H * W > ((int64_t)1 << 26)) return b2_fail(ctx, B2_ERR_ARG, "megaloc u8: at most 2^26 pixels per image");
  for (int i = 0; i < n; ++i)
    if (!images[i]) return b2_fail(ctx, B2_ERR_ARG, "megaloc u8: null image pointer");
  return B2_OK;
}

extern "C" int b2_megaloc_resize_u8_dev(b2_context* ctx, const uint8_t* const* images, int n, int H, int W, size_t pitch, uint8_t* out,
                                        void* stream) {
  if (!ctx || !out) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->ml) ctx->ml = new MegaLocState();
  int rc;
  if ((rc = ml_check_u8(ctx, images, n, H, W, pitch))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < n; b0 += ML_CHUNK) {
    const int Bc = n - b0 < ML_CHUNK ? n - b0 : ML_CHUNK;
    if ((rc = ml_resize(ctx, st, images + b0, Bc, H, W, pitch, out + (size_t)b0 * 3 * ML_RS * ML_RS))) return rc;
  }
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B2_OK;
}

extern "C" int b2_megaloc_describe_u8_dev(b2_context* ctx, const uint8_t* const* images, int n, int H, int W, size_t pitch, float* out,
                                          void* stream) {
  if (!ctx || !out) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  int rc;
  if ((rc = ml_check(ctx, n > 0 ? n : 1, ML_RS, ML_RS)) || (rc = ml_check_u8(ctx, images, n, H, W, pitch))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = ML_RS / ML_P, np = g * g;
  if ((rc = ml_prepare(ctx, st, n, g, g))) return rc;
  MegaLocState* s = ctx->ml;
  B2_CUDA(ctx, s->rsz.ensure((size_t)ML_CHUNK * 3 * ML_RS * ML_RS));
  const MlNorm nm{{0.485f, 0.456f, 0.406f}, {0.229f, 0.224f, 0.225f}};  // the plugin's ImageNet normalisation
  for (int b0 = 0; b0 < n; b0 += ML_CHUNK) {
    const int Bc = n - b0 < ML_CHUNK ? n - b0 : ML_CHUNK;
    if ((rc = ml_resize(ctx, st, images + b0, Bc, H, W, pitch, s->rsz.as<uint8_t>()))) return rc;
    const size_t units = (size_t)Bc * np * (ML_KPAD / 2);
    __half* ch = s->col.as<__half>();
    B2_LAUNCH(ctx, k_ml_im2col<true>, (unsigned)((units + 255) / 256), 256, 0, st, (const void*)s->rsz.p, Bc, ML_RS, ML_RS, nm, ch,
              ch + (size_t)Bc * np * ML_KPAD);
    B2_CHECK_LAUNCH(ctx);
    if ((rc = ml_chunk(ctx, st, Bc, g, g, b0))) return rc;
  }
  return ml_head(ctx, st, n, out);
}

// HOST buffers in / out (images [B][3][H][W] normalised fp32, out [B][8448])
extern "C" int b2_megaloc_describe_host(b2_context* ctx, const float* images, int B, int H, int W, float* out) {
  if (!ctx || !images || !out || B <= 0 || H <= 0 || W <= 0) return B2_ERR_ARG;
  DevBuf in_d, out_d;
  const size_t nin = (size_t)B * 3 * H * W * sizeof(float), nout = (size_t)B * ML_OUT * sizeof(float);
  cudaSetDevice(ctx->device);
  B2_CUDA(ctx, in_d.ensure(nin));
  B2_CUDA(ctx, out_d.ensure(nout));
  B2_CUDA(ctx, cudaMemcpy(in_d.p, images, nin, cudaMemcpyHostToDevice));
  const int rc = b2_megaloc_describe_dev(ctx, in_d.as<float>(), B, H, W, out_d.as<float>(), ctx->stream);
  if (rc != B2_OK) return rc;
  B2_CUDA(ctx, cudaMemcpy(out, out_d.p, nout, cudaMemcpyDeviceToHost));
  return B2_OK;
}
