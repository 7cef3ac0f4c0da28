// D2-Net detector-descriptor, single scale (gtsfm/frontend/detector_descriptor/d2net.py with USE_MULTISCALE = False, i.e.
// thirdparty/d2net/lib/pyramid.py process_multiscale(scales=[1]); the model is thirdparty/d2net/lib/model_test.py with
// use_relu=True and the 'torch' preprocessing of thirdparty/d2net/lib/utils.py).
//
//   uint8 image -> per-channel table (x / 255 in fp32, (x - mean) / std in fp64, rounded to fp32) -> VGG16 conv1_1 .. conv3_3
//   (ReLU, 2x2/2 max-pools after conv1_2 and conv2_2) -> AvgPool2d(2, stride=1) -> conv4_1 .. conv4_3 (3x3, dilation 2,
//   padding 2, ReLU) -> dense map [h][w][512] fp32 -> hard detection + handcrafted localisation -> score-ordered top-k ->
//   bilinear descriptors, L2-normalised.
//
// Kernels and where they run:
//   conv1_1          k_d2_conv0 (SIMT, fp32; the normalisation is a 3 x 256 table built on the host, padding is zero AFTER it)
//   conv1_2 .. 3_3   k_conv_ps<1> (conv_ps.cuh: persistent wgmma implicit GEMM, split-fp16 ~ fp32), pools fused; conv3_3 -> fp32
//   avg pool         k_d2_avgpool (SIMT, fp32 in, planes out)
//   conv4_1 .. 4_3   k_conv_ps<2> (the dilated instance); conv4_3 writes the fp32 dense map NHWC
//   detection        k_d2_detect: one warp per feature cell reads its 512 contiguous channels; every channel equal to the
//                    depth-wise max is tested (3x3 max with -inf padding, Hessian with zero padding, det > 0, tr^2/det <= 7.2f),
//                    localised (step = -H^-1 grad, |step| < 0.5) and kept when its four bilinear corners lie in the map.
//                    A cell whose maximum is <= 0 cannot detect: after the ReLU all its channels and (for a 3x3 maximum) all
//                    neighbours of the channel are 0, so det = 0.
//   order / top-k    k_d2_rank: the rank of each candidate's key (score descending, then the reference's torch.nonzero order
//                    (c, i, j)) by counting smaller keys; the first max_keypoints ranks are the output, already sorted.
//   description      k_d2_describe: one warp per kept keypoint, the reference's float32 bilinear weights, no FMA contraction.
// Counts stay on the device; a batched call synchronises once.
#include "common.cuh"
#include "conv_ps.cuh"

constexpr int D2_NCONV = 10, D2_D = 512, D2_MAX_IMAGES = 64;
constexpr int D2_MAX_EDGE = 1600, D2_MAX_SUM_EDGES = 2800;  // beyond these the reference resizes (scipy.misc.imresize)
static const int D2_CI[D2_NCONV] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512};
static const int D2_CO[D2_NCONV] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512};
static const int D2_POOL[D2_NCONV] = {0, 1, 0, 1, 0, 0, 0, 0, 0, 0};  // MaxPool2d(2, 2) after the layer
static const int D2_DIL[D2_NCONV] = {1, 1, 1, 1, 1, 1, 1, 2, 2, 2};
static const double D2_MEAN[3] = {0.485, 0.456, 0.406}, D2_STD[3] = {0.229, 0.224, 0.225};

struct D2Cand {
  unsigned long long key;  // (~score bits) << 32 | c << 22 | i << 11 | j: ascending = score descending, then (c, i, j)
  float fi, fj;            // localised feature-map position
  int pad[2];
};

__device__ __forceinline__ unsigned long long d2_key(float score, int c, int i, int j) {
  return ((unsigned long long)(~__float_as_uint(score)) << 32) | ((unsigned long long)c << 22) | ((unsigned)i << 11) | (unsigned)j;
}

struct D2NetState {
  bool loaded = false;
  DevBuf w0, bias, wh, wl, table, errflag;  // weights
  size_t woff[D2_NCONV] = {}, boff[D2_NCONV] = {};
  DevBuf actA, actB, f3, dense, cand, order, counts;  // work
};

void d2_destroy(b2_context* ctx) {
  if (!ctx->d2) return;
  D2NetState* s = ctx->d2;
  DevBuf* bufs[] = {&s->w0, &s->bias, &s->wh, &s->wl, &s->table, &s->errflag, &s->actA, &s->actB, &s->f3, &s->dense, &s->cand,
                    &s->order, &s->counts};
  for (DevBuf* b : bufs) b->release();
  delete s;
  ctx->d2 = nullptr;
}

// conv1_1: 3 -> 64 on the table-normalised uint8 image (gray: every channel reads the one byte), 3x3, pad 1, bias, ReLU -> planes.
// block = 32 pixels x 8 channel groups of 8; weights [27][64] and the table in shared memory.
__global__ void __launch_bounds__(256) k_d2_conv0(const uint8_t* __restrict__ img, size_t pitch, int C, const float* __restrict__ table,
                                                  const float* __restrict__ wt, const float* __restrict__ bias, int H, int W,
                                                  __half* __restrict__ oh, __half* __restrict__ ol) {
  __shared__ float ws[27 * 64];
  __shared__ float tb[3 * 256];
  for (int i = threadIdx.x; i < 27 * 64; i += 256) ws[i] = wt[i];
  for (int i = threadIdx.x; i < 3 * 256; i += 256) tb[i] = table[i];
  __syncthreads();
  const long long pix = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const int cg = threadIdx.x & 7;
  if (pix >= (long long)H * W) return;
  const int y = (int)(pix / W), x = (int)(pix % W);
  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = __ldg(bias + cg * 8 + c);
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int yy = y + dy, xx = x + dx;
      const bool in = yy >= 0 && yy < H && xx >= 0 && xx < W;
      const uint8_t* px = img + (size_t)yy * pitch + (size_t)xx * C;
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float v = in ? tb[ci * 256 + __ldg(px + (C == 3 ? ci : 0))] : 0.f;
        const float* wp = &ws[(((dy + 1) * 3 + (dx + 1)) * 3 + ci) * 64 + cg * 8];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = fmaf(v, wp[c], acc[c]);
      }
    }
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) tc::split2(fmaxf(acc[2 * i], 0.f), fmaxf(acc[2 * i + 1], 0.f), hi[i], lo[i]);
  *reinterpret_cast<uint4*>(oh + (size_t)pix * 64 + cg * 8) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(ol + (size_t)pix * 64 + cg * 8) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// AvgPool2d(2, stride=1) on fp32 NHWC [H][W][256] -> planes [H - 1][W - 1][256]: ((a00 + a01) + a10) + a11, then / 4.
__global__ void __launch_bounds__(256) k_d2_avgpool(const float* __restrict__ in, int H, int W, __half* __restrict__ oh,
                                                    __half* __restrict__ ol) {
  constexpr int C = 256;
  const long long e = ((long long)blockIdx.x * 256 + threadIdx.x) * 2;  // two channels per thread
  const int OW = W - 1;
  if (e >= (long long)(H - 1) * OW * C) return;
  const int c = (int)(e % C);
  const long long pix = e / C;
  const int y = (int)(pix / OW), x = (int)(pix % OW);
  const float* p = in + ((size_t)y * W + x) * C + c;
  const float2 a = *reinterpret_cast<const float2*>(p), b = *reinterpret_cast<const float2*>(p + C);
  const float2 d = *reinterpret_cast<const float2*>(p + (size_t)W * C), f = *reinterpret_cast<const float2*>(p + (size_t)W * C + C);
  const float s0 = __fadd_rn(__fadd_rn(__fadd_rn(a.x, b.x), d.x), f.x) * 0.25f;
  const float s1 = __fadd_rn(__fadd_rn(__fadd_rn(a.y, b.y), d.y), f.y) * 0.25f;
  uint32_t hi, lo;
  tc::split2(s0, s1, hi, lo);
  *reinterpret_cast<uint32_t*>(oh + e) = hi;
  *reinterpret_cast<uint32_t*>(ol + e) = lo;
}

// HardDetectionModule + HandcraftedLocalizationModule + interpolate_dense_features' corner test for every channel equal to
// its cell's depth-wise maximum.  One warp per cell of F [h][w][512].
__global__ void __launch_bounds__(256) k_d2_detect(const float* __restrict__ F, int h, int w, D2Cand* __restrict__ cand, int cap,
                                                   int* __restrict__ count) {
  const int cell = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (cell >= h * w) return;
  const int i = cell / w, j = cell % w;
  const float4* p = reinterpret_cast<const float4*>(F + (size_t)cell * D2_D);
  float v[16];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 q = p[lane + 32 * k];
    v[4 * k] = q.x, v[4 * k + 1] = q.y, v[4 * k + 2] = q.z, v[4 * k + 3] = q.w;
  }
  float m = v[0];
#pragma unroll
  for (int k = 1; k < 16; ++k) m = fmaxf(m, v[k]);
  m = warp_max(m);
  if (!(m > 0.f)) return;
  auto at = [&](int c, int di, int dj) -> float {  // conv2d's zero padding
    const int ii = i + di, jj = j + dj;
    return ii >= 0 && ii < h && jj >= 0 && jj < w ? __ldg(F + ((size_t)ii * w + jj) * D2_D + c) : 0.f;
  };
  unsigned ties = 0;  // this lane's channels equal to the depth-wise maximum (several only where channels tie)
#pragma unroll
  for (int k = 0; k < 16; ++k) ties |= (v[k] == m ? 1u : 0u) << k;
  while (ties) {
    const int k = __ffs(ties) - 1;
    ties &= ties - 1;
    const int c = (lane + 32 * (k >> 2)) * 4 + (k & 3);
    const float x0 = m;
    // 3x3 maximum of channel c (max_pool2d pads with -inf: out-of-map neighbours do not count)
    bool local_max = true;
    for (int di = -1; di <= 1; ++di)
      for (int dj = -1; dj <= 1; ++dj) {
        const int ii = i + di, jj = j + dj;
        if ((di || dj) && ii >= 0 && ii < h && jj >= 0 && jj < w && __ldg(F + ((size_t)ii * w + jj) * D2_D + c) > x0) local_max = false;
      }
    if (!local_max) continue;
    const float u = at(c, -1, 0), dn = at(c, 1, 0), l = at(c, 0, -1), r = at(c, 0, 1);
    const float ul = at(c, -1, -1), ur = at(c, -1, 1), dl = at(c, 1, -1), dr = at(c, 1, 1);
    const float m2 = -2.f * x0;
    const float dii = __fadd_rn(__fadd_rn(u, m2), dn);
    const float djj = __fadd_rn(__fadd_rn(l, m2), r);
    const float dij = __fadd_rn(__fadd_rn(__fadd_rn(0.25f * ul, -0.25f * ur), -0.25f * dl), 0.25f * dr);
    const float det = __fsub_rn(__fmul_rn(dii, djj), __fmul_rn(dij, dij));
    const float tr = __fadd_rn(dii, djj);
    if (!(det > 0.f) || !(__fdiv_rn(__fmul_rn(tr, tr), det) <= 7.2f)) continue;
    const float ih00 = __fdiv_rn(djj, det), ih01 = __fdiv_rn(-dij, det), ih11 = __fdiv_rn(dii, det);
    const float gi = __fadd_rn(-0.5f * u, 0.5f * dn), gj = __fadd_rn(-0.5f * l, 0.5f * r);
    const float si = -__fadd_rn(__fmul_rn(ih00, gi), __fmul_rn(ih01, gj));
    const float sj = -__fadd_rn(__fmul_rn(ih01, gi), __fmul_rn(ih11, gj));
    if (!(fabsf(si) < 0.5f && fabsf(sj) < 0.5f)) continue;
    const float fi = __fadd_rn((float)i, si), fj = __fadd_rn((float)j, sj);
    if (floorf(fi) < 0.f || ceilf(fi) >= (float)h || floorf(fj) < 0.f || ceilf(fj) >= (float)w) continue;
    const int slot = atomicAdd(count, 1);
    if (slot < cap) {
      D2Cand d;
      d.key = d2_key(x0, c, i, j);
      d.fi = fi, d.fj = fj, d.pad[0] = d.pad[1] = 0;
      cand[slot] = d;
    }
  }
}

// rank of every candidate among its image's candidates (keys are distinct); ranks below max_k are written to order[rank]
__global__ void __launch_bounds__(256) k_d2_rank(const D2Cand* __restrict__ cand, const int* __restrict__ count, int cap, int max_k,
                                                 int* __restrict__ order) {
  __shared__ unsigned long long sk[256];
  const int n = min(*count, cap);
  if (blockIdx.x * 256 >= n) return;  // uniform per block
  const int idx = blockIdx.x * 256 + threadIdx.x;
  const unsigned long long my = idx < n ? cand[idx].key : ~0ull;
  int rank = 0;
  for (int t0 = 0; t0 < n; t0 += 256) {
    __syncthreads();
    sk[threadIdx.x] = t0 + (int)threadIdx.x < n ? cand[t0 + threadIdx.x].key : ~0ull;
    __syncthreads();
    const int lim = min(256, n - t0);
    for (int q = 0; q < lim; ++q) rank += sk[q] < my;
  }
  if (idx < n && rank < max_k) order[rank] = idx;
}

// output slot r: position ((p * 2 + 0.5) * 2 + 0.5) as (x, y), the score, and the L2-normalised bilinear descriptor with
// interpolate_dense_features' float32 weights summed tl + tr + bl + br.  One warp per slot.
__global__ void __launch_bounds__(256) k_d2_describe(const float* __restrict__ F, int w, const D2Cand* __restrict__ cand,
                                                     const int* __restrict__ order, const int* __restrict__ count, int cap, int max_k,
                                                     float* __restrict__ out_xy, float* __restrict__ out_score, float* __restrict__ out_desc) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= min(min(*count, cap), max_k)) return;
  const D2Cand d = cand[order[r]];
  const float fi = d.fi, fj = d.fj;
  const int i0 = (int)floorf(fi), j0 = (int)floorf(fj), i1 = (int)ceilf(fi), j1 = (int)ceilf(fj);
  const float ai = __fsub_rn(fi, (float)i0), aj = __fsub_rn(fj, (float)j0);
  const float bi = __fsub_rn(1.f, ai), bj = __fsub_rn(1.f, aj);
  const float wtl = __fmul_rn(bi, bj), wtr = __fmul_rn(bi, aj), wbl = __fmul_rn(ai, bj), wbr = __fmul_rn(ai, aj);
  const float4* tl = reinterpret_cast<const float4*>(F + ((size_t)i0 * w + j0) * D2_D);
  const float4* tr = reinterpret_cast<const float4*>(F + ((size_t)i0 * w + j1) * D2_D);
  const float4* bl = reinterpret_cast<const float4*>(F + ((size_t)i1 * w + j0) * D2_D);
  const float4* br = reinterpret_cast<const float4*>(F + ((size_t)i1 * w + j1) * D2_D);
  auto mix = [&](float a, float b, float c, float e) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(wtl, a), __fmul_rn(wtr, b)), __fmul_rn(wbl, c)), __fmul_rn(wbr, e));
  };
  float4 o[4];
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 a = tl[lane + 32 * k], b = tr[lane + 32 * k], c = bl[lane + 32 * k], e = br[lane + 32 * k];
    o[k] = make_float4(mix(a.x, b.x, c.x, e.x), mix(a.y, b.y, c.y, e.y), mix(a.z, b.z, c.z, e.z), mix(a.w, b.w, c.w, e.w));
    ss += o[k].x * o[k].x + o[k].y * o[k].y + o[k].z * o[k].z + o[k].w * o[k].w;
  }
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  float4* dst = reinterpret_cast<float4*>(out_desc + (size_t)r * D2_D);
#pragma unroll
  for (int k = 0; k < 4; ++k) dst[lane + 32 * k] = make_float4(o[k].x / nrm, o[k].y / nrm, o[k].z / nrm, o[k].w / nrm);
  if (lane == 0) {
    const float y = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(fi, 2.f), 0.5f), 2.f), 0.5f);
    const float x = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(fj, 2.f), 0.5f), 2.f), 0.5f);
    out_xy[2 * r] = x, out_xy[2 * r + 1] = y;
    out_score[r] = __uint_as_float(~(unsigned)(d.key >> 32));
  }
}

// the preprocess_image('torch') value of every byte and channel, bit for bit: float32(u) / 255 in float32, then
// (x - mean) / std in float64 (numpy promotes against the float64 mean / std arrays), rounded to float32
static void d2_table(float* t) {
  for (int c = 0; c < 3; ++c)
    for (int u = 0; u < 256; ++u) {
      const float x = (float)u / 255.0f;
      t[c * 256 + u] = (float)(((double)x - D2_MEAN[c]) / D2_STD[c]);
    }
}

static size_t d2_blob_floats() {
  size_t n = 0;
  for (int l = 0; l < D2_NCONV; ++l) n += (size_t)D2_CO[l] * D2_CI[l] * 9 + D2_CO[l];
  return n;
}

extern "C" size_t b2_d2net_blob_floats(void) { return d2_blob_floats(); }

extern "C" int b2_d2net_norm_table(float* out) {
  if (!out) return B2_ERR_ARG;
  d2_table(out);
  return B2_OK;
}

extern "C" int b2_d2net_set_weights(b2_context* ctx, const float* blob, size_t n_floats) {
  if (!ctx || !blob) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (b2_force_simt(ctx)) return b2_fail(ctx, B2_ERR_STATE, "d2net runs on the wgmma path only (force_simt is set)");
  if (n_floats != d2_blob_floats()) return b2_fail(ctx, B2_ERR_ARG, "d2net blob must hold " + std::to_string(d2_blob_floats()) + " floats, got " + std::to_string(n_floats));
  if (!tma_encoder()) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled is not available (driver too old?)");
  cudaSetDevice(ctx->device);
  if (!ctx->d2) ctx->d2 = new D2NetState();
  D2NetState* s = ctx->d2;
  s->loaded = false;
  // layer 0 as fp32 [tap][ci][co]; layers 1..9 as [co][tap * Cin + ci] planes; biases concatenated (conv_ps.cuh, shared with NetVLAD)
  std::vector<float> stage, b, w0, table(3 * 256);
  conv_ps_repack(blob, D2_NCONV, D2_CI, D2_CO, stage, b, w0, s->woff, s->boff);
  const size_t btot = b.size();
  d2_table(table.data());
  DevBuf tmp;
  B2_CUDA(ctx, tmp.ensure(stage.size() * sizeof(float)));
  B2_CUDA(ctx, conv_ps_upload_planes(stage.data(), stage.size(), s->wh, s->wl, tmp, stage.size()));
  tmp.release();
  B2_CUDA(ctx, s->w0.ensure(w0.size() * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->w0.p, w0.data(), w0.size() * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, s->bias.ensure(btot * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->bias.p, b.data(), btot * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, s->table.ensure(table.size() * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->table.p, table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, s->errflag.ensure(16));
  B2_CUDA(ctx, cudaMemset(s->errflag.p, 0, 16));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_conv_ps<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CP_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_conv_ps<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CpGeom<2>::SMEM));
  s->loaded = true;
  return B2_OK;
}

// one VGG layer l >= 1 on split planes `in` [H][W][Cin] -> planes `oh` and / or fp32 `of` (ReLU always: use_relu covers conv4_3)
static int d2_conv(b2_context* ctx, cudaStream_t st, const __half* ih, int l, int H, int W, __half* oh, float* of) {
  D2NetState* s = ctx->d2;
  return conv_ps_run(ctx, st, ih, H, W, D2_CI[l], D2_CO[l], D2_POOL[l], 1, D2_DIL[l], s->wh.as<__half>() + s->woff[l], s->wl.as<__half>() + s->woff[l],
                     s->bias.as<float>() + s->boff[l], oh, of, s->errflag.as<int>(), "d2net");
}

static void d2_map_shape(int H, int W, int* h, int* w) {  // two 2x2/2 max-pools, then the 2x2 stride-1 average pool
  *h = H / 2 / 2 - 1, *w = W / 2 / 2 - 1;
}

static int d2_cap(int cells) { return 4 * cells + 1024; }  // candidates per image (several only where channels tie)

extern "C" int b2_d2net_detect_batched_dev(b2_context* ctx, b2_d2net_image* images, int n_images, int height, int width, int channels,
                                           size_t pitch, void* stream) {
  if (!ctx || !images) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (b2_force_simt(ctx)) return b2_fail(ctx, B2_ERR_STATE, "d2net runs on the wgmma path only (force_simt is set)");
  D2NetState* s = ctx->d2;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "d2net weights not set");
  if (n_images < 1 || n_images > D2_MAX_IMAGES) return b2_fail(ctx, B2_ERR_ARG, "d2net takes 1 .. 64 images per call");
  if (channels != 1 && channels != 3) return b2_fail(ctx, B2_ERR_ARG, "d2net takes gray (1 channel) or RGB (3 channel) uint8 images");
  if (height < 8 || width < 8) return b2_fail(ctx, B2_ERR_ARG, "d2net needs images of at least 8 x 8 pixels (two max-pools and the average pool)");
  if ((height > width ? height : width) > D2_MAX_EDGE || height + width > D2_MAX_SUM_EDGES)
    return b2_fail(ctx, B2_ERR_ARG, "d2net takes images with edges <= 1600 and summing to <= 2800 (the reference resizes larger ones)");
  if (pitch < (size_t)width * channels) return b2_fail(ctx, B2_ERR_ARG, "pitch is smaller than a row");
  for (int b = 0; b < n_images; ++b) {
    const b2_d2net_image& im = images[b];
    if (!im.image || im.max_keypoints < 0 || (im.max_keypoints > 0 && (!im.out_xy || !im.out_scores || !im.out_desc)))
      return b2_fail(ctx, B2_ERR_ARG, "d2net image " + std::to_string(b) + ": missing image / output pointer or negative max_keypoints");
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int H = height, W = width;
  int h, w;
  d2_map_shape(H, W, &h, &w);
  const int cells = h * w, cap = d2_cap(cells);
  int max_k = 0;
  for (int b = 0; b < n_images; ++b) max_k = images[b].max_keypoints > max_k ? images[b].max_keypoints : max_k;
  const size_t px = (size_t)H * W;
  B2_CUDA(ctx, s->actA.ensure(px * 64 * 2 * sizeof(__half)));  // conv1_1's output is the largest activation
  B2_CUDA(ctx, s->actB.ensure(px * 64 * 2 * sizeof(__half)));
  B2_CUDA(ctx, s->f3.ensure((size_t)(H / 4) * (W / 4) * 256 * sizeof(float)));
  B2_CUDA(ctx, s->dense.ensure((size_t)cells * D2_D * sizeof(float)));
  B2_CUDA(ctx, s->cand.ensure((size_t)cap * sizeof(D2Cand)));
  B2_CUDA(ctx, s->order.ensure((size_t)(max_k > 0 ? max_k : 1) * sizeof(int)));
  B2_CUDA(ctx, s->counts.ensure((size_t)n_images * sizeof(int)));
  B2_CUDA(ctx, cudaMemsetAsync(s->errflag.p, 0, 16, st));
  B2_CUDA(ctx, cudaMemsetAsync(s->counts.p, 0, (size_t)n_images * sizeof(int), st));
  __half* A = s->actA.as<__half>();
  __half* B = s->actB.as<__half>();
  float* dense = s->dense.as<float>();
  D2Cand* cand = s->cand.as<D2Cand>();
  int rc;
  for (int b = 0; b < n_images; ++b) {
    const b2_d2net_image& im = images[b];
    int* count = s->counts.as<int>() + b;
    B2_LAUNCH(ctx, k_d2_conv0, (unsigned)((px + 31) / 32), 256, 0, st, im.image, pitch, channels, s->table.as<float>(), s->w0.as<float>(),
              s->bias.as<float>(), H, W, A, A + px * 64);
    B2_CHECK_LAUNCH(ctx);
    // conv1_2 (pool) A->B, conv2_1 B->A, conv2_2 (pool) A->B, conv3_1 B->A, conv3_2 A->B, conv3_3 B->f3 (fp32)
    int ch = H, cw = W;
    __half* cur = A;
    __half* nxt = B;
    for (int l = 1; l <= 6; ++l) {
      const bool last = l == 6;
      if ((rc = d2_conv(ctx, st, cur, l, ch, cw, last ? nullptr : nxt, last ? s->f3.as<float>() : nullptr))) return rc;
      if (D2_POOL[l]) ch /= 2, cw /= 2;
      std::swap(cur, nxt);
    }
    const long long pe = (long long)(ch - 1) * (cw - 1) * 256 / 2;
    B2_LAUNCH(ctx, k_d2_avgpool, (unsigned)((pe + 255) / 256), 256, 0, st, s->f3.as<float>(), ch, cw, A, A + (size_t)h * w * 256);
    B2_CHECK_LAUNCH(ctx);
    // conv4_1 A->B, conv4_2 B->A, conv4_3 A->dense (fp32)
    if ((rc = d2_conv(ctx, st, A, 7, h, w, B, nullptr))) return rc;
    if ((rc = d2_conv(ctx, st, B, 8, h, w, A, nullptr))) return rc;
    if ((rc = d2_conv(ctx, st, A, 9, h, w, nullptr, dense))) return rc;
    B2_LAUNCH(ctx, k_d2_detect, cdiv(cells, 8), 256, 0, st, dense, h, w, cand, cap, count);
    B2_CHECK_LAUNCH(ctx);
    if (im.max_keypoints > 0) {
      B2_LAUNCH(ctx, k_d2_rank, cdiv(cap, 256), 256, 0, st, cand, count, cap, im.max_keypoints, s->order.as<int>());
      B2_CHECK_LAUNCH(ctx);
      B2_LAUNCH(ctx, k_d2_describe, cdiv(im.max_keypoints, 8), 256, 0, st, dense, w, cand, s->order.as<int>(), count, cap, im.max_keypoints,
                im.out_xy, im.out_scores, im.out_desc);
      B2_CHECK_LAUNCH(ctx);
    }
  }
  std::vector<int> cnt(n_images);
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(cnt.data(), s->counts.p, (size_t)n_images * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  for (int b = 0; b < n_images; ++b) {
    if (cnt[b] > cap) return b2_fail(ctx, B2_ERR_STATE, "d2net: more tied detections than the candidate workspace holds");
    images[b].out_total = cnt[b];
    images[b].out_n = cnt[b] < images[b].max_keypoints ? cnt[b] : images[b].max_keypoints;
  }
  return B2_OK;
}

extern "C" int b2_d2net_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels, int max_keypoints,
                                    float* out_xy, float* out_scores, float* out_desc, int* out_n, int* out_total) {
  if (!ctx || !image || !out_n || max_keypoints < 0 || height <= 0 || width <= 0 || (channels != 1 && channels != 3)) return B2_ERR_ARG;
  if (max_keypoints > 0 && (!out_xy || !out_scores || !out_desc)) return B2_ERR_ARG;
  DevBuf img_d, xy_d, sc_d, de_d;
  const size_t nin = (size_t)height * width * channels, k = max_keypoints > 0 ? (size_t)max_keypoints : 1;
  cudaSetDevice(ctx->device);
  B2_CUDA(ctx, img_d.ensure(nin));
  B2_CUDA(ctx, xy_d.ensure(k * 2 * sizeof(float)));
  B2_CUDA(ctx, sc_d.ensure(k * sizeof(float)));
  B2_CUDA(ctx, de_d.ensure(k * D2_D * sizeof(float)));
  int rc = B2_ERR_CUDA;
  b2_d2net_image im{img_d.as<uint8_t>(), max_keypoints, xy_d.as<float>(), sc_d.as<float>(), de_d.as<float>(), 0, 0};
  if (cudaMemcpy(img_d.p, image, nin, cudaMemcpyHostToDevice) == cudaSuccess) {
    rc = b2_d2net_detect_batched_dev(ctx, &im, 1, height, width, channels, (size_t)width * channels, ctx->stream);
    if (rc == B2_OK) {
      const size_t n = (size_t)im.out_n;
      if (n && (cudaMemcpy(out_xy, xy_d.p, n * 2 * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
          cudaMemcpy(out_scores, sc_d.p, n * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
          cudaMemcpy(out_desc, de_d.p, n * D2_D * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess))
        rc = b2_fail(ctx, B2_ERR_CUDA, "copy of the keypoints failed");
      *out_n = im.out_n;
      if (out_total) *out_total = im.out_total;
    }
  } else {
    b2_fail(ctx, B2_ERR_CUDA, "copy of the image failed");
  }
  img_d.release(), xy_d.release(), sc_d.release(), de_d.release();
  return rc;
}

// ---- test-only entry points: the dilated convolution, the average pool and the ordering, each on its own ---------------------

__global__ void k_d2_debug_keys(const float* __restrict__ score, const int* __restrict__ cij, int n, D2Cand* __restrict__ cand) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  D2Cand d;
  d.key = d2_key(score[t], cij[3 * t], cij[3 * t + 1], cij[3 * t + 2]);
  d.fi = d.fj = 0.f, d.pad[0] = d.pad[1] = 0;
  cand[t] = d;
}

extern "C" int b2_debug_conv_ps_host(b2_context* ctx, int dilation, const float* in, int H, int W, int Cin, int Cout, const float* weight,
                                     const float* bias, int relu, float* out) {
  if (!ctx || !in || !weight || !bias || !out || H <= 0 || W <= 0 || Cin % 64 || Cout % 64 || Cin <= 0 || Cout <= 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!tma_encoder()) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled is not available");
  cudaSetDevice(ctx->device);
  std::vector<float> wk((size_t)Cout * 9 * Cin);
  for (int o = 0; o < Cout; ++o)  // OIHW -> [co][tap * Cin + ci], the order conv_ps_repack gives layers >= 1
    for (int tp = 0; tp < 9; ++tp)
      for (int i = 0; i < Cin; ++i) wk[(size_t)o * 9 * Cin + (size_t)tp * Cin + i] = weight[((size_t)o * Cin + i) * 9 + tp];
  const size_t nin = (size_t)H * W * Cin, nout = (size_t)H * W * Cout;
  DevBuf tmp, wh, wl, ip, il, b, o, err;
  auto done = [&](int rc) {
    DevBuf* bufs[] = {&tmp, &wh, &wl, &ip, &il, &b, &o, &err};
    for (DevBuf* x : bufs) x->release();
    return rc;
  };
  const size_t big = nin > wk.size() ? nin : wk.size();
  // ip holds both planes (hi, then lo): allocated at full size first, so the upload below does not reallocate it
  if (ip.ensure(2 * nin * sizeof(__half)) || tmp.ensure(big * sizeof(float)) || conv_ps_upload_planes(wk.data(), wk.size(), wh, wl, tmp, big) ||
      conv_ps_upload_planes(in, nin, ip, il, tmp, big) || b.ensure(Cout * sizeof(float)) || o.ensure(nout * sizeof(float)) || err.ensure(16) ||
      cudaMemcpy(b.p, bias, Cout * sizeof(float), cudaMemcpyHostToDevice) || cudaMemset(err.p, 0, 16))
    return done(b2_fail(ctx, B2_ERR_CUDA, "debug conv: allocation or copy failed"));
  // the kernel reads the lo plane right after the hi one
  if (cudaMemcpy(ip.as<__half>() + nin, il.p, nin * sizeof(__half), cudaMemcpyDeviceToDevice))
    return done(b2_fail(ctx, B2_ERR_CUDA, "debug conv: plane copy failed"));
  if (cudaFuncSetAttribute(k_conv_ps<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CP_SMEM) ||
      cudaFuncSetAttribute(k_conv_ps<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CpGeom<2>::SMEM))
    return done(b2_fail(ctx, B2_ERR_CUDA, "debug conv: shared-memory attribute"));
  int rc = conv_ps_run(ctx, ctx->stream, ip.as<__half>(), H, W, Cin, Cout, 0, relu, dilation, wh.as<__half>(), wl.as<__half>(), b.as<float>(),
                       nullptr, o.as<float>(), err.as<int>(), "debug");
  if (rc) return done(rc);
  int e = 0;
  if (cudaStreamSynchronize(ctx->stream) || cudaMemcpy(&e, err.p, sizeof(int), cudaMemcpyDeviceToHost) ||
      cudaMemcpy(out, o.p, nout * sizeof(float), cudaMemcpyDeviceToHost))
    return done(b2_fail(ctx, B2_ERR_CUDA, std::string("debug conv: ") + cudaGetErrorString(cudaGetLastError())));
  return done(e ? b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)") : B2_OK);
}

extern "C" int b2_debug_d2net_avgpool_host(b2_context* ctx, const float* in, int H, int W, float* out) {
  if (!ctx || !in || !out || H < 2 || W < 2) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  const size_t nin = (size_t)H * W * 256, nout = (size_t)(H - 1) * (W - 1) * 256;
  DevBuf i, p;
  B2_CUDA(ctx, i.ensure(nin * sizeof(float)));
  B2_CUDA(ctx, p.ensure(nout * 2 * sizeof(__half)));
  B2_CUDA(ctx, cudaMemcpy(i.p, in, nin * sizeof(float), cudaMemcpyHostToDevice));
  B2_LAUNCH(ctx, k_d2_avgpool, (unsigned)((nout / 2 + 255) / 256), 256, 0, ctx->stream, i.as<float>(), H, W, p.as<__half>(), p.as<__half>() + nout);
  B2_CHECK_LAUNCH(ctx);
  std::vector<__half> hl(2 * nout);
  B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  B2_CUDA(ctx, cudaMemcpy(hl.data(), p.p, 2 * nout * sizeof(__half), cudaMemcpyDeviceToHost));
  for (size_t k = 0; k < nout; ++k) out[k] = __half2float(hl[k]) + __half2float(hl[nout + k]) * (1.0f / 2048.0f);  // hi + lo 2^-11
  i.release(), p.release();
  return B2_OK;
}

extern "C" int b2_debug_d2net_rank_host(b2_context* ctx, const float* scores, const int* cij, int n, int max_k, int* order) {
  if (!ctx || !scores || !cij || !order || n <= 0 || max_k <= 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  DevBuf sc, ij, cand, cnt, ord;
  B2_CUDA(ctx, sc.ensure(n * sizeof(float)));
  B2_CUDA(ctx, ij.ensure(3 * n * sizeof(int)));
  B2_CUDA(ctx, cand.ensure(n * sizeof(D2Cand)));
  B2_CUDA(ctx, cnt.ensure(sizeof(int)));
  B2_CUDA(ctx, ord.ensure(max_k * sizeof(int)));
  B2_CUDA(ctx, cudaMemcpy(sc.p, scores, n * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, cudaMemcpy(ij.p, cij, 3 * n * sizeof(int), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, cudaMemcpy(cnt.p, &n, sizeof(int), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, cudaMemset(ord.p, 0xff, max_k * sizeof(int)));
  B2_LAUNCH(ctx, k_d2_debug_keys, cdiv(n, 256), 256, 0, ctx->stream, sc.as<float>(), ij.as<int>(), n, cand.as<D2Cand>());
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_d2_rank, cdiv(n, 256), 256, 0, ctx->stream, cand.as<D2Cand>(), cnt.as<int>(), n, max_k, ord.as<int>());
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  B2_CUDA(ctx, cudaMemcpy(order, ord.p, (size_t)(max_k < n ? max_k : n) * sizeof(int), cudaMemcpyDeviceToHost));
  sc.release(), ij.release(), cand.release(), cnt.release(), ord.release();
  return B2_OK;
}
