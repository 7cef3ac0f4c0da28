// NetVLAD global image descriptor (SURVEY.md section 8f rank 4: the retrieval front of deep_front_end.yaml:6-15).
// Reference: thirdparty/hloc/netvlad.py:163-193 (forward), :52-75 (NetVLAD layer), :104-113 (VGG16 features[:-2] backbone),
// wrapped by gtsfm/frontend/global_descriptor/netvlad_global_descriptor.py:53-71.
//
//   image (3, H, W) in [0, 1] -> x 255, clamp, - mean -> 13 3x3 convolutions (ReLU after all but the last, 4 max-pools)
//   -> (512, H/16, W/16) -> per-location L2 normalisation -> soft assignment to K = 64 clusters (1x1 projection + softmax)
//   -> sum of assignment-weighted residuals to the centres -> intra-normalisation -> flatten (d major, k minor) -> L2
//   -> whitening Linear(32768 -> 4096) -> L2.
//
// The 12 convolutions with Cin >= 64 run on the SuperPoint convolution kernel (conv_ps.cuh: persistent wgmma implicit GEMM,
// halo reuse, split-fp16 = fp32-equivalent); the soft-assignment projection and the whitening layer run on the shared GEMM
// (gemm_ws.cuh), the latter over a BATCH of images with K = 32768 walked in chunks (see retrieval.cu on the accumulator).
// HBM layout: activations NHWC fp16 hi / lo planes, ping-pong; whitening weights as planes (2 x 268 MB), resident.
#include "common.cuh"
#include "conv_ps.cuh"
#include "linear.cuh"

constexpr int NV_NCONV = 13, NV_D = 512, NV_K = 64, NV_VLAD = NV_D * NV_K, NV_OUT = 4096, NV_KC = 512;
static const int NV_CI[NV_NCONV] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
static const int NV_CO[NV_NCONV] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
static const int NV_POOL[NV_NCONV] = {0, 1, 0, 1, 0, 0, 1, 0, 0, 1, 0, 0, 0};  // MaxPool2d(2, 2) after the layer

struct NetVladState {
  bool loaded = false;
  DevBuf w0, bias, wh, wl, sh, sl, centers, whh, whl, wbias, errflag;  // weights
  float mean[3] = {0, 0, 0};
  size_t woff[NV_NCONV] = {}, boff[NV_NCONV] = {};
  DevBuf actA, actB, feat, xn, xnp, scores, vlad, vh, vl, out;  // work
};

void nv_destroy(b2_context* ctx) {
  delete ctx->nv;
  ctx->nv = nullptr;
}

// conv1_1: 3 -> 64 channels on clamp(image * 255, 0, 255) - mean (netvlad.py:173-177), 3x3, pad 1, bias, ReLU -> planes.
// block = 32 pixels x 8 channel groups of 8; weights [27][64] in shared memory.
__global__ void __launch_bounds__(256) k_nv_conv0(const float* __restrict__ img /*[3][H][W]*/, const float* __restrict__ wt /*[27][64]*/,
                                                  const float* __restrict__ bias, float m0, float m1, float m2, int H, int W,
                                                  __half* __restrict__ oh, __half* __restrict__ ol) {
  __shared__ float ws[27 * 64];
  for (int i = threadIdx.x; i < 27 * 64; i += 256) ws[i] = wt[i];
  __syncthreads();
  const long long pix = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const int cg = threadIdx.x & 7;
  if (pix >= (long long)H * W) return;
  const int y = (int)(pix / W), x = (int)(pix % W);
  const float mean[3] = {m0, m1, m2};
  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = __ldg(bias + cg * 8 + c);
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int yy = y + dy, xx = x + dx;
      const bool in = yy >= 0 && yy < H && xx >= 0 && xx < W;
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        float v = 0.f;  // zero padding applies AFTER the mean subtraction (the convolution pads its input)
        if (in) v = fminf(fmaxf(__ldg(img + ((size_t)ci * H + yy) * W + xx) * 255.0f, 0.0f), 255.0f) - mean[ci];
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

// per-location L2 normalisation of the (cells, 512) feature map (F.normalize(dim=1), netvlad.py:184): fp32 copy + planes
__global__ void __launch_bounds__(256) k_nv_prenorm(const float* __restrict__ feat, int cells, float* __restrict__ xn, __half* __restrict__ ph,
                                                    __half* __restrict__ pl) {
  const int cell = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (cell >= cells) return;
  const float4* p = reinterpret_cast<const float4*>(feat + (size_t)cell * NV_D);
  float4 v[4];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = p[lane + 32 * i];
    ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
  }
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 o = make_float4(v[i].x / nrm, v[i].y / nrm, v[i].z / nrm, v[i].w / nrm);
    const size_t e = (size_t)cell * NV_D + (size_t)(lane + 32 * i) * 4;
    *reinterpret_cast<float4*>(xn + e) = o;
    uint32_t h0, l0, h1, l1;
    tc::split2(o.x, o.y, h0, l0);
    tc::split2(o.z, o.w, h1, l1);
    *reinterpret_cast<uint2*>(ph + e) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(pl + e) = make_uint2(l0, l1);
  }
}

// softmax over the 64 cluster scores of a location (netvlad.py:67), in place: one warp per location
__global__ void __launch_bounds__(256) k_nv_softmax(float* __restrict__ sc, int cells) {
  const int cell = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (cell >= cells) return;
  float* p = sc + (size_t)cell * NV_K;
  const float a = p[lane], b = p[lane + 32];
  const float m = warp_max(fmaxf(a, b));
  const float ea = expf(a - m), eb = expf(b - m);
  const float s = warp_sum(ea + eb);
  p[lane] = ea / s, p[lane + 32] = eb / s;
}

// VLAD aggregation of one image (netvlad.py:68-72): block k, thread d: sum_n s[n][k] (x[n][d] - c[d][k]), then intra-normalisation
// over d, written at d * 64 + k of the image's 32768-vector
__global__ void __launch_bounds__(NV_D) k_nv_vlad(const float* __restrict__ xn, const float* __restrict__ sc, const float* __restrict__ centers,
                                                  int cells, float* __restrict__ vlad) {
  __shared__ float red[NV_D / 32];
  __shared__ float stile[64];
  const int k = blockIdx.x, d = threadIdx.x;
  const float c = centers[(size_t)d * NV_K + k];
  float acc = 0.f;
  for (int n0 = 0; n0 < cells; n0 += 64) {
    __syncthreads();
    if (d < 64) stile[d] = n0 + d < cells ? sc[(size_t)(n0 + d) * NV_K + k] : 0.f;
    __syncthreads();
    const int lim = cells - n0 < 64 ? cells - n0 : 64;
    for (int j = 0; j < lim; ++j) acc = fmaf(stile[j], xn[(size_t)(n0 + j) * NV_D + d] - c, acc);
  }
  const float ss = warp_sum(acc * acc);
  if ((d & 31) == 0) red[d >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < NV_D / 32; ++i) tot += red[i];
  vlad[(size_t)d * NV_K + k] = acc / fmaxf(sqrtf(tot), 1e-12f);
}

// L2 normalisation of a row of `n` floats (one block per row); optionally also written as split planes
__global__ void __launch_bounds__(1024) k_nv_rownorm(const float* __restrict__ in, int n, float* __restrict__ out, __half* __restrict__ ph,
                                                     __half* __restrict__ pl) {
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
  for (int i = threadIdx.x; i < n; i += 1024) {
    const float v = r[i] / nrm;
    if (out) out[(size_t)blockIdx.x * n + i] = v;
    if (ph) {
      __half h, l;
      tc::split_h(v, h, l);
      ph[(size_t)blockIdx.x * n + i] = h, pl[(size_t)blockIdx.x * n + i] = l;
    }
  }
}

// blob: 13 x (conv weight OIHW, bias), score_proj [64][512], centers [512][64], whiten weight [4096][32768], whiten bias [4096], mean [3]
static size_t nv_blob_floats() {
  size_t n = 0;
  for (int l = 0; l < NV_NCONV; ++l) n += (size_t)NV_CO[l] * NV_CI[l] * 9 + NV_CO[l];
  return n + (size_t)NV_K * NV_D + (size_t)NV_D * NV_K + (size_t)NV_OUT * NV_VLAD + NV_OUT + 3;
}

extern "C" size_t b2_netvlad_blob_floats(void) { return nv_blob_floats(); }

extern "C" int b2_netvlad_set_weights(b2_context* ctx, const float* blob, size_t n_floats) {
  if (!ctx || !blob) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (n_floats != nv_blob_floats()) return b2_fail(ctx, B2_ERR_ARG, "netvlad blob must hold " + std::to_string(nv_blob_floats()) + " floats, got " + std::to_string(n_floats));
  if (!tma_encoder()) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled is not available (driver too old?)");
  cudaSetDevice(ctx->device);
  if (!ctx->nv) ctx->nv = new NetVladState();
  NetVladState* s = ctx->nv;
  // convolution weights: layer 0 as fp32 [tap][ci][co]; layers 1..12 as [co][tap * Cin + ci] planes; biases concatenated
  std::vector<float> stage, b, w0;
  size_t src = conv_ps_repack(blob, NV_NCONV, NV_CI, NV_CO, stage, b, w0, s->woff, s->boff);
  const size_t btot = b.size();
  DevBuf tmp;
  const size_t piece = (size_t)64 << 20;  // floats per staging piece of the device-side split
  B2_CUDA(ctx, tmp.ensure(piece * sizeof(float)));
  auto split_to = [&](const float* host, size_t n, DevBuf& h, DevBuf& l) { return conv_ps_upload_planes(host, n, h, l, tmp, piece); };
  B2_CUDA(ctx, split_to(stage.data(), stage.size(), s->wh, s->wl));
  B2_CUDA(ctx, s->w0.ensure(w0.size() * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->w0.p, w0.data(), w0.size() * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, s->bias.ensure(btot * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->bias.p, b.data(), btot * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(ctx, split_to(blob + src, (size_t)NV_K * NV_D, s->sh, s->sl));  // score_proj [64][512]
  src += (size_t)NV_K * NV_D;
  B2_CUDA(ctx, s->centers.ensure((size_t)NV_D * NV_K * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->centers.p, blob + src, (size_t)NV_D * NV_K * sizeof(float), cudaMemcpyHostToDevice));
  src += (size_t)NV_D * NV_K;
  B2_CUDA(ctx, split_to(blob + src, (size_t)NV_OUT * NV_VLAD, s->whh, s->whl));  // whitening [4096][32768]
  src += (size_t)NV_OUT * NV_VLAD;
  B2_CUDA(ctx, s->wbias.ensure(NV_OUT * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpy(s->wbias.p, blob + src, NV_OUT * sizeof(float), cudaMemcpyHostToDevice));
  src += NV_OUT;
  s->mean[0] = blob[src], s->mean[1] = blob[src + 1], s->mean[2] = blob[src + 2];
  tmp.release();
  B2_CUDA(ctx, s->errflag.ensure(16));
  B2_CUDA(ctx, cudaMemset(s->errflag.p, 0, 16));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_conv_ps<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CP_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  s->loaded = true;
  return B2_OK;
}

static int nv_conv(b2_context* ctx, cudaStream_t st, const DevBuf& in, int l, int H, int W, DevBuf* out_planes, float* out_f32) {
  NetVladState* s = ctx->nv;
  return conv_ps_run(ctx, st, in.as<__half>(), H, W, NV_CI[l], NV_CO[l], NV_POOL[l], l != NV_NCONV - 1, 1, s->wh.as<__half>() + s->woff[l],
                     s->wl.as<__half>() + s->woff[l], s->bias.as<float>() + s->boff[l], out_planes ? out_planes->as<__half>() : nullptr, out_f32,
                     s->errflag.as<int>(), "netvlad");
}

// images: DEVICE [B][3][H][W] fp32 in [0, 1] (what the reference's batch transform produces); out: DEVICE [B][4096] fp32
extern "C" int b2_netvlad_describe_dev(b2_context* ctx, const float* images, int B, int H, int W, float* out, void* stream) {
  if (!ctx || !images || !out || B <= 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  NetVladState* s = ctx->nv;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "netvlad weights not set");
  if (H < 16 || W < 16) return b2_fail(ctx, B2_ERR_ARG, "netvlad needs images of at least 16 x 16 pixels (four 2x2 max-pools)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t px = (size_t)H * W;
  int h = H, w = W;
  for (int l = 0; l < NV_NCONV; ++l)
    if (NV_POOL[l]) h /= 2, w /= 2;
  const int cells = h * w;
  B2_CUDA(ctx, s->actA.ensure(px * 64 * 2 * sizeof(__half)));
  B2_CUDA(ctx, s->actB.ensure(px * 64 * 2 * sizeof(__half)));  // largest output of the second buffer: conv1_2's input size is the bound
  B2_CUDA(ctx, s->feat.ensure((size_t)cells * NV_D * sizeof(float)));
  B2_CUDA(ctx, s->xn.ensure((size_t)cells * NV_D * sizeof(float)));
  B2_CUDA(ctx, s->xnp.ensure((size_t)cells * NV_D * 2 * sizeof(__half)));
  B2_CUDA(ctx, s->scores.ensure((size_t)cells * NV_K * sizeof(float)));
  B2_CUDA(ctx, s->vlad.ensure((size_t)B * NV_VLAD * sizeof(float)));
  B2_CUDA(ctx, s->vh.ensure((size_t)B * NV_VLAD * sizeof(__half)));
  B2_CUDA(ctx, s->vl.ensure((size_t)B * NV_VLAD * sizeof(__half)));
  B2_CUDA(ctx, s->out.ensure((size_t)B * NV_OUT * sizeof(float)));
  B2_CUDA(ctx, cudaMemsetAsync(s->errflag.p, 0, 16, st));
  TcWeights tw{nullptr, nullptr, nullptr, s->errflag.as<int>(), true};
  tw.sm_count = ctx->sm_count;
  int rc;
  for (int b = 0; b < B; ++b) {
    const float* img = images + (size_t)b * 3 * px;
    __half* a0 = s->actA.as<__half>();
    B2_LAUNCH(ctx, k_nv_conv0, (unsigned)((px + 31) / 32), 256, 0, st, img, s->w0.as<float>(), s->bias.as<float>(), s->mean[0], s->mean[1], s->mean[2],
              H, W, a0, a0 + px * 64);
    B2_CHECK_LAUNCH(ctx);
    DevBuf* cur = &s->actA;
    DevBuf* nxt = &s->actB;
    int ch = H, cw = W;
    for (int l = 1; l < NV_NCONV; ++l) {
      const bool last = l == NV_NCONV - 1;
      if ((rc = nv_conv(ctx, st, *cur, l, ch, cw, last ? nullptr : nxt, last ? s->feat.as<float>() : nullptr))) return rc;
      if (NV_POOL[l]) ch /= 2, cw /= 2;
      std::swap(cur, nxt);
    }
    // NetVLAD layer
    __half* xh = s->xnp.as<__half>();
    B2_LAUNCH(ctx, k_nv_prenorm, cdiv(cells, 8), 256, 0, st, s->feat.as<float>(), cells, s->xn.as<float>(), xh, xh + (size_t)cells * NV_D);
    B2_CHECK_LAUNCH(ctx);
    LinArgs a;
    a.a1p = {xh, xh + (size_t)cells * NV_D}, a.lda1 = NV_D, a.K1 = NV_D;
    a.bp = {s->sh.as<__half>(), s->sl.as<__half>()}, a.ldb = NV_D;
    a.cf = s->scores.as<float>(), a.ldc = NV_K, a.tc_want_f32 = true, a.M = cells, a.N = NV_K;
    if ((rc = run_linear(ctx, st, tw, &a, 1))) return rc;
    B2_LAUNCH(ctx, k_nv_softmax, cdiv(cells, 8), 256, 0, st, s->scores.as<float>(), cells);
    B2_CHECK_LAUNCH(ctx);
    B2_LAUNCH(ctx, k_nv_vlad, NV_K, NV_D, 0, st, s->xn.as<float>(), s->scores.as<float>(), s->centers.as<float>(), cells,
              s->vlad.as<float>() + (size_t)b * NV_VLAD);
    B2_CHECK_LAUNCH(ctx);
  }
  // global L2 normalisation of the VLAD vectors -> planes; whitening over the whole batch; final normalisation
  B2_LAUNCH(ctx, k_nv_rownorm, B, 1024, 0, st, s->vlad.as<float>(), NV_VLAD, (float*)nullptr, s->vh.as<__half>(), s->vl.as<__half>());
  B2_CHECK_LAUNCH(ctx);
  for (int kc = 0; kc < NV_VLAD; kc += NV_KC) {
    LinArgs a;
    a.a1p = {s->vh.as<__half>() + kc, s->vl.as<__half>() + kc}, a.lda1 = NV_VLAD, a.K1 = NV_KC;
    a.bp = {s->whh.as<__half>() + kc, s->whl.as<__half>() + kc}, a.ldb = NV_VLAD;
    a.cf = s->out.as<float>(), a.ldc = NV_OUT, a.tc_want_f32 = true, a.M = B, a.N = NV_OUT;
    if (kc == 0) a.bias = s->wbias.as<float>();
    else a.resid = s->out.as<float>(), a.ldr = NV_OUT;
    if ((rc = run_linear(ctx, st, tw, &a, 1))) return rc;
  }
  B2_LAUNCH(ctx, k_nv_rownorm, B, 1024, 0, st, s->out.as<float>(), NV_OUT, out, (__half*)nullptr, (__half*)nullptr);
  B2_CHECK_LAUNCH(ctx);
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&err, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

// HOST buffers in / out (images [B][3][H][W] fp32 in [0, 1], out [B][4096])
extern "C" int b2_netvlad_describe_host(b2_context* ctx, const float* images, int B, int H, int W, float* out) {
  if (!ctx || !images || !out || B <= 0 || H <= 0 || W <= 0) return B2_ERR_ARG;
  DevBuf in_d, out_d;
  const size_t nin = (size_t)B * 3 * H * W * sizeof(float), nout = (size_t)B * NV_OUT * sizeof(float);
  cudaSetDevice(ctx->device);
  B2_CUDA(ctx, in_d.ensure(nin));
  B2_CUDA(ctx, out_d.ensure(nout));
  B2_CUDA(ctx, cudaMemcpy(in_d.p, images, nin, cudaMemcpyHostToDevice));
  const int rc = b2_netvlad_describe_dev(ctx, in_d.as<float>(), B, H, W, out_d.as<float>(), ctx->stream);
  if (rc != B2_OK) return rc;
  B2_CUDA(ctx, cudaMemcpy(out, out_d.p, nout, cudaMemcpyDeviceToHost));
  return B2_OK;
}
