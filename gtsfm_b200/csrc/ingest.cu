// Image ingest on the device (SURVEY.md section 8f rank 2): the loader's cubic down-size to `max_resolution`
// (gtsfm/utils/images.py:102-129,150-220 -> cv2.resize(INTER_CUBIC), gtsfm/loader/loader_base.py:160-200) so that a decoded
// frame goes H2D once at full size and never returns to the host before detection.  Arithmetic = OpenCV's uint8 cubic
// resize in 11-bit fixed point (A = -0.75, taps rounded to int16, two 4-tap passes in int32, +2^21 >> 22, saturate), as
// restated in oracle/images_ref.py; gray conversion stays in b2_superpoint_*_dev (cv2's fixed-point RGB2GRAY).
// HBM-bound byte work: one thread per output pixel, all channels, 16 clamped source reads per channel served by L1/L2.
#include "common.cuh"

// per destination index: int32 first source index, 4 x int16 weights (12 bytes, padded to 16)
struct CubicTap {
  int s0;
  short w[4];
  int pad;
};

// taps of one axis (cv::resize INTER_CUBIC): fx = (float)((d + 0.5) * scale - 0.5), s = floor(fx), fx -= s, A = -0.75
__global__ void k_cubic_taps(CubicTap* __restrict__ tab, int n_dst, int n_src) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_dst) return;
  const double scale = (double)n_src / (double)n_dst;
  float fx = (float)(((double)d + 0.5) * scale - 0.5);
  const int s = (int)floorf(fx);
  fx = __fsub_rn(fx, (float)s);
  const float A = -0.75f;
  // (no fused multiply-adds: the restatement evaluates every product and sum in float32 separately)
  const float x1 = __fadd_rn(fx, 1.0f);
  const float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), __fmul_rn(5.0f, A)), x1), __fmul_rn(8.0f, A)), x1), __fmul_rn(4.0f, A));
  const float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(A, 2.0f), fx), __fadd_rn(A, 3.0f)), fx), fx), 1.0f);
  const float y = __fsub_rn(1.0f, fx);
  const float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(A, 2.0f), y), __fadd_rn(A, 3.0f)), y), y), 1.0f);
  const float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.0f, c0), c1), c2);
  const float c[4] = {c0, c1, c2, c3};
  CubicTap t;
  t.s0 = s - 1;
  t.pad = 0;
  for (int k = 0; k < 4; ++k) {
    int v = __float2int_rn(__fmul_rn(c[k], 2048.0f));  // saturate_cast<short>: round half to even
    v = v < -32768 ? -32768 : (v > 32767 ? 32767 : v);
    t.w[k] = (short)v;
  }
  tab[d] = t;
}

template <int C>
__global__ void __launch_bounds__(256) k_resize_cubic_u8(const uint8_t* __restrict__ src, int H, int W, size_t pitch, uint8_t* __restrict__ dst,
                                                          int NH, int NW, const CubicTap* __restrict__ xt, const CubicTap* __restrict__ yt) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= NW || y >= NH) return;
  const CubicTap tx = xt[x], ty = yt[y];
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int sy = min(max(ty.s0 + j, 0), H - 1);
    const uint8_t* row = src + (size_t)sy * pitch;
    int hor[C];
#pragma unroll
    for (int c = 0; c < C; ++c) hor[c] = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int sx = min(max(tx.s0 + i, 0), W - 1);
#pragma unroll
      for (int c = 0; c < C; ++c) hor[c] += (int)row[sx * C + c] * (int)tx.w[i];
    }
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] += hor[c] * (int)ty.w[j];
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int v = (acc[c] + (1 << 21)) >> 22;
    dst[((size_t)y * NW + x) * C + c] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
}

extern "C" int b2_image_resize_dev(b2_context* ctx, const uint8_t* src, int height, int width, int channels, size_t pitch, uint8_t* dst,
                                   int new_height, int new_width, void* stream) {
  if (!ctx || !src || !dst || height <= 0 || width <= 0 || new_height <= 0 || new_width <= 0) return B2_ERR_ARG;
  if (channels != 1 && channels != 3 && channels != 4) return b2_fail(ctx, B2_ERR_ARG, "channels must be 1, 3 or 4");
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(ctx, ctx->resize_taps.ensure((size_t)(new_width + new_height) * sizeof(CubicTap)));
  CubicTap* xt = ctx->resize_taps.as<CubicTap>();
  CubicTap* yt = xt + new_width;
  B2_LAUNCH(ctx, k_cubic_taps, cdiv(new_width, 128), 128, 0, st, xt, new_width, width);
  B2_LAUNCH(ctx, k_cubic_taps, cdiv(new_height, 128), 128, 0, st, yt, new_height, height);
  B2_CHECK_LAUNCH(ctx);
  const dim3 grid(cdiv(new_width, 32), cdiv(new_height, 8));
  if (channels == 1) B2_LAUNCH(ctx, k_resize_cubic_u8<1>, grid, 256, 0, st, src, height, width, pitch, dst, new_height, new_width, xt, yt);
  else if (channels == 3) B2_LAUNCH(ctx, k_resize_cubic_u8<3>, grid, 256, 0, st, src, height, width, pitch, dst, new_height, new_width, xt, yt);
  else B2_LAUNCH(ctx, k_resize_cubic_u8<4>, grid, 256, 0, st, src, height, width, pitch, dst, new_height, new_width, xt, yt);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}
