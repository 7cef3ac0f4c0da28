// SIFT detector-descriptor for sm_90a: cv2.SIFT_create() with its defaults (nOctaveLayers 3, contrastThreshold 0.04,
// edgeThreshold 10, sigma 1.6, firstOctave -1, no precise upscale) restated, uint8 descriptors.
//
// Reference semantics: gtsfm/frontend/detector_descriptor/sift.py:27-55 (gray conversion, cv2 detectAndCompute, top-k),
// which runs OpenCV's sift.simd.hpp.  oracle/sift_ref.py restates the pyramid with cv2 calls.
//
// Stages of one batch of same-shape images (every stage is one launch over the batch, blockIdx.z / .y = image):
//   k_sift_blur<1>   gray + 2x INTER_LINEAR upsample + Gaussian blur (sigma sqrt(1.6^2 - 1)) -> octave 0, level 0
//   k_sift_down      level 0 of octave o > 0 = every second pixel of level 3 of octave o - 1 (INTER_NEAREST)
//   k_sift_blur<0>   level i = blur(level i - 1), separable float, both passes fused in shared memory, BORDER_REFLECT_101
//   k_sift_extrema   DoG formed on the fly (G[i+1] - G[i], the same float subtraction cv2 stores), 26-neighbour extrema of
//                    layers 1..3, quadratic refinement, contrast and edge tests -> candidate list
//   k_sift_orient    warp per candidate: 36-bin orientation histogram, one keypoint per peak -> raw keypoint list
//   k_sift_rank      rank of every keypoint in cv2's KeyPoint order (all-pairs comparison) -> sorted list
//   k_sift_compact   drop consecutive duplicates, halve (firstOctave -1), apply the mask -> final list (what cv2 returns)
//   k_sift_topk      the max_keypoints largest responses, ties to the lower index, order kept (topk.cuh)
//   k_sift_describe  warp per selected keypoint: 4x4x8 descriptor, clip, normalise, saturate to uint8
// The lists are appended with integer atomics (their order varies run to run); the rank sort makes the output a function
// of the keypoint values only, so results are identical run to run and between batched and single-image calls.
//
// Workspace per image: the Gaussian pyramid, 6 levels x (4/3) x (2H x 2W) floats = 128 H W bytes, plus the keypoint lists,
// (4 H W / 32) x (32 + 2 x 3 x 24 + 8) bytes = 23 H W bytes.  Images are limited to SF_MAX_PIXELS = 2^24 pixels
// (e.g. 4096 x 4096, 2.5 GB of workspace) and a side of at most 16384; a batch holds at most SF_MAX_BATCH images.
#include <float.h>
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "image.cuh"
#include "topk.cuh"

namespace {

constexpr int SF_LAYERS = 3;              // nOctaveLayers
constexpr int SF_LEVELS = SF_LAYERS + 3;  // Gaussian levels per octave
constexpr int SF_BORDER = 5;              // SIFT_IMG_BORDER
constexpr int SF_MAX_OCT = 16;
constexpr int SF_MAX_R = 16;  // largest blur radius the tile supports (the default sigmas need 13)
constexpr int SF_TW = 64, SF_TH = 32;
constexpr int SF_ORI_BINS = 36;
constexpr int SF_D = 4, SF_N = 8, SF_DESC = SF_D * SF_D * SF_N;
constexpr int SF_HLEN = (SF_D + 2) * (SF_D + 2) * (SF_N + 2);  // 360 histogram cells incl. the interpolation borders
constexpr int SF_HPITCH = SF_HLEN + 1;                          // lane-private histograms: odd pitch, no bank conflicts
constexpr int SF_MAX_PIXELS = 1 << 24;
constexpr int SF_MAX_SIDE = 16384;
constexpr int SF_MAX_BATCH = 64;
constexpr float SF_SIGMA = 1.6f, SF_CONTRAST = 0.04f, SF_EDGE = 10.f;
enum { SC_CAND = 0, SC_RAW, SC_FIN, SC_DEDUP, SC_SEL, SC_N = 8 };

}  // namespace

struct SfImg {  // device table row of one image
  const uint8_t* img;
  const uint8_t* mask;
  b2_sift_keypoint* out_kp;
  uint8_t* out_desc;
  int max_kp;
  int pad;
};

struct SfCand {  // refined extremum before orientation assignment (octave-0 = doubled-image coordinates)
  float x, y, size, response;
  int octave;  // cv2's packed octave before the firstOctave shift: o + (layer << 8) + (xi byte << 16)
  int o, r, c;
};

struct SfTaps {
  int r;
  float k[2 * SF_MAX_R + 1];
};

struct SiftState {
  DevBuf pyr, cand, raw, sorted, fin, fresp, sel, counts, table, img, mask, okp, odesc;
};

void sf_destroy(b2_context* ctx) {
  delete ctx->sf;
  ctx->sf = nullptr;
}

// ------------------------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------------------------
// cv2 borderInterpolate(p, len, BORDER_REFLECT_101)
__device__ __forceinline__ int sf_reflect(int p, int len) {
  if (len == 1) return 0;
  while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// cv2 hal::fastAtan2 (degrees, [0, 360))
__device__ __forceinline__ float sf_atan(float y, float x) {
  const float p1 = 0.9997878412794807f * (float)(180 / M_PI), p3 = -0.3258083974640975f * (float)(180 / M_PI);
  const float p5 = 0.1555786518463281f * (float)(180 / M_PI), p7 = -0.04432655554792128f * (float)(180 / M_PI);
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + (float)DBL_EPSILON);
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + (float)DBL_EPSILON);
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}

// cv2 KeyPoint order used by KeyPointsFilter::removeDuplicatedSorted
__device__ __forceinline__ bool sf_less(const b2_sift_keypoint& a, const b2_sift_keypoint& b) {
  if (a.x != b.x) return a.x < b.x;
  if (a.y != b.y) return a.y < b.y;
  if (a.size != b.size) return a.size > b.size;
  if (a.angle != b.angle) return a.angle < b.angle;
  if (a.response != b.response) return a.response > b.response;
  return a.octave > b.octave;
}
__device__ __forceinline__ bool sf_same(const b2_sift_keypoint& a, const b2_sift_keypoint& b) {
  return a.x == b.x && a.y == b.y && a.size == b.size && a.angle == b.angle && a.response == b.response && a.octave == b.octave;
}

// exclusive prefix of `flag` over a 1024-thread block; *total = number of set flags.  All threads must call.
__device__ __forceinline__ int sf_block_scan(bool flag, int* wtot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) wtot[warp] = __popc(m);
  __syncthreads();
  if (warp == 0) {
    int w = wtot[lane], ws = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int u = __shfl_up_sync(0xffffffffu, ws, o);
      if (lane >= o) ws += u;
    }
    wtot[lane] = ws - w;
    if (lane == 31) wtot[32] = ws;
  }
  __syncthreads();
  const int pos = wtot[warp] + __popc(m & ((1u << lane) - 1));
  *total = wtot[32];
  __syncthreads();
  return pos;
}

// ------------------------------------------------------------------------------------------------------------------
// pyramid
// ------------------------------------------------------------------------------------------------------------------
struct SfBlurArgs {
  const float* src;  // MODE 0: source level of image 0; image b at src + b * stride
  const SfImg* imgs; // MODE 1: the uint8 images
  int channels, in_w, in_h;
  size_t pitch;
  float* dst;
  size_t stride;  // floats between two images' pyramids
  int w, h;       // level size
  SfTaps t;
};

// One 64 x 32 output tile: load the (32 + 2r) x (64 + 2r) input window (reflected), row pass into shared memory, column
// pass to global.  Row sums run over the taps left to right, column sums as centre + symmetric pairs (cv2's RowFilter
// and SymmColumnFilter).  MODE 1 forms the input on the fly: gray, then cv2's 2x INTER_LINEAR upsample, which is exact
// in float for integer input.
template <int MODE>
__global__ void __launch_bounds__(256) k_sift_blur(SfBlurArgs a) {
  __shared__ float in[(SF_TH + 2 * SF_MAX_R) * (SF_TW + 2 * SF_MAX_R)];
  __shared__ float mid[(SF_TH + 2 * SF_MAX_R) * SF_TW];
  const int b = blockIdx.z, r = a.t.r;
  const int x0 = blockIdx.x * SF_TW, y0 = blockIdx.y * SF_TH;
  const int iw = SF_TW + 2 * r, ih = SF_TH + 2 * r;
  const float* src = MODE == 0 ? a.src + (size_t)b * a.stride : nullptr;
  for (int i = threadIdx.x; i < iw * ih; i += blockDim.x) {
    const int yy = sf_reflect(y0 - r + i / iw, a.h), xx = sf_reflect(x0 - r + i % iw, a.w);
    float v;
    if (MODE == 0) {
      v = __ldg(src + (size_t)yy * a.w + xx);
    } else {
      const SfImg& im = a.imgs[b];
      // resize INTER_LINEAR, scale 2: fx = (x + 0.5) / 2 - 0.5, clamped at both borders
      float fx = xx * 0.5f - 0.25f, fy = yy * 0.5f - 0.25f;
      int sx = (int)floorf(fx), sy = (int)floorf(fy);
      fx -= sx, fy -= sy;
      if (sx < 0) sx = 0, fx = 0.f;
      if (sx >= a.in_w - 1) sx = a.in_w - 1, fx = 0.f;
      if (sy < 0) sy = 0, fy = 0.f;
      if (sy >= a.in_h - 1) sy = a.in_h - 1, fy = 0.f;
      const int sx1 = fx > 0.f ? sx + 1 : sx, sy1 = fy > 0.f ? sy + 1 : sy;
      const uint8_t* p0 = im.img + (size_t)sy * a.pitch;
      const uint8_t* p1 = im.img + (size_t)sy1 * a.pitch;
      const int c = a.channels;
      const float g00 = b2_gray_u8(p0 + (size_t)sx * c, c), g01 = b2_gray_u8(p0 + (size_t)sx1 * c, c);
      const float g10 = b2_gray_u8(p1 + (size_t)sx * c, c), g11 = b2_gray_u8(p1 + (size_t)sx1 * c, c);
      v = (g00 * (1.f - fx) + g01 * fx) * (1.f - fy) + (g10 * (1.f - fx) + g11 * fx) * fy;
    }
    in[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SF_TW * ih; i += blockDim.x) {
    const int y = i / SF_TW, x = i % SF_TW;
    const float* p = in + y * iw + x;
    float s = 0.f;
    for (int t = 0; t <= 2 * r; ++t) s = fmaf(a.t.k[t], p[t], s);
    mid[y * SF_TW + x] = s;
  }
  __syncthreads();
  float* dst = a.dst + (size_t)b * a.stride;
  for (int i = threadIdx.x; i < SF_TW * SF_TH; i += blockDim.x) {
    const int y = i / SF_TW, x = i % SF_TW;
    if (y0 + y >= a.h || x0 + x >= a.w) continue;
    const float* p = mid + (y + r) * SF_TW + x;
    float s = a.t.k[r] * p[0];
    for (int j = 1; j <= r; ++j) s = fmaf(a.t.k[r + j], p[j * SF_TW] + p[-j * SF_TW], s);
    dst[(size_t)(y0 + y) * a.w + x0 + x] = s;
  }
}

__global__ void __launch_bounds__(256) k_sift_down(const float* __restrict__ src, int sw, float* __restrict__ dst, int w, int h,
                                                    size_t stride) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const size_t off = (size_t)blockIdx.z * stride;
  dst[off + (size_t)y * w + x] = src[off + (size_t)(2 * y) * sw + 2 * x];
}

// ------------------------------------------------------------------------------------------------------------------
// extrema, refinement, orientation
// ------------------------------------------------------------------------------------------------------------------
struct SfOctArgs {
  const float* g;  // level 0 of this octave, image 0; level l at g + l * P, image b at + b * stride
  size_t P, stride;
  int w, h, o;
  SfCand* cand;
  b2_sift_keypoint* raw;
  int* counts;  // [image][SC_N]
  int cand_cap, kp_cap;
};

struct SfDog {
  const float* g;
  size_t P;
  int w;
  __device__ __forceinline__ float operator()(int l, int r, int c) const {
    const size_t i = (size_t)r * w + c;
    return __ldg(g + (size_t)(l + 1) * P + i) - __ldg(g + (size_t)l * P + i);
  }
};

// sift.simd.hpp adjustLocalExtrema: up to 5 Newton steps of the 3-D quadratic fit (the 3x3 system solved by Cramer's rule,
// as Matx33f::solve(DECOMP_LU) does), then the contrast and edge tests.
__device__ bool sf_adjust(const SfDog& D, int w, int h, int o, int layer, int r, int c, SfCand& out) {
  const float img_scale = 1.f / 255.f, deriv_scale = img_scale * 0.5f, second_scale = img_scale, cross_scale = img_scale * 0.25f;
  float xi = 0.f, xr = 0.f, xc = 0.f;
  int i = 0;
  for (; i < 5; ++i) {
    const float dx = (D(layer, r, c + 1) - D(layer, r, c - 1)) * deriv_scale;
    const float dy = (D(layer, r + 1, c) - D(layer, r - 1, c)) * deriv_scale;
    const float ds = (D(layer + 1, r, c) - D(layer - 1, r, c)) * deriv_scale;
    const float v2 = D(layer, r, c) * 2.f;
    const float dxx = (D(layer, r, c + 1) + D(layer, r, c - 1) - v2) * second_scale;
    const float dyy = (D(layer, r + 1, c) + D(layer, r - 1, c) - v2) * second_scale;
    const float dss = (D(layer + 1, r, c) + D(layer - 1, r, c) - v2) * second_scale;
    const float dxy = (D(layer, r + 1, c + 1) - D(layer, r + 1, c - 1) - D(layer, r - 1, c + 1) + D(layer, r - 1, c - 1)) * cross_scale;
    const float dxs = (D(layer + 1, r, c + 1) - D(layer + 1, r, c - 1) - D(layer - 1, r, c + 1) + D(layer - 1, r, c - 1)) * cross_scale;
    const float dys = (D(layer + 1, r + 1, c) - D(layer + 1, r - 1, c) - D(layer - 1, r + 1, c) + D(layer - 1, r - 1, c)) * cross_scale;
    const float a00 = dxx, a01 = dxy, a02 = dxs, a10 = dxy, a11 = dyy, a12 = dys, a20 = dxs, a21 = dys, a22 = dss;
    const float b0 = dx, b1 = dy, b2 = ds;
    float det = a00 * (a11 * a22 - a21 * a12) - a01 * (a10 * a22 - a20 * a12) + a02 * (a10 * a21 - a20 * a11);
    float X0 = 0.f, X1 = 0.f, X2 = 0.f;
    if (det != 0.f) {
      det = 1.f / det;
      X0 = det * (b0 * (a11 * a22 - a12 * a21) - a01 * (b1 * a22 - a12 * b2) + a02 * (b1 * a21 - a11 * b2));
      X1 = det * (a00 * (b1 * a22 - a12 * b2) - b0 * (a10 * a22 - a12 * a20) + a02 * (a10 * b2 - b1 * a20));
      X2 = det * (a00 * (a11 * b2 - b1 * a21) - a01 * (a10 * b2 - b1 * a20) + b0 * (a10 * a21 - a11 * a20));
    }
    xi = -X2, xr = -X1, xc = -X0;
    if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
    const float big = (float)(INT_MAX / 3);
    if (!(fabsf(xi) <= big && fabsf(xr) <= big && fabsf(xc) <= big)) return false;
    c += __float2int_rn(xc);
    r += __float2int_rn(xr);
    layer += __float2int_rn(xi);
    if (layer < 1 || layer > SF_LAYERS || c < SF_BORDER || c >= w - SF_BORDER || r < SF_BORDER || r >= h - SF_BORDER) return false;
  }
  if (i >= 5) return false;
  const float dx = (D(layer, r, c + 1) - D(layer, r, c - 1)) * deriv_scale;
  const float dy = (D(layer, r + 1, c) - D(layer, r - 1, c)) * deriv_scale;
  const float ds = (D(layer + 1, r, c) - D(layer - 1, r, c)) * deriv_scale;
  const float t = dx * xc + dy * xr + ds * xi;
  const float v = D(layer, r, c);
  const float contr = v * img_scale + t * 0.5f;
  if (fabsf(contr) * SF_LAYERS < SF_CONTRAST) return false;
  const float v2 = v * 2.f;
  const float dxx = (D(layer, r, c + 1) + D(layer, r, c - 1) - v2) * second_scale;
  const float dyy = (D(layer, r + 1, c) + D(layer, r - 1, c) - v2) * second_scale;
  const float dxy = (D(layer, r + 1, c + 1) - D(layer, r + 1, c - 1) - D(layer, r - 1, c + 1) + D(layer, r - 1, c - 1)) * cross_scale;
  const float tr = dxx + dyy, det = dxx * dyy - dxy * dxy;
  if (det <= 0.f || tr * tr * SF_EDGE >= (SF_EDGE + 1) * (SF_EDGE + 1) * det) return false;
  const float scale = (float)(1 << o);
  out.x = ((float)c + xc) * scale;
  out.y = ((float)r + xr) * scale;
  out.octave = o + (layer << 8) + (__double2int_rn(((double)xi + 0.5) * 255.0) << 16);
  out.size = SF_SIGMA * powf(2.f, ((float)layer + xi) / SF_LAYERS) * scale * 2.f;
  out.response = fabsf(contr);
  out.o = o, out.r = r, out.c = c;
  return true;
}

// thread per pixel of [5, h - 5) x [5, w - 5), layers 1..3; |DoG| > floor(0.5 * 0.04 / 3 * 255) = 1
__global__ void __launch_bounds__(256) k_sift_extrema(SfOctArgs a) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x + SF_BORDER, r = blockIdx.y + SF_BORDER, b = blockIdx.z;
  if (c >= a.w - SF_BORDER) return;
  const SfDog D{a.g + (size_t)b * a.stride, a.P, a.w};
  const float thr = 1.f;
  for (int l = 1; l <= SF_LAYERS; ++l) {
    const float v = D(l, r, c);
    if (!(fabsf(v) > thr)) continue;
    bool ext = true;
    for (int dl = -1; dl <= 1 && ext; ++dl)
      for (int dr = -1; dr <= 1 && ext; ++dr)
        for (int dc = -1; dc <= 1; ++dc) {
          if (!dl && !dr && !dc) continue;
          const float u = D(l + dl, r + dr, c + dc);
          if (v > 0.f ? u > v : u < v) {
            ext = false;
            break;
          }
        }
    if (!ext) continue;
    SfCand k;
    if (!sf_adjust(D, a.w, a.h, a.o, l, r, c, k)) continue;
    const int slot = atomicAdd(a.counts + b * SC_N + SC_CAND, 1);
    if (slot < a.cand_cap) a.cand[(size_t)b * a.cand_cap + slot] = k;
  }
}

// warp per candidate of this octave: calcOrientationHist (square window of radius round(4.5 scl), Gaussian weight
// sigma 1.5 scl, bin round(ori / 10)), [1 4 6 4 1] / 16 circular smoothing, one keypoint per peak >= 0.8 max.
// Lane-private histograms summed in lane order keep the result independent of scheduling.
constexpr int SF_OR_WARPS = 4;
__global__ void __launch_bounds__(32 * SF_OR_WARPS) k_sift_orient(SfOctArgs a) {
  __shared__ float lh[SF_OR_WARPS][32][SF_ORI_BINS + 1];
  __shared__ float hs[SF_OR_WARPS][SF_ORI_BINS];
  const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5, b = blockIdx.y;
  const int n = min(a.counts[b * SC_N + SC_CAND], a.cand_cap);
  const float* gb = a.g + (size_t)b * a.stride;
  for (int ci = blockIdx.x * SF_OR_WARPS + wq; ci < n; ci += gridDim.x * SF_OR_WARPS) {
    const SfCand k = a.cand[(size_t)b * a.cand_cap + ci];
    if (k.o != a.o) continue;
    const int layer = (k.octave >> 8) & 255;
    const float* G = gb + (size_t)layer * a.P;
    const float scl = k.size * 0.5f / (float)(1 << a.o);
    const int rad = __float2int_rn(4.5f * scl);
    const float sigma = 1.5f * scl, expf_scale = -1.f / (2.f * sigma * sigma);
    for (int j = 0; j < SF_ORI_BINS; ++j) lh[wq][lane][j] = 0.f;
    const int side = 2 * rad + 1;
    for (int s = lane; s < side * side; s += 32) {
      const int i = s / side - rad, j = s % side - rad;
      const int y = k.r + i, x = k.c + j;
      if (y <= 0 || y >= a.h - 1 || x <= 0 || x >= a.w - 1) continue;
      const float dx = G[(size_t)y * a.w + x + 1] - G[(size_t)y * a.w + x - 1];
      const float dy = G[(size_t)(y - 1) * a.w + x] - G[(size_t)(y + 1) * a.w + x];
      const float wgt = expf((float)(i * i + j * j) * expf_scale);
      const float ori = sf_atan(dy, dx), mag = sqrtf(dx * dx + dy * dy);
      int bin = __float2int_rn((SF_ORI_BINS / 360.f) * ori);
      if (bin >= SF_ORI_BINS) bin -= SF_ORI_BINS;
      if (bin < 0) bin += SF_ORI_BINS;
      lh[wq][lane][bin] += wgt * mag;
    }
    __syncwarp();
    for (int j = lane; j < SF_ORI_BINS; j += 32) {
      float t = 0.f;
      for (int l = 0; l < 32; ++l) t += lh[wq][l][j];
      hs[wq][j] = t;
    }
    __syncwarp();
    if (lane == 0) {
      const float* t = hs[wq];
      float hist[SF_ORI_BINS];
      float mx = 0.f;
      for (int j = 0; j < SF_ORI_BINS; ++j) {
        const int m2 = (j + SF_ORI_BINS - 2) % SF_ORI_BINS, m1 = (j + SF_ORI_BINS - 1) % SF_ORI_BINS;
        const int p1 = (j + 1) % SF_ORI_BINS, p2 = (j + 2) % SF_ORI_BINS;
        hist[j] = (t[m2] + t[p2]) * (1.f / 16.f) + (t[m1] + t[p1]) * (4.f / 16.f) + t[j] * (6.f / 16.f);
        mx = j ? fmaxf(mx, hist[j]) : hist[j];
      }
      const float mag_thr = mx * 0.8f;
      for (int j = 0; j < SF_ORI_BINS; ++j) {
        const int l = j > 0 ? j - 1 : SF_ORI_BINS - 1, r2 = j < SF_ORI_BINS - 1 ? j + 1 : 0;
        if (hist[j] > hist[l] && hist[j] > hist[r2] && hist[j] >= mag_thr) {
          float bin = j + 0.5f * (hist[l] - hist[r2]) / (hist[l] - 2 * hist[j] + hist[r2]);
          bin = bin < 0 ? SF_ORI_BINS + bin : bin >= SF_ORI_BINS ? bin - SF_ORI_BINS : bin;
          float angle = 360.f - (360.f / SF_ORI_BINS) * bin;
          if (fabsf(angle - 360.f) < FLT_EPSILON) angle = 0.f;
          const int slot = atomicAdd(a.counts + b * SC_N + SC_RAW, 1);
          if (slot < a.kp_cap) a.raw[(size_t)b * a.kp_cap + slot] = {k.x, k.y, k.size, angle, k.response, k.octave};
        }
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------------------
// order, de-duplication, mask, top-k
// ------------------------------------------------------------------------------------------------------------------
struct SfListArgs {
  const SfImg* imgs;
  b2_sift_keypoint *raw, *sorted, *fin;
  float* fresp;
  int* sel;
  int* counts;
  int kp_cap, W, H;
};

// sorted[rank(i)] = raw[i], rank = #{j : raw[j] before raw[i]} + #{j < i : raw[j] equal to raw[i]}
constexpr int SF_RANK_T = 256;
__global__ void __launch_bounds__(SF_RANK_T) k_sift_rank(SfListArgs a) {
  __shared__ b2_sift_keypoint tile[SF_RANK_T];
  const int b = blockIdx.y;
  const int n = min(a.counts[b * SC_N + SC_RAW], a.kp_cap);
  const b2_sift_keypoint* raw = a.raw + (size_t)b * a.kp_cap;
  for (int base = blockIdx.x * SF_RANK_T; base < n; base += gridDim.x * SF_RANK_T) {
    const int i = base + threadIdx.x;
    b2_sift_keypoint me{};
    if (i < n) me = raw[i];
    int rank = 0;
    for (int t0 = 0; t0 < n; t0 += SF_RANK_T) {
      __syncthreads();
      if (t0 + threadIdx.x < n) tile[threadIdx.x] = raw[t0 + threadIdx.x];
      __syncthreads();
      const int m = min(SF_RANK_T, n - t0);
      if (i < n)
        for (int j = 0; j < m; ++j) rank += sf_less(tile[j], me) || (t0 + j < i && sf_same(tile[j], me));
    }
    if (i < n) a.sorted[(size_t)b * a.kp_cap + rank] = me;
  }
}

// one CTA per image: keep an entry unless it equals its predecessor in (x, y, size, angle); halve pt and size and lower the
// octave byte (firstOctave -1); then cv2's runByPixelsMask: keep where mask[(int)(y + 0.5)][(int)(x + 0.5)] != 0.
__global__ void __launch_bounds__(1024) k_sift_compact(SfListArgs a) {
  __shared__ int wtot[33];
  __shared__ int carry, carry_dd;
  const int b = blockIdx.x;
  const int n = min(a.counts[b * SC_N + SC_RAW], a.kp_cap);
  const b2_sift_keypoint* s = a.sorted + (size_t)b * a.kp_cap;
  const uint8_t* mask = a.imgs[b].mask;
  if (threadIdx.x == 0) carry = 0, carry_dd = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    bool dd = false, keep = false;
    b2_sift_keypoint k{};
    if (i < n) {
      k = s[i];
      dd = i == 0 || !(s[i - 1].x == k.x && s[i - 1].y == k.y && s[i - 1].size == k.size && s[i - 1].angle == k.angle);
      k.x *= 0.5f, k.y *= 0.5f, k.size *= 0.5f;
      k.octave = (k.octave & ~255) | ((k.octave - 1) & 255);
      keep = dd;
      if (dd && mask) {
        const int my = min(max((int)(k.y + 0.5f), 0), a.H - 1), mx = min(max((int)(k.x + 0.5f), 0), a.W - 1);
        keep = mask[(size_t)my * a.W + mx] != 0;
      }
    }
    int tot_dd, tot;
    sf_block_scan(dd, wtot, &tot_dd);
    const int pos = sf_block_scan(keep, wtot, &tot) + carry;
    if (keep) {
      a.fin[(size_t)b * a.kp_cap + pos] = k;
      a.fresp[(size_t)b * a.kp_cap + pos] = k.response;
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tot, carry_dd += tot_dd;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    a.counts[b * SC_N + SC_FIN] = carry;
    a.counts[b * SC_N + SC_DEDUP] = carry_dd;
  }
}

__global__ void __launch_bounds__(1024) k_sift_topk(SfListArgs a) {
  const int b = blockIdx.x;
  const int n = a.counts[b * SC_N + SC_FIN], k = a.imgs[b].max_kp;
  b2_topk_select_cta(a.fresp + (size_t)b * a.kp_cap, n, k > 0 ? k : INT_MAX, a.sel + (size_t)b * a.kp_cap, a.counts + b * SC_N + SC_SEL);
}

// ------------------------------------------------------------------------------------------------------------------
// descriptor: calcSIFTDescriptor on the Gaussian level of the keypoint's (octave, layer)
// ------------------------------------------------------------------------------------------------------------------
struct SfDescArgs {
  SfListArgs l;
  const float* pyr;
  size_t stride;
  int oct_w[SF_MAX_OCT], oct_h[SF_MAX_OCT];
  size_t oct_off[SF_MAX_OCT];
  int n_oct;
};

__global__ void __launch_bounds__(32) k_sift_describe(SfDescArgs a) {
  __shared__ float lh[32 * SF_HPITCH];
  const int lane = threadIdx.x, b = blockIdx.y;
  const int n = a.l.counts[b * SC_N + SC_SEL];
  const SfImg& im = a.l.imgs[b];
  for (int q = blockIdx.x; q < n; q += gridDim.x) {
    const b2_sift_keypoint kp = a.l.fin[(size_t)b * a.l.kp_cap + a.l.sel[(size_t)b * a.l.kp_cap + q]];
    if (lane == 0) im.out_kp[q] = kp;
    // unpackOctave
    int octave = kp.octave & 255;
    const int layer = (kp.octave >> 8) & 255;
    octave = octave < 128 ? octave : (-128 | octave);
    const float scale = octave >= 0 ? 1.f / (float)(1 << octave) : (float)(1 << -octave);
    const int oi = octave + 1;
    const int rows = a.oct_h[oi], cols = a.oct_w[oi];
    const float* img = a.pyr + (size_t)b * a.stride + a.oct_off[oi] + (size_t)layer * rows * cols;
    const float size = kp.size * scale, ptx = kp.x * scale, pty = kp.y * scale;
    float ori = 360.f - kp.angle;
    if (fabsf(ori - 360.f) < FLT_EPSILON) ori = 0.f;
    const float scl = size * 0.5f;
    const int px = __float2int_rn(ptx), py = __float2int_rn(pty);
    float cos_t = cosf(ori * (float)(M_PI / 180)), sin_t = sinf(ori * (float)(M_PI / 180));
    const float bins_per_rad = SF_N / 360.f, exp_scale = -1.f / (SF_D * SF_D * 0.5f), hist_width = 3.f * scl;
    int radius = __float2int_rn(hist_width * 1.4142135623730951f * (SF_D + 1) * 0.5f);
    radius = min(radius, (int)sqrt((double)cols * cols + (double)rows * rows));
    cos_t /= hist_width;
    sin_t /= hist_width;
    float* h = lh + lane * SF_HPITCH;
    for (int j = 0; j < SF_HLEN; ++j) h[j] = 0.f;
    const int side = 2 * radius + 1;
    for (long long s = lane; s < (long long)side * side; s += 32) {
      const int i = (int)(s / side) - radius, j = (int)(s % side) - radius;
      const float c_rot = j * cos_t - i * sin_t, r_rot = j * sin_t + i * cos_t;
      float rbin = r_rot + SF_D / 2 - 0.5f, cbin = c_rot + SF_D / 2 - 0.5f;
      const int r = py + i, c = px + j;
      if (!(rbin > -1 && rbin < SF_D && cbin > -1 && cbin < SF_D && r > 0 && r < rows - 1 && c > 0 && c < cols - 1)) continue;
      const float dx = img[(size_t)r * cols + c + 1] - img[(size_t)r * cols + c - 1];
      const float dy = img[(size_t)(r - 1) * cols + c] - img[(size_t)(r + 1) * cols + c];
      const float wgt = expf((c_rot * c_rot + r_rot * r_rot) * exp_scale);
      float obin = (sf_atan(dy, dx) - ori) * bins_per_rad;
      const float mag = sqrtf(dx * dx + dy * dy) * wgt;
      const int r0 = (int)floorf(rbin), c0 = (int)floorf(cbin);
      int o0 = (int)floorf(obin);
      rbin -= r0, cbin -= c0, obin -= o0;
      if (o0 < 0) o0 += SF_N;
      if (o0 >= SF_N) o0 -= SF_N;
      const float v_r1 = mag * rbin, v_r0 = mag - v_r1;
      const float v_rc11 = v_r1 * cbin, v_rc10 = v_r1 - v_rc11;
      const float v_rc01 = v_r0 * cbin, v_rc00 = v_r0 - v_rc01;
      const float v_rco111 = v_rc11 * obin, v_rco110 = v_rc11 - v_rco111;
      const float v_rco101 = v_rc10 * obin, v_rco100 = v_rc10 - v_rco101;
      const float v_rco011 = v_rc01 * obin, v_rco010 = v_rc01 - v_rco011;
      const float v_rco001 = v_rc00 * obin, v_rco000 = v_rc00 - v_rco001;
      const int idx = ((r0 + 1) * (SF_D + 2) + c0 + 1) * (SF_N + 2) + o0;
      h[idx] += v_rco000;
      h[idx + 1] += v_rco001;
      h[idx + (SF_N + 2)] += v_rco010;
      h[idx + (SF_N + 3)] += v_rco011;
      h[idx + (SF_D + 2) * (SF_N + 2)] += v_rco100;
      h[idx + (SF_D + 2) * (SF_N + 2) + 1] += v_rco101;
      h[idx + (SF_D + 3) * (SF_N + 2)] += v_rco110;
      h[idx + (SF_D + 3) * (SF_N + 2) + 1] += v_rco111;
    }
    __syncwarp();
    // sum the 32 lane histograms in lane order; hold the totals in registers, then write them to lane 0's row
    float tot[(SF_HLEN + 31) / 32];
#pragma unroll
    for (int u = 0; u < (SF_HLEN + 31) / 32; ++u) {
      const int j = lane + 32 * u;
      float t = 0.f;
      if (j < SF_HLEN)
        for (int l = 0; l < 32; ++l) t += lh[l * SF_HPITCH + j];
      tot[u] = t;
    }
    __syncwarp();
#pragma unroll
    for (int u = 0; u < (SF_HLEN + 31) / 32; ++u)
      if (lane + 32 * u < SF_HLEN) lh[lane + 32 * u] = tot[u];
    __syncwarp();
    // fold the circular orientation bins; lane owns descriptor elements lane + 32 u
    float d[SF_DESC / 32];
#pragma unroll
    for (int u = 0; u < SF_DESC / 32; ++u) {
      const int e = lane + 32 * u, k = e % SF_N, j = (e / SF_N) % SF_D, i = e / (SF_N * SF_D);
      const int idx = ((i + 1) * (SF_D + 2) + (j + 1)) * (SF_N + 2);
      float v = lh[idx + k];
      if (k < 2) v += lh[idx + SF_N + k];
      d[u] = v;
    }
    float nrm2 = 0.f;
#pragma unroll
    for (int u = 0; u < SF_DESC / 32; ++u) nrm2 += d[u] * d[u];
    nrm2 = warp_sum(nrm2);
    const float thr = sqrtf(nrm2) * 0.2f;
    nrm2 = 0.f;
#pragma unroll
    for (int u = 0; u < SF_DESC / 32; ++u) {
      d[u] = fminf(d[u], thr);
      nrm2 += d[u] * d[u];
    }
    nrm2 = warp_sum(nrm2);
    const float f = 512.f / fmaxf(sqrtf(nrm2), FLT_EPSILON);
    uint8_t* out = im.out_desc + (size_t)q * SF_DESC;
#pragma unroll
    for (int u = 0; u < SF_DESC / 32; ++u) out[lane + 32 * u] = (uint8_t)min(max(__float2int_rn(d[u] * f), 0), 255);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
namespace {

// cv2 getGaussianKernel (the bit-exact double computation, rounded to float), ksize = cvRound(8 sigma + 1) | 1
SfTaps sf_taps(double sigma) {
  SfTaps t;
  const int n = ((int)lrint(sigma * 4 * 2 + 1)) | 1;
  t.r = (n - 1) / 2;
  const double scale2X = -0.125 / (sigma * sigma);
  std::vector<double> v(t.r);
  double sum = 0.0;
  for (int i = 0, x = 1 - n; i < t.r; i++, x += 2) {
    v[i] = exp((double)(x * x) * scale2X);
    sum += v[i];
  }
  sum = sum * 2.0 + 1.0;
  const double mul = 1.0 / sum;
  for (int i = 0; i < t.r; ++i) t.k[i] = t.k[n - 1 - i] = (float)(v[i] * mul);
  t.k[t.r] = (float)mul;
  return t;
}

struct SfGeom {
  int n_oct = 0;
  int w[SF_MAX_OCT], h[SF_MAX_OCT];
  size_t off[SF_MAX_OCT];
  size_t floats = 0;  // pyramid floats per image
  int cand_cap = 0, kp_cap = 0;
};

SfGeom sf_geom(int H, int W) {
  SfGeom g;
  const int m = 2 * (H < W ? H : W);
  int n = (int)lrint(log((double)m) / log(2.) - 2) + 1;
  if (n > SF_MAX_OCT) n = SF_MAX_OCT;
  g.n_oct = n > 0 ? n : 0;
  int w = 2 * W, h = 2 * H;
  for (int o = 0; o < g.n_oct; ++o) {
    g.w[o] = w, g.h[o] = h, g.off[o] = g.floats;
    g.floats += (size_t)SF_LEVELS * w * h;
    w /= 2, h /= 2;
  }
  const long long cap = (long long)4 * H * W / 32;
  g.cand_cap = (int)(cap > 4096 ? cap : 4096);
  g.kp_cap = 2 * g.cand_cap;
  return g;
}

// everything up to and including the top-k; all counts stay on the device
int sf_enqueue(b2_context* ctx, const SfImg* host_imgs, int n_img, int H, int W, int channels, size_t pitch, cudaStream_t st, SfGeom& g) {
  if (!ctx->sf) ctx->sf = new SiftState();
  SiftState* s = ctx->sf;
  g = sf_geom(H, W);
  const size_t nb = (size_t)n_img;
  B2_CUDA(ctx, s->pyr.ensure(nb * (g.floats ? g.floats : 1) * sizeof(float)));
  B2_CUDA(ctx, s->cand.ensure(nb * g.cand_cap * sizeof(SfCand)));
  B2_CUDA(ctx, s->raw.ensure(nb * g.kp_cap * sizeof(b2_sift_keypoint)));
  B2_CUDA(ctx, s->sorted.ensure(nb * g.kp_cap * sizeof(b2_sift_keypoint)));
  B2_CUDA(ctx, s->fin.ensure(nb * g.kp_cap * sizeof(b2_sift_keypoint)));
  B2_CUDA(ctx, s->fresp.ensure(nb * g.kp_cap * sizeof(float)));
  B2_CUDA(ctx, s->sel.ensure(nb * g.kp_cap * sizeof(int)));
  B2_CUDA(ctx, s->counts.ensure(nb * SC_N * sizeof(int)));
  B2_CUDA(ctx, s->table.ensure(nb * sizeof(SfImg)));
  B2_CUDA(ctx, cudaMemcpyAsync(s->table.p, host_imgs, nb * sizeof(SfImg), cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(s->counts.p, 0, nb * SC_N * sizeof(int), st));
  const SfImg* imgs = s->table.as<SfImg>();
  float* pyr = s->pyr.as<float>();
  const size_t stride = g.floats;
  int* counts = s->counts.as<int>();

  // Gaussian pyramid (sigmas as buildGaussianPyramid computes them, in double)
  double sig[SF_LEVELS];
  sig[0] = SF_SIGMA;
  const double k = pow(2., 1. / SF_LAYERS);
  for (int i = 1; i < SF_LEVELS; ++i) {
    const double prev = pow(k, (double)(i - 1)) * SF_SIGMA, total = prev * k;
    sig[i] = sqrt(total * total - prev * prev);
  }
  SfTaps taps[SF_LEVELS];
  taps[0] = sf_taps(sqrt(std::max((double)SF_SIGMA * SF_SIGMA - 0.5 * 0.5 * 4, 0.01)));
  for (int i = 1; i < SF_LEVELS; ++i) taps[i] = sf_taps(sig[i]);
  for (int o = 0; o < g.n_oct; ++o) {
    const int w = g.w[o], h = g.h[o];
    const size_t P = (size_t)w * h;
    float* lev0 = pyr + g.off[o];
    const dim3 tiles(cdiv(w, SF_TW), cdiv(h, SF_TH), n_img);
    if (o == 0) {
      SfBlurArgs a{nullptr, imgs, channels, W, H, pitch, lev0, stride, w, h, taps[0]};
      B2_LAUNCH(ctx, k_sift_blur<1>, tiles, 256, 0, st, a);
    } else {
      const float* src = pyr + g.off[o - 1] + (size_t)SF_LAYERS * g.w[o - 1] * g.h[o - 1];
      B2_LAUNCH(ctx, k_sift_down, dim3(cdiv(w, 256), h, n_img), 256, 0, st, src, g.w[o - 1], lev0, w, h, stride);
    }
    B2_CHECK_LAUNCH(ctx);
    for (int i = 1; i < SF_LEVELS; ++i) {
      SfBlurArgs a{lev0 + (i - 1) * P, imgs, channels, W, H, pitch, lev0 + i * P, stride, w, h, taps[i]};
      B2_LAUNCH(ctx, k_sift_blur<0>, tiles, 256, 0, st, a);
      B2_CHECK_LAUNCH(ctx);
    }
  }
  ctx->debug["sift_pyramid"] = {pyr, (int64_t)g.floats};

  // extrema and orientation, per octave
  for (int o = 0; o < g.n_oct; ++o) {
    const int w = g.w[o], h = g.h[o];
    if (w <= 2 * SF_BORDER || h <= 2 * SF_BORDER) continue;
    SfOctArgs a{pyr + g.off[o], (size_t)w * h, stride, w, h, o, s->cand.as<SfCand>(), s->raw.as<b2_sift_keypoint>(), counts, g.cand_cap, g.kp_cap};
    B2_LAUNCH(ctx, k_sift_extrema, dim3(cdiv(w - 2 * SF_BORDER, 256), h - 2 * SF_BORDER, n_img), 256, 0, st, a);
    B2_CHECK_LAUNCH(ctx);
  }
  for (int o = 0; o < g.n_oct; ++o) {
    const int w = g.w[o], h = g.h[o];
    if (w <= 2 * SF_BORDER || h <= 2 * SF_BORDER) continue;
    SfOctArgs a{pyr + g.off[o], (size_t)w * h, stride, w, h, o, s->cand.as<SfCand>(), s->raw.as<b2_sift_keypoint>(), counts, g.cand_cap, g.kp_cap};
    B2_LAUNCH(ctx, k_sift_orient, dim3(2 * ctx->sm_count, n_img), 32 * SF_OR_WARPS, 0, st, a);
    B2_CHECK_LAUNCH(ctx);
  }
  SfListArgs l{imgs, s->raw.as<b2_sift_keypoint>(), s->sorted.as<b2_sift_keypoint>(), s->fin.as<b2_sift_keypoint>(), s->fresp.as<float>(),
               s->sel.as<int>(), counts, g.kp_cap, W, H};
  const int rank_grid = std::min(cdiv(g.kp_cap, SF_RANK_T), 4 * ctx->sm_count);
  B2_LAUNCH(ctx, k_sift_rank, dim3(rank_grid, n_img), SF_RANK_T, 0, st, l);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_sift_compact, n_img, 1024, 0, st, l);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_sift_topk, n_img, 1024, 0, st, l);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

int sf_describe(b2_context* ctx, int n_img, int max_out, const SfGeom& g, cudaStream_t st) {
  SiftState* s = ctx->sf;
  SfDescArgs a;
  a.l = {s->table.as<SfImg>(), s->raw.as<b2_sift_keypoint>(), s->sorted.as<b2_sift_keypoint>(), s->fin.as<b2_sift_keypoint>(), s->fresp.as<float>(),
         s->sel.as<int>(), s->counts.as<int>(), g.kp_cap, 0, 0};
  a.pyr = s->pyr.as<float>();
  a.stride = g.floats;
  a.n_oct = g.n_oct;
  for (int o = 0; o < SF_MAX_OCT; ++o) {
    a.oct_w[o] = o < g.n_oct ? g.w[o] : 0;
    a.oct_h[o] = o < g.n_oct ? g.h[o] : 0;
    a.oct_off[o] = o < g.n_oct ? g.off[o] : 0;
  }
  const int grid = std::max(1, std::min(max_out, 16 * ctx->sm_count));
  B2_LAUNCH(ctx, k_sift_describe, dim3(grid, n_img), 32, 0, st, a);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

int sf_check_shape(b2_context* ctx, int H, int W, int channels, size_t pitch) {
  if (H < 1 || W < 1) return b2_fail(ctx, B2_ERR_ARG, "sift: empty image");
  if (channels != 1 && channels != 3 && channels != 4) return b2_fail(ctx, B2_ERR_ARG, "sift: channels must be 1, 3 or 4");
  if ((long long)H * W > SF_MAX_PIXELS || H > SF_MAX_SIDE || W > SF_MAX_SIDE)
    return b2_fail(ctx, B2_ERR_ARG, "sift: image larger than 2^24 pixels or 16384 per side");
  if (pitch < (size_t)W * channels) return b2_fail(ctx, B2_ERR_ARG, "sift: pitch smaller than a row");
  return B2_OK;
}

int sf_overflow(b2_context* ctx, const int* counts, int n_img, const SfGeom& g) {
  for (int b = 0; b < n_img; ++b)
    if (counts[b * SC_N + SC_CAND] > g.cand_cap || counts[b * SC_N + SC_RAW] > g.kp_cap)
      return b2_fail(ctx, B2_ERR_STATE, "sift: more keypoints than the workspace holds (4 H W / 32 extrema per image)");
  return B2_OK;
}

}  // namespace

extern "C" int b2_sift_detect_batched_dev(b2_context* ctx, b2_sift_image* images, int n_images, int height, int width, int channels,
                                          size_t pitch, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!images || n_images < 1 || n_images > SF_MAX_BATCH) return b2_fail(ctx, B2_ERR_ARG, "sift: 1..64 images per batch");
  int rc = sf_check_shape(ctx, height, width, channels, pitch);
  if (rc) return rc;
  std::vector<SfImg> t(n_images);
  int max_out = 0;
  for (int b = 0; b < n_images; ++b) {
    const b2_sift_image& q = images[b];
    if (!q.image || q.max_keypoints < 1 || !q.out_keypoints || !q.out_desc)
      return b2_fail(ctx, B2_ERR_ARG, "sift: null pointer or max_keypoints < 1");
    t[b] = SfImg{q.image, q.mask, q.out_keypoints, q.out_desc, q.max_keypoints, 0};
    max_out = std::max(max_out, q.max_keypoints);
  }
  cudaStream_t st = (cudaStream_t)stream;
  SfGeom g;
  rc = sf_enqueue(ctx, t.data(), n_images, height, width, channels, pitch, st, g);
  if (rc) return rc;
  rc = sf_describe(ctx, n_images, max_out, g, st);
  if (rc) return rc;
  std::vector<int> counts((size_t)n_images * SC_N);
  B2_CUDA(ctx, cudaMemcpyAsync(counts.data(), ctx->sf->counts.p, counts.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  rc = sf_overflow(ctx, counts.data(), n_images, g);
  if (rc) return rc;
  for (int b = 0; b < n_images; ++b) {
    images[b].out_n = counts[b * SC_N + SC_SEL];
    images[b].out_total = counts[b * SC_N + SC_FIN];
  }
  return B2_OK;
}

extern "C" int b2_sift_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels, const uint8_t* mask,
                                   b2_sift_keypoint* out_keypoints, uint8_t* out_desc, int capacity, int* out_n) {
  if (!ctx || !image || !out_n || capacity < 0 || (capacity > 0 && (!out_keypoints || !out_desc))) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  int rc = sf_check_shape(ctx, height, width, channels, (size_t)width * channels);
  if (rc) return rc;
  if (!ctx->sf) ctx->sf = new SiftState();
  SiftState* s = ctx->sf;
  cudaStream_t st = ctx->stream;
  const size_t ib = (size_t)height * width * channels, mb = (size_t)height * width;
  B2_CUDA(ctx, s->img.ensure(ib));
  B2_CUDA(ctx, cudaMemcpyAsync(s->img.p, image, ib, cudaMemcpyHostToDevice, st));
  if (mask) {
    B2_CUDA(ctx, s->mask.ensure(mb));
    B2_CUDA(ctx, cudaMemcpyAsync(s->mask.p, mask, mb, cudaMemcpyHostToDevice, st));
  }
  SfImg t{s->img.as<uint8_t>(), mask ? s->mask.as<uint8_t>() : nullptr, nullptr, nullptr, 0, 0};
  SfGeom g;
  rc = sf_enqueue(ctx, &t, 1, height, width, channels, (size_t)width * channels, st, g);
  if (rc) return rc;
  int counts[SC_N];
  B2_CUDA(ctx, cudaMemcpyAsync(counts, s->counts.p, sizeof(counts), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  rc = sf_overflow(ctx, counts, 1, g);
  if (rc) return rc;
  const int n = counts[SC_SEL];
  *out_n = n;
  if (n > capacity) return b2_fail(ctx, B2_SIFT_CAPACITY, "sift: more keypoints than the output capacity (*out_n = needed)");
  if (n == 0) return B2_OK;
  B2_CUDA(ctx, s->okp.ensure((size_t)n * sizeof(b2_sift_keypoint)));
  B2_CUDA(ctx, s->odesc.ensure((size_t)n * SF_DESC));
  t.out_kp = s->okp.as<b2_sift_keypoint>(), t.out_desc = s->odesc.as<uint8_t>(), t.max_kp = n;
  B2_CUDA(ctx, cudaMemcpyAsync(s->table.p, &t, sizeof(t), cudaMemcpyHostToDevice, st));
  rc = sf_describe(ctx, 1, n, g, st);
  if (rc) return rc;
  B2_CUDA(ctx, cudaMemcpyAsync(out_keypoints, s->okp.p, (size_t)n * sizeof(b2_sift_keypoint), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(out_desc, s->odesc.p, (size_t)n * SF_DESC, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B2_OK;
}
