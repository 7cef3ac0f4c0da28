// ORB detector-descriptor for sm_90a: cv2.ORB_create() with its defaults (nfeatures 500, scaleFactor 1.2f, nlevels 8,
// edgeThreshold 31, firstLevel 0, WTA_K 2, HARRIS_SCORE, patchSize 31, fastThreshold 20) restated, bit for bit.
//
// Reference semantics: gtsfm/frontend/detector_descriptor/orb.py:41-57 (gray conversion, cv2 detectAndCompute, top-k).
// oracle/orb_ref.py restates every stage in NumPy and is what the stage tests compare against.
//
// Stages of one batch of same-shape images (every stage is one launch over the batch, blockIdx.y = image):
//   k_orb_gray     level 0 = gray (cv2's fixed-point RGB2GRAY), level-0 mask = (mask != 0) * 255
//   k_orb_resize   level l = INTER_LINEAR_EXACT resize of level l - 1 (Q8 taps from double coordinates, Q16 sums); the
//                  mask likewise, then everything below 255 set to 0 (cv2's threshold 254, THRESH_TOZERO)
//   k_orb_fast     FAST-9/16 score map, threshold 20 (uint8, 0 = no corner)
//   k_orb_nms      strict 3 x 3 maxima of the score map inside the 31-pixel border where the level mask is set -> the
//                  level's candidate list (appended with atomics; the list is used as a set)
//   k_orb_blur     GaussianBlur(7 x 7, sigma 2) of the level as ORB runs it: cv2's separable float filter (ORB blurs a
//                  sub-matrix, which leaves out cv2's fixed-point path), each pass a chain of fused multiply-adds
//   k_orb_select   per (image, level): retainBest(2 n_l) by FAST score (256-bin histogram), Harris response (block 7,
//                  integer sums, the float formula operation by operation), retainBest(n_l) by Harris, rank in the output
//                  order -> the level's keypoints
//   k_orb_finish   per image: the levels concatenated, the max_keypoints largest responses (ties to the lower index), order kept
//   k_orb_describe warp per keypoint: intensity-centroid angle (integer moments, fastAtan2), rBRIEF on the blurred level
// Output order (cv2's within-level order comes from std::nth_element and is not reproduced): level ascending, then
// response descending, then y, then x, all in level coordinates.  The order is a function of the keypoint values only, so
// results are identical run to run and between batched and single-image calls.
//
// The file is compiled with -fmad=false: every float and double product and sum rounds as cv2's host code rounds it;
// the blur's fused multiply-adds are written out as __fmaf_rn.
//
// Workspace per image: 4 byte planes of the pyramid (levels, level masks, FAST scores, blurred levels), 3.3 H W bytes each,
// plus the lists, sized for the most candidates a level can have (one strict 3 x 3 maximum per 2 x 2 block), 0.82 H W
// entries x 32 bytes: about 40 H W bytes.  Images are limited to 2^24 pixels and 16384 per side; a batch holds at most 64.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "image.cuh"

namespace {

constexpr int OB_LEVELS = 8;
constexpr int OB_FEATURES = 500;
constexpr double OB_SCALE = (double)1.2f;  // ORB_create's scaleFactor is a float
constexpr int OB_EDGE = 31;                // edgeThreshold: keypoints keep 31 <= x < w - 31 on their level
constexpr int OB_PATCH = 31, OB_HALF = OB_PATCH / 2;
constexpr int OB_FAST_T = 20;
constexpr float OB_HARRIS_K = 0.04f;
constexpr int OB_HARRIS_R = 3;  // block 7
constexpr int OB_DESC = 32;
constexpr int OB_MAX_PIXELS = 1 << 24;
constexpr int OB_MAX_SIDE = 16384;
constexpr int OB_MAX_BATCH = 64;
// per-image counters: candidates, selection-1 survivors and kept keypoints per level, then the image's totals
enum { OC_CAND = 0, OC_SEL = OB_LEVELS, OC_KEPT = 2 * OB_LEVELS, OC_TOTAL = 3 * OB_LEVELS, OC_OUT, OC_N = 32 };

// cv2 ORB's rBRIEF test pattern, (x, y) pairs; test i compares points 2i and 2i + 1
__device__ const signed char ob_pattern[4 * 256] = {
#include "orb_pattern.inc"
};

}  // namespace

struct ObImg {  // device table row of one image
  const uint8_t* img;
  const uint8_t* mask;
  b2_sift_keypoint* out_kp;
  uint8_t* out_desc;
  int max_kp;
  int pad;
};

struct ObKp {  // a kept keypoint in level coordinates
  int x, y;
  float response;
};

struct ObArgs {
  const ObImg* imgs;
  int channels, W, H;
  size_t pitch;
  uint8_t *lev, *mlev, *score, *blur;  // byte planes: image b's level l at b * L + off[l]
  size_t L;
  int *cand, *sel, *aux, *job;  // lists: image b's level l at b * C + coff[l]
  float* harris;
  ObKp* kp;
  int* counts;  // OC_N per image
  size_t C;
  int w[OB_LEVELS], h[OB_LEVELS], coff[OB_LEVELS], ccap[OB_LEVELS], nper[OB_LEVELS], umax[OB_HALF + 1];
  size_t off[OB_LEVELS];
  float scale[OB_LEVELS];
  float taps[7];
  double rsx, rsy;  // resize: source / destination coordinate scale of the level being built
};

struct OrbState {
  DevBuf lev, mlev, score, blur, cand, sel, aux, job, harris, kp, counts, table, img, mask, okp, odesc;
};

void ob_destroy(b2_context* ctx) {
  delete ctx->ob;
  ctx->ob = nullptr;
}

// ------------------------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------------------------
// cv2 borderInterpolate(p, len, BORDER_REFLECT_101)
__device__ __forceinline__ int ob_reflect(int p, int len) {
  if (len == 1) return 0;
  while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// INTER_LINEAR_EXACT taps of destination coordinate d: source offset and Q8 weights of src[o] and src[o + 1]
__device__ __forceinline__ void ob_taps(int d, int src, double scale, int& o, int& c0, int& c1) {
  const double f = scale * ((double)d + 0.5) - 0.5;
  const int i = (int)floor(f);
  o = 0, c0 = 256, c1 = 0;
  if (i >= 0 && src > 1) {
    if (i < src - 1) {
      o = i;
      c1 = __double2int_rn((f - (double)i) * 256.0);
      c0 = 256 - c1;
    } else {
      o = src - 1;
    }
  }
}

// exclusive prefix of `flag` over a 1024-thread block; *total = number of set flags.  All threads must call.
__device__ __forceinline__ int ob_block_scan(bool flag, int* wtot, int* total) {
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

__device__ __forceinline__ int warp_isum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------------------------
// pyramid
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_orb_gray(ObArgs a) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= a.W * a.H) return;
  const int y = i / a.W, x = i - y * a.W;
  const ObImg& im = a.imgs[b];
  a.lev[b * a.L + i] = b2_gray_u8(im.img + (size_t)y * a.pitch + (size_t)x * a.channels, a.channels);
  if (im.mask) a.mlev[b * a.L + i] = im.mask[i] ? 255 : 0;
}

__global__ void __launch_bounds__(256) k_orb_resize(ObArgs a, int l) {
  const int b = blockIdx.y;
  const int w = a.w[l], h = a.h[l], sw = a.w[l - 1], sh = a.h[l - 1];
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= w * h) return;
  const int y = i / w, x = i - y * w;
  int xo, xc0, xc1, yo, yc0, yc1;
  ob_taps(x, sw, a.rsx, xo, xc0, xc1);
  ob_taps(y, sh, a.rsy, yo, yc0, yc1);
  const int xo1 = min(xo + 1, sw - 1), yo1 = min(yo + 1, sh - 1);
  const bool masked = a.imgs[b].mask != nullptr;
  for (int plane = 0; plane < (masked ? 2 : 1); ++plane) {
    const uint8_t* s = (plane ? a.mlev : a.lev) + b * a.L + a.off[l - 1];
    const int h0 = s[yo * sw + xo] * xc0 + s[yo * sw + xo1] * xc1;
    const int h1 = s[yo1 * sw + xo] * xc0 + s[yo1 * sw + xo1] * xc1;
    const int v = (h0 * yc0 + h1 * yc1 + (1 << 15)) >> 16;
    if (plane == 0)
      a.lev[b * a.L + a.off[l] + i] = (uint8_t)v;
    else
      a.mlev[b * a.L + a.off[l] + i] = v == 255 ? 255 : 0;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// FAST, candidates, blur
// ------------------------------------------------------------------------------------------------------------------
// FAST-9/16 score as cv2's cornerScore<16> computes it: max(threshold, the largest minimum of (centre - pixel) over 9
// contiguous circle pixels, or of (pixel - centre)) - 1, for a corner (that largest minimum > threshold); 0 otherwise.
__global__ void __launch_bounds__(256) k_orb_fast(ObArgs a, int l) {
  const int b = blockIdx.y;
  const int w = a.w[l], h = a.h[l];
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= w * h) return;
  const int y = i / w, x = i - y * w;
  uint8_t out = 0;
  if (x >= 3 && y >= 3 && x < w - 3 && y < h - 3) {
    const int cx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    const int cy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    const uint8_t* p = a.lev + b * a.L + a.off[l] + i;
    const int c = p[0];
    // darker (c - p) and brighter (p - c) differences as two arrays, both reduced by arc minima: written as the minimum of
    // the arc and the negated maximum of the other side, the 3-input min/max ptxas (CUDA 12.9, sm_90a) forms from it drops
    // the negation
    int dk[16], br[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int q = p[cy[k] * w + cx[k]];
      dk[k] = c - q;
      br[k] = q - c;
    }
    int best = INT_MIN;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      int m0 = INT_MAX, m1 = INT_MAX;
#pragma unroll
      for (int j = 0; j < 9; ++j) {
        m0 = min(m0, dk[(k + j) & 15]);
        m1 = min(m1, br[(k + j) & 15]);
      }
      best = max(best, max(m0, m1));
    }
    if (best > OB_FAST_T) out = (uint8_t)(max(best, OB_FAST_T) - 1);
  }
  a.score[b * a.L + a.off[l] + i] = out;
}

// strict 3 x 3 maxima inside the border where the level mask is set; launched over the interior only
__global__ void __launch_bounds__(256) k_orb_nms(ObArgs a, int l) {
  const int b = blockIdx.y;
  const int w = a.w[l], iw = w - 2 * OB_EDGE, ih = a.h[l] - 2 * OB_EDGE;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= iw * ih) return;
  const int y = OB_EDGE + i / iw, x = OB_EDGE + i % iw;
  const uint8_t* s = a.score + b * a.L + a.off[l] + (size_t)y * w + x;
  const int c = s[0];
  if (c == 0) return;
  if (!(c > s[-w - 1] && c > s[-w] && c > s[-w + 1] && c > s[-1] && c > s[1] && c > s[w - 1] && c > s[w] && c > s[w + 1])) return;
  if (a.imgs[b].mask && a.mlev[b * a.L + a.off[l] + (size_t)y * w + x] == 0) return;
  const int slot = atomicAdd(&a.counts[b * OC_N + OC_CAND + l], 1);
  if (slot < a.ccap[l]) a.cand[b * a.C + a.coff[l] + slot] = (y << 16) | x;
}

__global__ void __launch_bounds__(256) k_orb_blur(ObArgs a, int l) {
  const int b = blockIdx.y;
  const int w = a.w[l], h = a.h[l];
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= w * h) return;
  const int y = i / w, x = i - y * w;
  const uint8_t* src = a.lev + b * a.L + a.off[l];
  int xs[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) xs[k] = ob_reflect(x - 3 + k, w);
  float r[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    const uint8_t* row = src + (size_t)ob_reflect(y - 3 + j, h) * w;
    float s = (float)row[xs[0]] * a.taps[0];
#pragma unroll
    for (int k = 1; k < 7; ++k) s = __fmaf_rn((float)row[xs[k]], a.taps[k], s);
    r[j] = s;
  }
  float s = r[3] * a.taps[3];
#pragma unroll
  for (int k = 1; k <= 3; ++k) s = __fmaf_rn(r[3 - k] + r[3 + k], a.taps[3 + k], s);
  a.blur[b * a.L + a.off[l] + i] = (uint8_t)min(max(__float2int_rn(s), 0), 255);
}

// ------------------------------------------------------------------------------------------------------------------
// selection
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ob_harris(const uint8_t* img, int w, int x, int y) {
  int sa = 0, sb = 0, sc = 0;
  for (int i = -OB_HARRIS_R; i <= OB_HARRIS_R; ++i)
    for (int j = -OB_HARRIS_R; j <= OB_HARRIS_R; ++j) {
      const uint8_t* p = img + (size_t)(y + i) * w + (x + j);
      const int ix = (p[1] - p[-1]) * 2 + (p[-w + 1] - p[-w - 1]) + (p[w + 1] - p[w - 1]);
      const int iy = (p[w] - p[-w]) * 2 + (p[w - 1] - p[-w - 1]) + (p[w + 1] - p[-w + 1]);
      sa += ix * ix;
      sb += iy * iy;
      sc += ix * iy;
    }
  const float scale = 1.f / ((float)(4 * (2 * OB_HARRIS_R + 1)) * 255.f);
  const float s4 = scale * scale * scale * scale;
  const float fa = (float)sa, fb = (float)sb, fc = (float)sc;
  return (fa * fb - fc * fc - OB_HARRIS_K * (fa + fb) * (fa + fb)) * s4;
}

// one 1024-thread block per (level, image)
__global__ void __launch_bounds__(1024) k_orb_select(ObArgs a) {
  const int l = blockIdx.x, b = blockIdx.y;
  __shared__ int hist[256];
  __shared__ int wtot[33];
  __shared__ int thr, carry, kept;
  int* cnt = a.counts + b * OC_N;
  const int n = min(cnt[OC_CAND + l], a.ccap[l]);
  const int w = a.w[l];
  const int want1 = 2 * a.nper[l], want2 = a.nper[l];
  const uint8_t* score = a.score + b * a.L + a.off[l];
  const uint8_t* img = a.lev + b * a.L + a.off[l];
  const int* cand = a.cand + b * a.C + a.coff[l];
  int* sel = a.sel + b * a.C + a.coff[l];
  int* keep = a.aux + b * a.C + a.coff[l];
  float* resp = a.harris + b * a.C + a.coff[l];
  ObKp* out = a.kp + b * a.C + a.coff[l];
  for (int i = threadIdx.x; i < 256; i += 1024) hist[i] = 0;
  if (threadIdx.x == 0) carry = 0, kept = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += 1024) atomicAdd(&hist[score[(cand[i] >> 16) * w + (cand[i] & 0xffff)]], 1);
  __syncthreads();
  // retainBest(2 n_l): keep every candidate whose score is >= the (2 n_l)-th largest
  if (threadIdx.x == 0) {
    int t = 0;
    if (n > want1) {
      t = 256;
      int acc = 0;
      for (int s = 255; s >= 0 && want1 > 0; --s) {
        acc += hist[s];
        if (acc >= want1) {
          t = s;
          break;
        }
      }
    }
    thr = t;
  }
  __syncthreads();
  const int t = thr;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    int c = 0;
    bool f = false;
    if (i < n) {
      c = cand[i];
      f = score[(c >> 16) * w + (c & 0xffff)] >= t;
    }
    int tot;
    const int pos = ob_block_scan(f, wtot, &tot) + carry;
    if (f) {
      sel[pos] = c;
      resp[pos] = ob_harris(img, w, c & 0xffff, c >> 16);
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  const int m = carry;
  if (threadIdx.x == 0) cnt[OC_SEL + l] = m;
  // retainBest(n_l) by Harris response: keep i when fewer than n_l responses are larger
  for (int i = threadIdx.x; i < m; i += 1024) {
    const float r = resp[i];
    int gt = 0;
    if (m > want2)
      for (int j = 0; j < m; ++j) gt += resp[j] > r;
    keep[i] = m <= want2 || gt < want2;
  }
  __syncthreads();
  // rank among the kept: response descending, then y, then x
  for (int i = threadIdx.x; i < m; i += 1024) {
    if (!keep[i]) continue;
    const float r = resp[i];
    const int yx = sel[i];
    int pos = 0;
    for (int j = 0; j < m; ++j) pos += keep[j] && (resp[j] > r || (resp[j] == r && sel[j] < yx));
    out[pos] = ObKp{yx & 0xffff, yx >> 16, r};
    atomicAdd(&kept, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) cnt[OC_KEPT + l] = kept;
}

// one 1024-thread block per image: concatenate the levels, keep the max_kp largest responses (ties to the lower index)
__global__ void __launch_bounds__(1024) k_orb_finish(ObArgs a) {
  const int b = blockIdx.x;
  __shared__ int wtot[33];
  __shared__ int koff[OB_LEVELS + 1], carry;
  int* cnt = a.counts + b * OC_N;
  if (threadIdx.x == 0) {
    koff[0] = 0;
    for (int l = 0; l < OB_LEVELS; ++l) koff[l + 1] = koff[l] + cnt[OC_KEPT + l];
    carry = 0;
    cnt[OC_TOTAL] = koff[OB_LEVELS];
  }
  __syncthreads();
  const int total = koff[OB_LEVELS], max_kp = a.imgs[b].max_kp;
  const ObKp* kp = a.kp + b * a.C;
  auto at = [&](int g) {
    int l = 0;
    while (g >= koff[l + 1]) ++l;
    return kp[a.coff[l] + g - koff[l]].response;
  };
  int* job = a.job + b * a.C;
  for (int base = 0; base < total; base += 1024) {
    const int g = base + threadIdx.x;
    bool take = false;
    if (g < total) {
      take = true;
      if (total > max_kp) {
        const float r = at(g);
        int rank = 0;
        for (int h = 0; h < total; ++h) {
          const float q = at(h);
          rank += q > r || (q == r && h < g);
        }
        take = rank < max_kp;
      }
    }
    int tot;
    const int pos = ob_block_scan(take, wtot, &tot) + carry;
    if (take) job[pos] = g;
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) cnt[OC_OUT] = carry;
}

// warp per output keypoint: angle, then the 32 descriptor bytes (lane i writes byte i)
__global__ void __launch_bounds__(256) k_orb_describe(ObArgs a) {
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int* cnt = a.counts + b * OC_N;
  const int n_out = cnt[OC_OUT];
  const ObImg& im = a.imgs[b];
  int koff[OB_LEVELS + 1];
  koff[0] = 0;
#pragma unroll
  for (int l = 0; l < OB_LEVELS; ++l) koff[l + 1] = koff[l] + cnt[OC_KEPT + l];
  for (int q = blockIdx.x * 8 + (threadIdx.x >> 5); q < n_out; q += gridDim.x * 8) {
    const int g = a.job[b * a.C + q];
    int l = 0;
    while (g >= koff[l + 1]) ++l;
    const ObKp k = a.kp[b * a.C + a.coff[l] + g - koff[l]];
    const int w = a.w[l];
    const uint8_t* img = a.lev + b * a.L + a.off[l];
    // intensity centroid over the radius-15 disc: lane v sums row k.y + v - 15
    int m10 = 0, m01 = 0;
    if (lane < OB_PATCH) {
      const int dy = lane - OB_HALF, d = a.umax[dy < 0 ? -dy : dy];
      const uint8_t* row = img + (size_t)(k.y + dy) * w + k.x;
      int su = 0, s = 0;
      for (int u = -d; u <= d; ++u) {
        su += u * row[u];
        s += row[u];
      }
      m10 = su, m01 = dy * s;
    }
    m10 = warp_isum(m10);
    m01 = warp_isum(m01);
    const float angle = b2_fast_atan2((float)m01, (float)m10);
    const float sc = a.scale[l];
    const float ptx = (float)k.x * sc, pty = (float)k.y * sc;
    // the descriptor's centre as cv2 recovers it from the scaled point
    const float inv = 1.f / sc;
    const int cx = __float2int_rn(ptx * inv), cy = __float2int_rn(pty * inv);
    const float rad = angle * (float)(3.141592653589793 / 180.0);
    const float ca = (float)cos((double)rad), sa = (float)sin((double)rad);
    const uint8_t* bl = a.blur + b * a.L + a.off[l];
    int val = 0;
#pragma unroll
    for (int bit = 0; bit < 8; ++bit) {
      int v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int t = 2 * (16 * lane + 2 * bit + e);
        const float px = (float)ob_pattern[t], py = (float)ob_pattern[t + 1];
        const int ix = __float2int_rn(px * ca - py * sa), iy = __float2int_rn(px * sa + py * ca);
        v[e] = bl[(size_t)(cy + iy) * w + (cx + ix)];
      }
      val |= (v[0] < v[1]) << bit;
    }
    im.out_desc[(size_t)q * OB_DESC + lane] = (uint8_t)val;
    if (lane == 0) im.out_kp[q] = b2_sift_keypoint{ptx, pty, (float)OB_PATCH * sc, angle, k.response, l};
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
namespace {

struct ObGeom {
  int w[OB_LEVELS], h[OB_LEVELS], coff[OB_LEVELS], ccap[OB_LEVELS], nper[OB_LEVELS];
  size_t off[OB_LEVELS];
  float scale[OB_LEVELS];
  size_t L = 0, C = 0;
};

// level sizes cvRound(side / s_l) with s_l = (float)pow(1.2f, l) in float; byte planes padded to 16 bytes per level;
// candidate lists sized ceil(h / 2) ceil(w / 2) (one strict 3 x 3 maximum per 2 x 2 block at most)
ObGeom ob_geom(int H, int W) {
  ObGeom g;
  const float factor = (float)(1.0 / OB_SCALE);
  float share = OB_FEATURES * (1 - factor) / (1 - (float)pow((double)factor, (double)OB_LEVELS));
  int sum = 0;
  for (int l = 0; l < OB_LEVELS; ++l) {
    g.scale[l] = (float)pow(OB_SCALE, (double)l);
    g.w[l] = (int)lrintf((float)W / g.scale[l]);
    g.h[l] = (int)lrintf((float)H / g.scale[l]);
    g.off[l] = g.L;
    g.L += ((size_t)g.w[l] * g.h[l] + 15) & ~(size_t)15;
    g.ccap[l] = ((g.w[l] + 1) / 2) * ((g.h[l] + 1) / 2);
    g.coff[l] = (int)g.C;
    g.C += g.ccap[l];
    if (l < OB_LEVELS - 1) {
      g.nper[l] = (int)lrintf(share);
      sum += g.nper[l];
      share *= factor;
    } else {
      g.nper[l] = std::max(OB_FEATURES - sum, 0);
    }
  }
  return g;
}

ObArgs ob_args(OrbState* s, const ObGeom& g, int channels, int W, int H, size_t pitch) {
  ObArgs a;
  a.imgs = s->table.as<ObImg>();
  a.channels = channels, a.W = W, a.H = H, a.pitch = pitch;
  a.lev = s->lev.as<uint8_t>(), a.mlev = s->mlev.as<uint8_t>(), a.score = s->score.as<uint8_t>(), a.blur = s->blur.as<uint8_t>();
  a.L = g.L;
  a.cand = s->cand.as<int>(), a.sel = s->sel.as<int>(), a.aux = s->aux.as<int>(), a.job = s->job.as<int>();
  a.harris = s->harris.as<float>();
  a.kp = s->kp.as<ObKp>();
  a.counts = s->counts.as<int>();
  a.C = g.C;
  for (int l = 0; l < OB_LEVELS; ++l) {
    a.w[l] = g.w[l], a.h[l] = g.h[l], a.coff[l] = g.coff[l], a.ccap[l] = g.ccap[l], a.nper[l] = g.nper[l];
    a.off[l] = g.off[l], a.scale[l] = g.scale[l];
  }
  // umax: the half-width of every row of the radius-15 disc, made symmetric (ORB's computeKeyPoints)
  int um[OB_HALF + 2] = {0};
  const int vmax = (int)floor(OB_HALF * sqrt(2.f) / 2 + 1), vmin = (int)ceil(OB_HALF * sqrt(2.f) / 2);
  for (int v = 0; v <= vmax; ++v) um[v] = (int)lrint(sqrt((double)OB_HALF * OB_HALF - v * v));
  for (int v = OB_HALF, v0 = 0; v >= vmin; --v) {
    while (um[v0] == um[v0 + 1]) ++v0;
    um[v] = v0;
    ++v0;
  }
  for (int v = 0; v <= OB_HALF; ++v) a.umax[v] = um[v];
  // cv2 getGaussianKernel(7, 2, CV_32F): computed in double, rounded to float
  const double scale2x = -0.125 / (2.0 * 2.0);
  double v[3], sum = 0.0;
  for (int i = 0, x = -6; i < 3; ++i, x += 2) sum += (v[i] = exp((double)(x * x) * scale2x));
  const double mul = 1.0 / (sum * 2.0 + 1.0);
  for (int i = 0; i < 3; ++i) a.taps[i] = a.taps[6 - i] = (float)(v[i] * mul);
  a.taps[3] = (float)mul;
  a.rsx = a.rsy = 0.0;
  return a;
}

// everything up to the per-level keypoint lists; counts stay on the device
int ob_enqueue(b2_context* ctx, const ObImg* host_imgs, int n_img, int H, int W, int channels, size_t pitch, cudaStream_t st,
               ObGeom& g, ObArgs& a) {
  if (!ctx->ob) ctx->ob = new OrbState();
  OrbState* s = ctx->ob;
  g = ob_geom(H, W);
  const size_t nb = (size_t)n_img;
  for (DevBuf* p : {&s->lev, &s->mlev, &s->score, &s->blur}) B2_CUDA(ctx, p->ensure(nb * g.L));
  for (DevBuf* p : {&s->cand, &s->sel, &s->aux, &s->job, &s->harris}) B2_CUDA(ctx, p->ensure(nb * g.C * 4));
  B2_CUDA(ctx, s->kp.ensure(nb * g.C * sizeof(ObKp)));
  B2_CUDA(ctx, s->counts.ensure(nb * OC_N * sizeof(int)));
  B2_CUDA(ctx, s->table.ensure(nb * sizeof(ObImg)));
  B2_CUDA(ctx, cudaMemcpyAsync(s->table.p, host_imgs, nb * sizeof(ObImg), cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(s->counts.p, 0, nb * OC_N * sizeof(int), st));
  a = ob_args(s, g, channels, W, H, pitch);
  B2_LAUNCH(ctx, k_orb_gray, dim3(cdiv(W * H, 256), n_img), 256, 0, st, a);
  B2_CHECK_LAUNCH(ctx);
  for (int l = 1; l < OB_LEVELS; ++l) {
    a.rsx = 1.0 / ((double)g.w[l] / g.w[l - 1]);
    a.rsy = 1.0 / ((double)g.h[l] / g.h[l - 1]);
    B2_LAUNCH(ctx, k_orb_resize, dim3(cdiv(g.w[l] * g.h[l], 256), n_img), 256, 0, st, a, l);
    B2_CHECK_LAUNCH(ctx);
  }
  for (int l = 0; l < OB_LEVELS; ++l) {
    const int P = g.w[l] * g.h[l];
    B2_LAUNCH(ctx, k_orb_fast, dim3(cdiv(P, 256), n_img), 256, 0, st, a, l);
    B2_CHECK_LAUNCH(ctx);
    if (g.w[l] > 2 * OB_EDGE && g.h[l] > 2 * OB_EDGE) {
      B2_LAUNCH(ctx, k_orb_nms, dim3(cdiv((g.w[l] - 2 * OB_EDGE) * (g.h[l] - 2 * OB_EDGE), 256), n_img), 256, 0, st, a, l);
      B2_CHECK_LAUNCH(ctx);
    }
    B2_LAUNCH(ctx, k_orb_blur, dim3(cdiv(P, 256), n_img), 256, 0, st, a, l);
    B2_CHECK_LAUNCH(ctx);
  }
  B2_LAUNCH(ctx, k_orb_select, dim3(OB_LEVELS, n_img), 1024, 0, st, a);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_orb_finish, n_img, 1024, 0, st, a);
  B2_CHECK_LAUNCH(ctx);
  const int64_t planes = (int64_t)(nb * g.L / 4), lists = (int64_t)(nb * g.C);
  ctx->debug["orb_levels"] = {reinterpret_cast<const float*>(s->lev.p), planes};
  ctx->debug["orb_masks"] = {reinterpret_cast<const float*>(s->mlev.p), planes};
  ctx->debug["orb_scores"] = {reinterpret_cast<const float*>(s->score.p), planes};
  ctx->debug["orb_blurred"] = {reinterpret_cast<const float*>(s->blur.p), planes};
  ctx->debug["orb_sel"] = {reinterpret_cast<const float*>(s->sel.p), lists};
  ctx->debug["orb_harris"] = {s->harris.as<float>(), lists};
  ctx->debug["orb_counts"] = {reinterpret_cast<const float*>(s->counts.p), (int64_t)(nb * OC_N)};
  return B2_OK;
}

int ob_describe(b2_context* ctx, int n_img, int max_out, const ObArgs& a, cudaStream_t st) {
  const int grid = std::max(1, std::min(cdiv(max_out, 8), 4 * ctx->sm_count));
  B2_LAUNCH(ctx, k_orb_describe, dim3(grid, n_img), 256, 0, st, a);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

int ob_check_shape(b2_context* ctx, int H, int W, int channels, size_t pitch) {
  if (H < 1 || W < 1) return b2_fail(ctx, B2_ERR_ARG, "orb: empty image");
  if (channels != 1 && channels != 3 && channels != 4) return b2_fail(ctx, B2_ERR_ARG, "orb: channels must be 1, 3 or 4");
  if ((long long)H * W > OB_MAX_PIXELS || H > OB_MAX_SIDE || W > OB_MAX_SIDE)
    return b2_fail(ctx, B2_ERR_ARG, "orb: image larger than 2^24 pixels or 16384 per side");
  if (pitch < (size_t)W * channels) return b2_fail(ctx, B2_ERR_ARG, "orb: pitch smaller than a row");
  return B2_OK;
}

}  // namespace

extern "C" int b2_orb_detect_batched_dev(b2_context* ctx, b2_orb_image* images, int n_images, int height, int width, int channels,
                                         size_t pitch, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!images || n_images < 1 || n_images > OB_MAX_BATCH) return b2_fail(ctx, B2_ERR_ARG, "orb: 1..64 images per batch");
  int rc = ob_check_shape(ctx, height, width, channels, pitch);
  if (rc) return rc;
  std::vector<ObImg> t(n_images);
  int max_out = 0;
  for (int b = 0; b < n_images; ++b) {
    const b2_orb_image& q = images[b];
    if (!q.image || q.max_keypoints < 1 || !q.out_keypoints || !q.out_desc)
      return b2_fail(ctx, B2_ERR_ARG, "orb: null pointer or max_keypoints < 1");
    t[b] = ObImg{q.image, q.mask, q.out_keypoints, q.out_desc, q.max_keypoints, 0};
    max_out = std::max(max_out, q.max_keypoints);
  }
  cudaStream_t st = (cudaStream_t)stream;
  ObGeom g;
  ObArgs a;
  rc = ob_enqueue(ctx, t.data(), n_images, height, width, channels, pitch, st, g, a);
  if (rc) return rc;
  rc = ob_describe(ctx, n_images, max_out, a, st);
  if (rc) return rc;
  std::vector<int> counts((size_t)n_images * OC_N);
  B2_CUDA(ctx, cudaMemcpyAsync(counts.data(), ctx->ob->counts.p, counts.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (int b = 0; b < n_images; ++b) {
    images[b].out_n = counts[b * OC_N + OC_OUT];
    images[b].out_total = counts[b * OC_N + OC_TOTAL];
  }
  return B2_OK;
}

extern "C" int b2_orb_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels, const uint8_t* mask,
                                  b2_sift_keypoint* out_keypoints, uint8_t* out_desc, int capacity, int* out_n) {
  if (!ctx || !image || !out_n || capacity < 0 || (capacity > 0 && (!out_keypoints || !out_desc))) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  int rc = ob_check_shape(ctx, height, width, channels, (size_t)width * channels);
  if (rc) return rc;
  if (!ctx->ob) ctx->ob = new OrbState();
  OrbState* s = ctx->ob;
  cudaStream_t st = ctx->stream;
  const size_t ib = (size_t)height * width * channels, mb = (size_t)height * width;
  B2_CUDA(ctx, s->img.ensure(ib));
  B2_CUDA(ctx, cudaMemcpyAsync(s->img.p, image, ib, cudaMemcpyHostToDevice, st));
  if (mask) {
    B2_CUDA(ctx, s->mask.ensure(mb));
    B2_CUDA(ctx, cudaMemcpyAsync(s->mask.p, mask, mb, cudaMemcpyHostToDevice, st));
  }
  ObImg t{s->img.as<uint8_t>(), mask ? s->mask.as<uint8_t>() : nullptr, nullptr, nullptr, INT_MAX, 0};
  ObGeom g;
  ObArgs a;
  rc = ob_enqueue(ctx, &t, 1, height, width, channels, (size_t)width * channels, st, g, a);
  if (rc) return rc;
  int counts[OC_N];
  B2_CUDA(ctx, cudaMemcpyAsync(counts, s->counts.p, sizeof(counts), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  const int n = counts[OC_OUT];
  *out_n = n;
  if (n > capacity) return b2_fail(ctx, B2_SIFT_CAPACITY, "orb: more keypoints than the output capacity (*out_n = needed)");
  if (n == 0) return B2_OK;
  B2_CUDA(ctx, s->okp.ensure((size_t)n * sizeof(b2_sift_keypoint)));
  B2_CUDA(ctx, s->odesc.ensure((size_t)n * OB_DESC));
  t.out_kp = s->okp.as<b2_sift_keypoint>(), t.out_desc = s->odesc.as<uint8_t>();
  B2_CUDA(ctx, cudaMemcpyAsync(s->table.p, &t, sizeof(t), cudaMemcpyHostToDevice, st));
  rc = ob_describe(ctx, 1, n, a, st);
  if (rc) return rc;
  B2_CUDA(ctx, cudaMemcpyAsync(out_keypoints, s->okp.p, (size_t)n * sizeof(b2_sift_keypoint), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(out_desc, s->odesc.p, (size_t)n * OB_DESC, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B2_OK;
}
