// SuperPoint detect + describe for sm_90a.
//
// Reference semantics restated (file:line relative to the reference repo):
//   thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:145-202 (forward), :47-62 (simple_nms),
//   :65-70 (remove_borders), :80-92 (sample_descriptors); wrapper gtsfm/frontend/detector_descriptor/superpoint.py:63-93
//   and gtsfm/utils/images.py:15-40 (cv2 RGB->gray).
//
// Data layout in HBM: activations NHWC fp32 (channel-contiguous: one pixel's 64/128/256 channels are one 256/512/1024 B
// segment, which is what both the implicit-GEMM K loop and the bilinear descriptor gather want); conv weights repacked
// at load to [tap][cin][cout]; 1x1 weights to [cin][cout]; score / NMS maps (H8, W8) fp32; dense descriptors
// (Hc, Wc, 256) fp32; keypoints as (x, y) float pairs in torch.nonzero (row-major) order.
#include <stdlib.h>

#include "common.cuh"
#include "conv_ps.cuh"
#include "image.cuh"
#include "linear.cuh"
#include "topk.cuh"

namespace {

constexpr int SP_NCONV = 12;
// name order: conv1a conv1b conv2a conv2b conv3a conv3b conv4a conv4b convPa convPb convDa convDb
constexpr int SP_CO[SP_NCONV] = {64, 64, 64, 64, 128, 128, 128, 128, 256, 65, 256, 256};
constexpr int SP_CI[SP_NCONV] = {1, 64, 64, 64, 64, 128, 128, 128, 128, 256, 128, 256};
constexpr int SP_K[SP_NCONV] = {3, 3, 3, 3, 3, 3, 3, 3, 3, 1, 3, 1};
constexpr size_t SP_NFLOATS = 1300865;

}  // namespace

struct SuperPointState {
  bool loaded = false;
  DevBuf wblob;
  float* w[SP_NCONV] = {};
  float* b[SP_NCONV] = {};
  // wgmma path: 3x3 weights as [cout][tap * cin] split-fp16 planes (B operand of the implicit GEMM)
  DevBuf wsplit_h, wsplit_l, errflag, conv_dbg, logits;
  struct ConvMapCache {
    ConvPsMaps maps;
    const void *ih = nullptr, *wh = nullptr;
    int H = 0, W = 0;
  } conv_maps[12];
  size_t wsoff[SP_NCONV] = {};
  bool use_tc = true;
  // workspace
  DevBuf gray, a0, a1, feat, head, heat, nms, rowcnt, rowoff, dense, kpxy, kpsc;
  int H = 0, W = 0, Hc = 0, Wc = 0;
  int n_kp = 0;
  bool have_dense = false;
  uint64_t map_token = 0;  // identifies the dense descriptor map a detect call left behind (checked by describe)
  DevBuf sel_idx, sel_cnt; // device top-k selection of b2_superpoint_extract_dev
  // CUDA graph of the network (sp_detect_impl)
  static constexpr int GKEY = 20, GSLOTS = 4;
  struct GraphSlot {
    uint64_t key[GKEY] = {};
    cudaGraphExec_t exec = nullptr;
    uint64_t launches = 0;
  } gslot[GSLOTS];
  cudaStream_t cap_stream = nullptr;
  int gnext = 0, gcaptures = 0;
};

static inline uint32_t __float_as_uint_host(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}

void sp_destroy(b2_context* ctx) {
  if (!ctx->sp) return;
  SuperPointState* s = ctx->sp;
  DevBuf* bufs[] = {&s->wblob, &s->wsplit_h, &s->wsplit_l, &s->errflag, &s->conv_dbg, &s->logits, &s->gray, &s->a0, &s->a1, &s->feat, &s->head, &s->heat, &s->nms,
                    &s->rowcnt, &s->rowoff, &s->dense, &s->kpxy, &s->kpsc, &s->sel_idx, &s->sel_cnt};
  for (DevBuf* b : bufs) b->release();
  for (auto& g : s->gslot)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  if (s->cap_stream) cudaStreamDestroy(s->cap_stream);
  delete s;
  ctx->sp = nullptr;
}

// ------------------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------------------

// cv2 COLOR_RGB2GRAY / COLOR_RGBA2GRAY (image.cuh)
__global__ void k_to_gray(const uint8_t* __restrict__ img, size_t pitch, int channels, int H, int W,
                          uint8_t* __restrict__ gray) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y;
  if (x >= W) return;
  gray[(size_t)y * W + x] = b2_gray_u8(img + (size_t)y * pitch + (size_t)x * channels, channels);
}

// conv1a: 1 -> 64 channels, 3x3, pad 1, bias, ReLU; input gray u8 / 255 (gtsfm/.../superpoint.py:74).
// HBM-bound (writes 64 channels per pixel: 256 B as planes or fp32).  Lane = (pixel of a quad, 8-channel group): the 72
// weights + 8 biases of the channel group live in registers for the whole grid-stride loop, and a warp's store is 4 pixels x
// 128 contiguous bytes per plane.
constexpr int C1A_THREADS = 256;
__global__ void __launch_bounds__(C1A_THREADS) k_conv1a(const uint8_t* __restrict__ gray, const float* __restrict__ wt /*[9][64]*/,
                                                         const float* __restrict__ bias, float* __restrict__ out, int H, int W,
                                                         __half* __restrict__ oh, __half* __restrict__ ol) {
  const int lane = threadIdx.x & 31, cg = lane & 7, sub = lane >> 3;
  float w[9][8], b[8];
#pragma unroll
  for (int tp = 0; tp < 9; ++tp)
#pragma unroll
    for (int c = 0; c < 8; ++c) w[tp][c] = __ldg(wt + tp * 64 + cg * 8 + c);
#pragma unroll
  for (int c = 0; c < 8; ++c) b[c] = __ldg(bias + cg * 8 + c);
  // a warp step = 4 consecutive pixels of one row: lanes 0..17 fetch and normalise the 3 x 6 input window once, every lane
  // then picks its 9 taps by shuffle
  const int qpr = (W + 3) / 4;  // quads per row
  const long long nquad = (long long)H * qpr;
  const long long warp0 = (long long)blockIdx.x * (C1A_THREADS / 32) + (threadIdx.x >> 5), nwarp = (long long)gridDim.x * (C1A_THREADS / 32);
  const int wr = lane / 6, wc = lane % 6;  // window cell of lanes 0..17
  for (long long q = warp0; q < nquad; q += nwarp) {
    const int y = (int)(q / qpr), x0 = (int)(q % qpr) * 4;
    const long long pix = (long long)y * W + x0 + sub;
    float win = 0.f;
    {
      const int yy = y + wr - 1, xx = x0 + wc - 1;
      if (lane < 18 && yy >= 0 && yy < H && xx >= 0 && xx < W) win = (float)__ldg(gray + (size_t)yy * W + xx) / 255.0f;
    }
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = b[c];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const float v = __shfl_sync(0xffffffffu, win, dy * 6 + sub + dx);
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = fmaf(v, w[dy * 3 + dx][c], acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = fmaxf(acc[c], 0.f);
    if (x0 + sub >= W) continue;
    if (oh) {  // split fp16 planes for the wgmma convolutions
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) tc::split2(acc[2 * i], acc[2 * i + 1], hi[i], lo[i]);
      *reinterpret_cast<uint4*>(oh + (size_t)pix * 64 + cg * 8) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<uint4*>(ol + (size_t)pix * 64 + cg * 8) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    } else {
      float4* d = reinterpret_cast<float4*>(out + (size_t)pix * 64 + cg * 8);
      d[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      d[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
  }
}

// Generic 3x3 conv, pad 1, bias + ReLU, optional fused 2x2/2 max-pool, NHWC fp32, SIMT fp32 FMA (exact-fp32 path).
// Block tile: 8 rows x 16 cols of pixels x 64 output channels; thread micro-tile 2x4 pixels x 4 channels.
constexpr int CT_H = 8, CT_W = 16, CK = 8, CKP = 12;  // CKP: padded per-pixel stride in smem (floats)
template <int POOL>
__global__ void __launch_bounds__(256) k_conv3x3(const float* __restrict__ in, const float* __restrict__ wt,
                                                  const float* __restrict__ bias, float* __restrict__ out, int H, int W,
                                                  int Cin, int Cout) {
  __shared__ __align__(16) float in_s[(CT_H + 2) * (CT_W + 2) * CKP];
  __shared__ __align__(16) float w_s[9 * CK * 64];
  const int t = threadIdx.x;
  const int cg = t & 15, pg = t >> 4;
  const int prow = (pg >> 2) * 2, pcol = (pg & 3) * 4;
  const int y0 = blockIdx.y * CT_H, x0 = blockIdx.x * CT_W;
  const int co0 = blockIdx.z * 64;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;

  for (int c0 = 0; c0 < Cin; c0 += CK) {
    // input patch (10 x 18 pixels x CK channels), zero padded
    for (int i = t; i < (CT_H + 2) * (CT_W + 2) * (CK / 4); i += 256) {
      int q = i % (CK / 4);
      int p = i / (CK / 4);
      int py = p / (CT_W + 2), px = p % (CT_W + 2);
      int yy = y0 + py - 1, xx = x0 + px - 1;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy >= 0 && yy < H && xx >= 0 && xx < W)
        v = *reinterpret_cast<const float4*>(in + ((size_t)yy * W + xx) * Cin + c0 + q * 4);
      *reinterpret_cast<float4*>(&in_s[p * CKP + q * 4]) = v;
    }
    // weights [tap][c0..c0+CK)[co0..co0+64)
    for (int i = t; i < 9 * CK * 16; i += 256) {
      int q = i & 15;
      int k = (i >> 4) % CK;
      int tap = i / (16 * CK);
      *reinterpret_cast<float4*>(&w_s[(tap * CK + k) * 64 + q * 4]) =
          *reinterpret_cast<const float4*>(wt + ((size_t)tap * Cin + c0 + k) * Cout + co0 + q * 4);
    }
    __syncthreads();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3, dx = tap % 3;
#pragma unroll
      for (int k4 = 0; k4 < CK / 4; ++k4) {
        float4 wv[4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wv[kk] = *reinterpret_cast<const float4*>(&w_s[(tap * CK + k4 * 4 + kk) * 64 + cg * 4]);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float4 a = *reinterpret_cast<const float4*>(
                &in_s[((prow + i + dy) * (CT_W + 2) + (pcol + j + dx)) * CKP + k4 * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
              acc[i][j][0] = fmaf(av[kk], wv[kk].x, acc[i][j][0]);
              acc[i][j][1] = fmaf(av[kk], wv[kk].y, acc[i][j][1]);
              acc[i][j][2] = fmaf(av[kk], wv[kk].z, acc[i][j][2]);
              acc[i][j][3] = fmaf(av[kk], wv[kk].w, acc[i][j][3]);
            }
          }
        }
      }
    }
    __syncthreads();
  }
  const float4 bv = *reinterpret_cast<const float4*>(bias + co0 + cg * 4);
  const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
  if (POOL == 0) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int yy = y0 + prow + i, xx = x0 + pcol + j;
        if (yy < H && xx < W) {
          float4 o = make_float4(fmaxf(acc[i][j][0] + bb[0], 0.f), fmaxf(acc[i][j][1] + bb[1], 0.f),
                                 fmaxf(acc[i][j][2] + bb[2], 0.f), fmaxf(acc[i][j][3] + bb[3], 0.f));
          *reinterpret_cast<float4*>(out + ((size_t)yy * W + xx) * Cout + co0 + cg * 4) = o;
        }
      }
  } else {
    const int Ho = H >> 1, Wo = W >> 1;
    const int yo = (y0 + prow) >> 1;
#pragma unroll
    for (int jp = 0; jp < 2; ++jp) {
      int xo = ((x0 + pcol) >> 1) + jp;
      if (yo < Ho && xo < Wo) {
        float o[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float m = fmaxf(fmaxf(acc[0][2 * jp][c], acc[0][2 * jp + 1][c]), fmaxf(acc[1][2 * jp][c], acc[1][2 * jp + 1][c]));
          o[c] = fmaxf(m + bb[c], 0.f);  // max commutes with the monotone bias-add + ReLU
        }
        *reinterpret_cast<float4*>(out + ((size_t)yo * Wo + xo) * Cout + co0 + cg * 4) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// convPb (1x1, 256 -> 65) + softmax over 65 + drop dustbin + depth-to-space (superpoint.py:162-166).
// block = 128 threads, 16 cells.
constexpr int PB_CELLS = 16;
__global__ void __launch_bounds__(128) k_head_scores(const float* __restrict__ cpa /*[cells][256]*/,
                                                      const float* __restrict__ wt /*[256][65]*/,
                                                      const float* __restrict__ bias, float* __restrict__ heat, int Hc,
                                                      int Wc) {
  __shared__ float xs[PB_CELLS][256];
  __shared__ float lg[PB_CELLS][66];
  const int t = threadIdx.x;
  const int ncell = Hc * Wc;
  const int cell0 = blockIdx.x * PB_CELLS;
  for (int i = t; i < PB_CELLS * 64; i += 128) {
    int c = i >> 6, q = i & 63;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cell0 + c < ncell) v = *reinterpret_cast<const float4*>(cpa + (size_t)(cell0 + c) * 256 + q * 4);
    *reinterpret_cast<float4*>(&xs[c][q * 4]) = v;
  }
  __syncthreads();
  if (t < 65) {
    float acc[PB_CELLS];
    const float b = bias[t];
#pragma unroll
    for (int c = 0; c < PB_CELLS; ++c) acc[c] = b;
    for (int k = 0; k < 256; ++k) {
      float w = wt[k * 65 + t];
#pragma unroll
      for (int c = 0; c < PB_CELLS; ++c) acc[c] = fmaf(xs[c][k], w, acc[c]);
    }
#pragma unroll
    for (int c = 0; c < PB_CELLS; ++c) lg[c][t] = acc[c];
  }
  __syncthreads();
  const int warp = t >> 5, lane = t & 31;
  for (int c = warp; c < PB_CELLS; c += 4) {
    int cell = cell0 + c;
    if (cell >= ncell) break;
    float v0 = lg[c][lane], v1 = lg[c][lane + 32], v2 = lane == 0 ? lg[c][64] : -INFINITY;
    float m = warp_max(fmaxf(fmaxf(v0, v1), v2));
    float e0 = expf(v0 - m), e1 = expf(v1 - m), e2 = lane == 0 ? expf(v2 - m) : 0.f;
    float s = warp_sum(e0 + e1 + e2);
    int r = cell / Wc, cc = cell % Wc;
    int W8 = Wc * 8;
    // channel k -> pixel (8r + k/8, 8c + k%8)
    heat[(size_t)(8 * r + (lane >> 3)) * W8 + 8 * cc + (lane & 7)] = e0 / s;
    heat[(size_t)(8 * r + 4 + (lane >> 3)) * W8 + 8 * cc + (lane & 7)] = e1 / s;
  }
}

// wgmma path of the two 1x1 heads: the channel mixing runs on k_gemm_ws (linear.cuh), these finish the job.
// softmax over the 65 logits of a cell, drop the dustbin, depth-to-space (superpoint.py:162-166): one warp per cell.
__global__ void __launch_bounds__(256) k_head_softmax(const float* __restrict__ logits, int ld, float* __restrict__ heat, int Hc, int Wc) {
  const int cell = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (cell >= Hc * Wc) return;
  const float* lg = logits + (size_t)cell * ld;
  const float v0 = lg[lane], v1 = lg[lane + 32], v2 = lane == 0 ? lg[64] : -INFINITY;
  const float m = warp_max(fmaxf(fmaxf(v0, v1), v2));
  const float e0 = expf(v0 - m), e1 = expf(v1 - m), e2 = lane == 0 ? expf(v2 - m) : 0.f;
  const float s = warp_sum(e0 + e1 + e2);
  const int r = cell / Wc, cc = cell % Wc, W8 = Wc * 8;
  heat[(size_t)(8 * r + (lane >> 3)) * W8 + 8 * cc + (lane & 7)] = e0 / s;  // channel k -> pixel (8r + k/8, 8c + k%8)
  heat[(size_t)(8 * r + 4 + (lane >> 3)) * W8 + 8 * cc + (lane & 7)] = e1 / s;
}
// per-cell L2 normalisation of the dense descriptor map, in place (superpoint.py:192): one warp per cell
__global__ void __launch_bounds__(256) k_head_l2norm(float* __restrict__ dense, int ncell) {
  const int cell = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (cell >= ncell) return;
  float4* p = reinterpret_cast<float4*>(dense + (size_t)cell * 256);
  float4 a = p[lane], b = p[lane + 32];
  const float ss = warp_sum(a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w + b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w);
  const float nrm = fmaxf(sqrtf(ss), 1e-12f);
  p[lane] = make_float4(a.x / nrm, a.y / nrm, a.z / nrm, a.w / nrm);
  p[lane + 32] = make_float4(b.x / nrm, b.y / nrm, b.z / nrm, b.w / nrm);
}

// simple_nms with radius 4 (superpoint.py:47-62), fused over a tile with a 20-pixel halo, followed by the
// threshold + border test (superpoint.py:170-178) feeding per-row keypoint counts.
// tile 64 x 40: a VGA score map is 10 x 12 = 120 tiles = ONE wave of 1-CTA-per-SM blocks (64 x 32 gives 150 tiles = two waves on
// 132 SMs)
constexpr int NT_W = 64, NT_H = 40, NR = 4, NHALO = 5 * NR;
constexpr int NRW = NT_W + 2 * NHALO, NRH = NT_H + 2 * NHALO;  // 104 x 80 region = tile + the 20-px halo the five pools need
constexpr int NREG = NRW * NRH;
// shared-memory planes carry a 4-cell sentinel frame (-inf for scores, 0 for masks) so that every 9-tap window is a fixed,
// fully unrolled run of 9 loads with no bounds logic: pitch 112, 88 rows
constexpr int NPW = NRW + 2 * NR, NPH = NRH + 2 * NR;
constexpr int NPLANE = NPW * NPH;
constexpr int NMS_THREADS = 1024;
__device__ __forceinline__ int nms_idx(int c) {  // region cell c (row-major 104 x 80) -> index inside a padded plane
  const int y = c / NRW, x = c - y * NRW;
  return (y + NR) * NPW + x + NR;
}
// separable 9 x 9 max (F.max_pool2d(kernel 9, stride 1, padding 4), -inf padding) over the region
__device__ __forceinline__ void pool9_f(const float* __restrict__ src, float* __restrict__ tmp, float* __restrict__ dst) {
  for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
    const int i = nms_idx(c);
    float m = src[i - 4];
#pragma unroll
    for (int d = -3; d <= 4; ++d) m = fmaxf(m, src[i + d]);
    tmp[i] = m;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
    const int i = nms_idx(c);
    float m = tmp[i - 4 * NPW];
#pragma unroll
    for (int d = -3; d <= 4; ++d) m = fmaxf(m, tmp[i + d * NPW]);
    dst[i] = m;
  }
  __syncthreads();
}
__device__ __forceinline__ void dilate9_b(const uint8_t* __restrict__ src, uint8_t* __restrict__ tmp, uint8_t* __restrict__ dst) {
  for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
    const int i = nms_idx(c);
    unsigned m = src[i - 4];
#pragma unroll
    for (int d = -3; d <= 4; ++d) m |= src[i + d];
    tmp[i] = (uint8_t)m;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
    const int i = nms_idx(c);
    unsigned m = tmp[i - 4 * NPW];
#pragma unroll
    for (int d = -3; d <= 4; ++d) m |= tmp[i + d * NPW];
    dst[i] = (uint8_t)m;
  }
  __syncthreads();
}

// simple_nms(scores, 4) (superpoint.py:47-62) fused with the threshold / border test and the per-row survivor counts: one
// pass over a 64 x 40 tile whose 20-px halo makes the three rounds of 9 x 9 pools local.  1024 threads (32 warps hide the
// shared-memory latency of the unrolled 9-tap runs); float equality compares exactly as the reference does.
__global__ void __launch_bounds__(NMS_THREADS) k_nms(const float* __restrict__ heat, float* __restrict__ nms, int H8, int W8,
                                                      float thr, int border, int* __restrict__ rowcnt) {
  extern __shared__ __align__(16) unsigned char smraw[];
  float* S = reinterpret_cast<float*>(smraw);  // scores (-inf outside the image)
  float* T = S + NPLANE;                       // suppressed scores
  float* X = T + NPLANE;                       // pooled scores
  float* T2 = X + NPLANE;                      // row-pass scratch
  uint8_t* M = reinterpret_cast<uint8_t*>(T2 + NPLANE);  // max_mask
  uint8_t* P = M + NPLANE;                               // scratch
  uint8_t* Q = P + NPLANE;                               // supp_mask
  const int x0 = blockIdx.x * NT_W - NHALO, y0 = blockIdx.y * NT_H - NHALO;
  for (int i = threadIdx.x; i < NPLANE; i += NMS_THREADS) {  // sentinel frames (the region cells are overwritten below)
    S[i] = -INFINITY, T[i] = -INFINITY, T2[i] = -INFINITY;
    M[i] = 0, P[i] = 0;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
    const int ry = c / NRW, rx = c - ry * NRW;
    const int x = x0 + rx, y = y0 + ry;
    S[nms_idx(c)] = (x >= 0 && x < W8 && y >= 0 && y < H8) ? heat[(size_t)y * W8 + x] : -INFINITY;
  }
  __syncthreads();
  pool9_f(S, T2, X);
  for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
    const int i = nms_idx(c);
    M[i] = (S[i] != -INFINITY && S[i] == X[i]) ? 1 : 0;  // (outside the image S = -inf: never a maximum)
  }
  __syncthreads();
  for (int it = 0; it < 2; ++it) {
    dilate9_b(M, P, Q);  // supp_mask = max_pool(max_mask) > 0
    for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
      const int i = nms_idx(c);
      T[i] = Q[i] ? (S[i] == -INFINITY ? -INFINITY : 0.f) : S[i];
    }
    __syncthreads();
    pool9_f(T, T2, X);  // supp_scores in T, pooled into X
    for (int c = threadIdx.x; c < NREG; c += NMS_THREADS) {
      const int i = nms_idx(c);
      const bool fresh = (T[i] == X[i]) && !Q[i] && S[i] != -INFINITY;
      M[i] = M[i] | (fresh ? 1 : 0);
    }
    __syncthreads();
  }
  // central tile: where(max_mask, scores, 0) + count survivors of threshold / border per row
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < NT_W * NT_H; i += NMS_THREADS) {
    int tx = i % NT_W, ty = i / NT_W;
    int x = blockIdx.x * NT_W + tx, y = blockIdx.y * NT_H + ty;
    bool inside = x < W8 && y < H8;
    float v = 0.f;
    if (inside) {
      int r = (ty + NHALO + NR) * NPW + tx + NHALO + NR;
      v = M[r] ? S[r] : 0.f;
      nms[(size_t)y * W8 + x] = v;
    }
    bool kp = inside && v > thr && y >= border && y < H8 - border && x >= border && x < W8 - border;
    unsigned m = __ballot_sync(0xffffffffu, kp);
    if (lane == 0 && m) atomicAdd(&rowcnt[y], __popc(m));  // a warp covers 32 consecutive x of one row (NT_W = 64)
  }
}

// exclusive scan of per-row counts (H8 <= a few thousand): single block.
__global__ void __launch_bounds__(1024) k_scan_rows(const int* __restrict__ cnt, int* __restrict__ off, int n) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    int i = base + threadIdx.x;
    int v = i < n ? cnt[i] : 0;
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int u = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += u;
    }
    if (lane == 31) warp_tot[warp] = s;
    __syncthreads();
    if (warp == 0) {
      int w = warp_tot[lane];
      int ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int u = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += u;
      }
      warp_tot[lane] = ws - w;  // exclusive
    }
    __syncthreads();
    int excl = carry + warp_tot[warp] + s - v;
    if (i < n) off[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) off[n] = carry;
}

// ordered compaction: one warp per row, keypoints in ascending x; (x, y) float pairs (superpoint.py:187 flip).
__global__ void __launch_bounds__(256) k_compact(const float* __restrict__ nms, int H8, int W8, float thr, int border,
                                                  const int* __restrict__ rowoff, float* __restrict__ xy,
                                                  float* __restrict__ score, int cap) {
  int y = blockIdx.x * 8 + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (y >= H8 || y < border || y >= H8 - border) return;
  int off = rowoff[y];
  if (rowoff[y + 1] == off) return;
  for (int xb = 0; xb < W8; xb += 32) {
    int x = xb + lane;
    float v = x < W8 ? nms[(size_t)y * W8 + x] : 0.f;
    bool kp = v > thr && x >= border && x < W8 - border;
    unsigned m = __ballot_sync(0xffffffffu, kp);
    if (kp) {
      int pos = off + __popc(m & ((1u << lane) - 1));
      if (pos < cap) {
        xy[2 * (size_t)pos] = (float)x;
        xy[2 * (size_t)pos + 1] = (float)y;
        score[pos] = v;
      }
    }
    off += __popc(m);
  }
}

// convDb (1x1, 256 -> 256) + L2 normalise over channels (superpoint.py:191-192). block = 256 threads (one per
// output channel), 8 cells.
constexpr int DB_CELLS = 8;
__global__ void __launch_bounds__(256) k_head_desc(const float* __restrict__ cda, const float* __restrict__ wt /*[256][256]*/,
                                                    const float* __restrict__ bias, float* __restrict__ dense, int ncell) {
  __shared__ float xs[DB_CELLS][256];
  __shared__ float red[DB_CELLS][8];
  const int t = threadIdx.x;
  const int cell0 = blockIdx.x * DB_CELLS;
  for (int c = 0; c < DB_CELLS; ++c) xs[c][t] = (cell0 + c < ncell) ? cda[(size_t)(cell0 + c) * 256 + t] : 0.f;
  __syncthreads();
  float acc[DB_CELLS];
  const float b = bias[t];
#pragma unroll
  for (int c = 0; c < DB_CELLS; ++c) acc[c] = b;
  for (int k = 0; k < 256; ++k) {
    float w = wt[k * 256 + t];
#pragma unroll
    for (int c = 0; c < DB_CELLS; ++c) acc[c] = fmaf(xs[c][k], w, acc[c]);
  }
  const int warp = t >> 5, lane = t & 31;
#pragma unroll
  for (int c = 0; c < DB_CELLS; ++c) {
    float s = warp_sum(acc[c] * acc[c]);
    if (lane == 0) red[c][warp] = s;
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < DB_CELLS; ++c) {
    float ss = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) ss += red[c][w];
    float nrm = fmaxf(sqrtf(ss), 1e-12f);
    if (cell0 + c < ncell) dense[(size_t)(cell0 + c) * 256 + t] = acc[c] / nrm;
  }
}

// sample_descriptors (superpoint.py:80-92) with align_corners=True, zero padding, then per-keypoint L2 normalise.
// one warp per keypoint; each lane owns 8 channels (2 x float4).
__global__ void __launch_bounds__(256) k_sample_desc(const float* __restrict__ dense, int Hc, int Wc,
                                                      const float* __restrict__ xy, int n, const int* __restrict__ n_dev, float* __restrict__ out) {
  int kp = blockIdx.x * 8 + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (n_dev) n = min(n, *n_dev);
  if (kp >= n) return;
  float x = xy[2 * (size_t)kp], y = xy[2 * (size_t)kp + 1];
  // keypoints - s/2 + 0.5 ; / (w*s - s/2 - 0.5) ; *2 - 1 ; grid_sample unnormalise ((g + 1) / 2) * (size - 1)
  float gx = ((x - 4.0f) + 0.5f) / (float)(Wc * 8 - 4 - 0.5);
  float gy = ((y - 4.0f) + 0.5f) / (float)(Hc * 8 - 4 - 0.5);
  gx = gx * 2.0f - 1.0f;
  gy = gy * 2.0f - 1.0f;
  float ix = ((gx + 1.0f) / 2.0f) * (float)(Wc - 1);
  float iy = ((gy + 1.0f) / 2.0f) * (float)(Hc - 1);
  float fx = floorf(ix), fy = floorf(iy);
  int x0 = (int)fx, y0 = (int)fy;
  float wx1 = ix - fx, wy1 = iy - fy;
  float wx0 = (fx + 1.0f) - ix, wy0 = (fy + 1.0f) - iy;
  float wgt[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};  // nw, ne, sw, se
  int cxs[4] = {x0, x0 + 1, x0, x0 + 1};
  int cys[4] = {y0, y0, y0 + 1, y0 + 1};
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (cxs[q] >= 0 && cxs[q] < Wc && cys[q] >= 0 && cys[q] < Hc) {
      const float4* p = reinterpret_cast<const float4*>(dense + ((size_t)cys[q] * Wc + cxs[q]) * 256);
      float4 a = p[lane], b = p[lane + 32];
      v[0] = fmaf(a.x, wgt[q], v[0]);
      v[1] = fmaf(a.y, wgt[q], v[1]);
      v[2] = fmaf(a.z, wgt[q], v[2]);
      v[3] = fmaf(a.w, wgt[q], v[3]);
      v[4] = fmaf(b.x, wgt[q], v[4]);
      v[5] = fmaf(b.y, wgt[q], v[5]);
      v[6] = fmaf(b.z, wgt[q], v[6]);
      v[7] = fmaf(b.w, wgt[q], v[7]);
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) ss = fmaf(v[c], v[c], ss);
  ss = warp_sum(ss);
  float nrm = fmaxf(sqrtf(ss), 1e-12f);
  float4* o = reinterpret_cast<float4*>(out + (size_t)kp * 256);
  o[lane] = make_float4(v[0] / nrm, v[1] / nrm, v[2] / nrm, v[3] / nrm);
  o[lane + 32] = make_float4(v[4] / nrm, v[5] / nrm, v[6] / nrm, v[7] / nrm);
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------

static int sp_conv3x3(b2_context* ctx, cudaStream_t st, const float* in, int li, float* out, int H, int W, bool pool) {
  SuperPointState* s = ctx->sp;
  dim3 grid(cdiv(W, CT_W), cdiv(H, CT_H), SP_CO[li] / 64);
  b2_prof_work(ctx, "k_conv3x3", 2.0 * 9.0 * H * W * SP_CI[li] * SP_CO[li]);
  if (pool)
    B2_LAUNCH(ctx, k_conv3x3<1>, grid, 256, 0, st, in, s->w[li], s->b[li], out, H, W, SP_CI[li], SP_CO[li]);
  else
    B2_LAUNCH(ctx, k_conv3x3<0>, grid, 256, 0, st, in, s->w[li], s->b[li], out, H, W, SP_CI[li], SP_CO[li]);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// wgmma implicit-GEMM convolution on split-fp16 NHWC planes (conv_ps.cuh: persistent, halo reuse, resident weights).
// `in` / `out` buffers hold the hi plane followed by the lo plane (+ pixels * channels halves).
static int sp_conv3x3_tc(b2_context* ctx, cudaStream_t st, const DevBuf& in, int li, int H, int W, bool pool, DevBuf* out_planes,
                         float* out_f32) {
  SuperPointState* s = ctx->sp;
  const int Cin = SP_CI[li], Cout = SP_CO[li];
  const int OH = pool ? H / 2 : H, OW = pool ? W / 2 : W;
  const __half* ih = in.as<__half>();
  const __half* il = ih + (size_t)H * W * Cin;
  const __half* wh = s->wsplit_h.as<__half>() + s->wsoff[li];
  const __half* wl = s->wsplit_l.as<__half>() + s->wsoff[li];
  SuperPointState::ConvMapCache& mc = s->conv_maps[li];  // the maps only change with the image size / a reallocation
  if (mc.ih != ih || mc.wh != wh || mc.H != H || mc.W != W) {
    bool ok = tma_map_nhwc_halo(&mc.maps.ah, ih, H, W, Cin) && tma_map_nhwc_halo(&mc.maps.al, il, H, W, Cin) &&
              tma_map_2d(&mc.maps.wh, wh, Cout, 9 * Cin, 9 * Cin, 64) && tma_map_2d(&mc.maps.wl, wl, Cout, 9 * Cin, 9 * Cin, 64);
    if (!ok) return b2_fail(ctx, B2_ERR_CUDA, "cuTensorMapEncodeTiled failed (conv)");
    mc.ih = ih, mc.wh = wh, mc.H = H, mc.W = W;
  }
  const ConvPsMaps& maps = mc.maps;
  ConvPsArgs a{};
  a.H = H, a.W = W, a.Cin = Cin, a.Cout = Cout, a.pool = pool ? 1 : 0, a.relu = 1, a.bias = s->b[li];
  if (out_planes) a.Oh = out_planes->as<__half>(), a.Ol = a.Oh + (size_t)OH * OW * Cout;
  a.Of = out_f32, a.err_flag = s->errflag.as<int>();
  if (getenv("B2_CONV_DBG")) {  // profiling runs: per-CTA timestamps of layer li, read back through b2_debug_fetch("conv_dbg")
    const size_t per_layer = (size_t)ctx->sm_count * 8;
    if (s->conv_dbg.ensure(12 * per_layer * sizeof(float)) == cudaSuccess) {
      a.dbg = s->conv_dbg.as<float>() + li * per_layer;
      ctx->debug["conv_dbg"] = {s->conv_dbg.as<float>(), (int64_t)(12 * per_layer)};
    }
  }
  const int nblk = Cout / 64, units = cdiv(W, CP_TW) * cdiv(H, CP_TH) * nblk;
  int grid = ctx->sm_count < units ? ctx->sm_count : units;
  grid -= grid % nblk;  // a CTA keeps one 64-channel block of the weights resident: CTA c serves block c % nblk
  b2_prof_work(ctx, "k_conv_ps", 2.0 * 9.0 * H * W * Cin * Cout);
  B2_LAUNCH(ctx, k_conv_ps<1>, grid, CP_THREADS, CP_SMEM, st, maps, a);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// 1x1 head (convPb / convDb) on the shared wgmma GEMM: out[cell][n] = sum_k in[cell][k] * W[n][k] + bias[n]  (fp32-equivalent)
static int sp_head_gemm(b2_context* ctx, cudaStream_t st, const DevBuf& in_planes, int li, int cells, float* out, int ldc) {
  SuperPointState* s = ctx->sp;
  const int K = SP_CI[li], N = SP_CO[li];
  TcWeights tw{nullptr, nullptr, nullptr, s->errflag.as<int>(), true};
  tw.sm_count = ctx->sm_count;
  LinArgs a;
  a.a1p = {in_planes.as<__half>(), in_planes.as<__half>() + (size_t)cells * K}, a.lda1 = K, a.K1 = K;
  a.bp = {s->wsplit_h.as<__half>() + s->wsoff[li], s->wsplit_l.as<__half>() + s->wsoff[li]}, a.ldb = K;
  a.bias = s->b[li], a.cf = out, a.ldc = ldc, a.tc_want_f32 = true, a.M = cells, a.N = N;
  return run_linear(ctx, st, tw, &a, 1);
}

static size_t nms_smem_bytes() { return (size_t)NPLANE * 4 * sizeof(float) + (size_t)NPLANE * 3; }

extern "C" int b2_superpoint_set_weights(b2_context* ctx, const float* blob, size_t n_floats) {
  if (!ctx || !blob) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (n_floats != SP_NFLOATS)
    return b2_fail(ctx, B2_ERR_ARG, "superpoint blob must hold 1300865 floats, got " + std::to_string(n_floats));
  cudaSetDevice(ctx->device);
  if (!ctx->sp) ctx->sp = new SuperPointState();
  SuperPointState* s = ctx->sp;
  // repack on host: 3x3 OIHW -> [tap][cin][cout]; 1x1 OI -> [cin][cout]
  std::vector<float> packed(SP_NFLOATS);
  size_t src = 0, dst = 0;
  size_t woff[SP_NCONV], boff[SP_NCONV];
  for (int l = 0; l < SP_NCONV; ++l) {
    const int co = SP_CO[l], ci = SP_CI[l], kk = SP_K[l] * SP_K[l];
    const float* w = blob + src;
    woff[l] = dst;
    for (int o = 0; o < co; ++o)
      for (int i = 0; i < ci; ++i)
        for (int tp = 0; tp < kk; ++tp) packed[dst + ((size_t)tp * ci + i) * co + o] = w[((size_t)o * ci + i) * kk + tp];
    src += (size_t)co * ci * kk;
    dst += (size_t)co * ci * kk;
    boff[l] = dst;
    for (int o = 0; o < co; ++o) packed[dst + o] = blob[src + o];
    src += co;
    dst += co;
    // keep every tensor 16-byte aligned for float4 loads: all sizes are multiples of 4 except convPb (65 outputs)
  }
  // alignment: lay tensors out individually aligned to 256 B on the device
  size_t total = 0;
  size_t dwoff[SP_NCONV], dboff[SP_NCONV];
  for (int l = 0; l < SP_NCONV; ++l) {
    size_t nw = (size_t)SP_CO[l] * SP_CI[l] * SP_K[l] * SP_K[l];
    dwoff[l] = total;
    total += (nw + 63) / 64 * 64;
    dboff[l] = total;
    total += ((size_t)SP_CO[l] + 63) / 64 * 64;
  }
  B2_CUDA(ctx, s->wblob.ensure(total * sizeof(float)));
  for (int l = 0; l < SP_NCONV; ++l) {
    size_t nw = (size_t)SP_CO[l] * SP_CI[l] * SP_K[l] * SP_K[l];
    s->w[l] = s->wblob.as<float>() + dwoff[l];
    s->b[l] = s->wblob.as<float>() + dboff[l];
    B2_CUDA(ctx, cudaMemcpy(s->w[l], packed.data() + woff[l], nw * sizeof(float), cudaMemcpyHostToDevice));
    B2_CUDA(ctx, cudaMemcpy(s->b[l], packed.data() + boff[l], SP_CO[l] * sizeof(float), cudaMemcpyHostToDevice));
  }
  // wgmma path: [cout][tap * cin + ci] fp32 -> split planes (one device split kernel over a host-built fp32 staging copy)
  {
    size_t tot = 0;
    for (int l = 0; l < SP_NCONV; ++l) {
      s->wsoff[l] = tot;
      if (SP_K[l] == 3 && SP_CI[l] >= 64) tot += (size_t)SP_CO[l] * 9 * SP_CI[l];
      if (SP_K[l] == 1) tot += (size_t)SP_CO[l] * SP_CI[l];  // 1x1 heads: [cout][cin], the checkpoint's own order
    }
    std::vector<float> stage(tot);
    size_t src2 = 0;
    for (int l = 0; l < SP_NCONV; ++l) {
      const int co = SP_CO[l], ci = SP_CI[l], kk = SP_K[l] * SP_K[l];
      if (SP_K[l] == 3 && ci >= 64) {
        const float* w = blob + src2;  // OIHW
        float* d = stage.data() + s->wsoff[l];
        for (int o = 0; o < co; ++o)
          for (int tp = 0; tp < 9; ++tp)
            for (int i = 0; i < ci; ++i) d[(size_t)o * 9 * ci + tp * ci + i] = w[((size_t)o * ci + i) * 9 + tp];
      } else if (SP_K[l] == 1) {
        std::copy(blob + src2, blob + src2 + (size_t)co * ci, stage.data() + s->wsoff[l]);
      }
      src2 += (size_t)co * ci * kk + co;
    }
    DevBuf tmp;
    B2_CUDA(ctx, tmp.ensure(tot * sizeof(float)));
    B2_CUDA(ctx, s->wsplit_h.ensure(tot * sizeof(__half)));
    B2_CUDA(ctx, s->wsplit_l.ensure(tot * sizeof(__half)));
    B2_CUDA(ctx, s->errflag.ensure(16));
    B2_CUDA(ctx, cudaMemset(s->errflag.p, 0, 16));
    B2_CUDA(ctx, cudaMemcpy(tmp.p, stage.data(), tot * sizeof(float), cudaMemcpyHostToDevice));
    B2_LAUNCH(ctx, k_split_f32, (unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)0, tmp.as<float>(), tot, s->wsplit_h.as<__half>(),
              s->wsplit_l.as<__half>());
    B2_CHECK_LAUNCH(ctx);
    B2_CUDA(ctx, cudaDeviceSynchronize());
    tmp.release();
    B2_CUDA(ctx, cudaFuncSetAttribute(k_conv_ps<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CP_SMEM));
    B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
    s->use_tc = !b2_force_simt(ctx) && tma_encoder() != nullptr;
  }
  B2_CUDA(ctx, cudaFuncSetAttribute(k_nms, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nms_smem_bytes()));
  s->loaded = true;
  return B2_OK;
}

// Everything between the grey image and the compacted keypoint list + dense descriptor map, enqueued on `st`.  Buffers are
// sized by the caller; the sequence is a pure function of (H, W, thr, border, cap, output pointers), which is what lets
// sp_detect_impl replay it as a CUDA graph.
static int sp_enqueue_network(b2_context* ctx, cudaStream_t st, int H, int W, float thr, int border, float* out_xy, float* out_score, int cap) {
  SuperPointState* s = ctx->sp;
  const int H2 = H / 2, W2 = W / 2, H4 = H2 / 2, W4 = W2 / 2, Hc = H4 / 2, Wc = W4 / 2;
  const int H8 = Hc * 8, W8 = Wc * 8;
  const size_t px = (size_t)H * W;
  float* a0 = s->a0.as<float>();
  float* a1 = s->a1.as<float>();
  float* feat = s->feat.as<float>();
  float* head = s->head.as<float>();
  int rc;
  const bool tcp = s->use_tc;
  DevBuf& featp = s->kpxy;  // (wgmma path) split planes of conv4b's output: operand of convPa and convDa
  if (tcp) {
    __half* p0 = s->a0.as<__half>();
    B2_LAUNCH(ctx, k_conv1a, (unsigned)(ctx->sm_count * 8), C1A_THREADS, 0, st, s->gray.as<uint8_t>(), s->w[0], s->b[0], a0, H, W, p0, p0 + px * 64);
    B2_CHECK_LAUNCH(ctx);
    // encoder (superpoint.py:148-158) as TMA-fed wgmma implicit GEMMs on split-fp16 planes; pools fused
    if ((rc = sp_conv3x3_tc(ctx, st, s->a0, 1, H, W, true, &s->a1, nullptr))) return rc;      // conv1b + pool
    if ((rc = sp_conv3x3_tc(ctx, st, s->a1, 2, H2, W2, false, &s->a0, nullptr))) return rc;   // conv2a
    if ((rc = sp_conv3x3_tc(ctx, st, s->a0, 3, H2, W2, true, &s->a1, nullptr))) return rc;    // conv2b + pool
    if ((rc = sp_conv3x3_tc(ctx, st, s->a1, 4, H4, W4, false, &s->a0, nullptr))) return rc;   // conv3a
    if ((rc = sp_conv3x3_tc(ctx, st, s->a0, 5, H4, W4, true, &s->a1, nullptr))) return rc;    // conv3b + pool
    if ((rc = sp_conv3x3_tc(ctx, st, s->a1, 6, Hc, Wc, false, &s->a0, nullptr))) return rc;   // conv4a
    if ((rc = sp_conv3x3_tc(ctx, st, s->a0, 7, Hc, Wc, false, &featp, feat))) return rc;      // conv4b (planes + fp32)
    if ((rc = sp_conv3x3_tc(ctx, st, featp, 8, Hc, Wc, false, &s->head, nullptr))) return rc;  // convPa -> planes for the score head
  } else {
  B2_LAUNCH(ctx, k_conv1a, (unsigned)(ctx->sm_count * 8), C1A_THREADS, 0, st, s->gray.as<uint8_t>(), s->w[0], s->b[0], a0, H, W, (__half*)nullptr,
            (__half*)nullptr);
  B2_CHECK_LAUNCH(ctx);
  // encoder (superpoint.py:148-158); pools fused into conv1b / conv2b / conv3b
  if ((rc = sp_conv3x3(ctx, st, a0, 1, a1, H, W, true))) return rc;      // conv1b + pool -> (H2, W2, 64) in a1
  if ((rc = sp_conv3x3(ctx, st, a1, 2, a0, H2, W2, false))) return rc;   // conv2a
  if ((rc = sp_conv3x3(ctx, st, a0, 3, a1, H2, W2, true))) return rc;    // conv2b + pool -> (H4, W4, 64)
  if ((rc = sp_conv3x3(ctx, st, a1, 4, a0, H4, W4, false))) return rc;   // conv3a -> 128
  if ((rc = sp_conv3x3(ctx, st, a0, 5, a1, H4, W4, true))) return rc;    // conv3b + pool -> (Hc, Wc, 128)
  if ((rc = sp_conv3x3(ctx, st, a1, 6, a0, Hc, Wc, false))) return rc;   // conv4a
  if ((rc = sp_conv3x3(ctx, st, a0, 7, feat, Hc, Wc, false))) return rc; // conv4b
  // detector head (superpoint.py:161-167)
  if ((rc = sp_conv3x3(ctx, st, feat, 8, head, Hc, Wc, false))) return rc;  // convPa
  }
  if (tcp) {  // convPb as a GEMM (65 logits per cell, row pitch 68), then softmax + depth-to-space
    if ((rc = sp_head_gemm(ctx, st, s->head, 9, Hc * Wc, s->logits.as<float>(), 68))) return rc;
    B2_LAUNCH(ctx, k_head_softmax, cdiv(Hc * Wc, 8), 256, 0, st, s->logits.as<float>(), 68, s->heat.as<float>(), Hc, Wc);
  } else {
    B2_LAUNCH(ctx, k_head_scores, cdiv(Hc * Wc, PB_CELLS), 128, 0, st, head, s->w[9], s->b[9], s->heat.as<float>(), Hc, Wc);
  }
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaMemsetAsync(s->rowcnt.p, 0, (size_t)(H8 + 1) * sizeof(int), st));
  B2_LAUNCH(ctx, k_nms, dim3(cdiv(W8, NT_W), cdiv(H8, NT_H)), NMS_THREADS, nms_smem_bytes(), st, s->heat.as<float>(),
            s->nms.as<float>(), H8, W8, thr, border, s->rowcnt.as<int>());
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_scan_rows, 1, 1024, 0, st, s->rowcnt.as<int>(), s->rowoff.as<int>(), H8);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_compact, cdiv(H8, 8), 256, 0, st, s->nms.as<float>(), H8, W8, thr, border, s->rowoff.as<int>(), out_xy,
            out_score, cap);
  B2_CHECK_LAUNCH(ctx);
  // descriptor head (superpoint.py:190-192): dense map stays resident for the describe stage
  if (tcp) {
    if ((rc = sp_conv3x3_tc(ctx, st, featp, 10, Hc, Wc, false, &s->head, nullptr))) return rc;  // convDa -> planes
    if ((rc = sp_head_gemm(ctx, st, s->head, 11, Hc * Wc, s->dense.as<float>(), 256))) return rc;  // convDb
    B2_LAUNCH(ctx, k_head_l2norm, cdiv(Hc * Wc, 8), 256, 0, st, s->dense.as<float>(), Hc * Wc);
  } else {
    if ((rc = sp_conv3x3(ctx, st, feat, 10, head, Hc, Wc, false))) return rc;  // convDa
    B2_LAUNCH(ctx, k_head_desc, cdiv(Hc * Wc, DB_CELLS), 256, 0, st, head, s->w[11], s->b[11], s->dense.as<float>(), Hc * Wc);
  }
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// true when bench.py is timing (CUDA events per launch) a kernel that sp_enqueue_network launches: events cannot be placed
// inside a replayed graph, so those runs launch directly
static bool sp_prof_in_network(const ProfState& p) {
  if (!p.on) return false;
  static const char* const names[] = {"k_conv1a", "k_conv_ps", "k_gemm_ws", "k_head_softmax", "k_head_l2norm", "k_nms", "k_scan_rows", "k_compact"};
  for (const char* n : names)
    if (strncmp(n, p.name.c_str(), p.name.size()) == 0) return true;
  return false;
}

static int sp_detect_impl(b2_context* ctx, const uint8_t* image, int H, int W, int channels, size_t pitch, float thr,
                          int nms_radius, int border, float* out_xy, float* out_score, int cap, int* out_n,
                          cudaStream_t st, uint64_t* out_token = nullptr, bool defer_sync = false) {
  // defer_sync: enqueue only - the keypoint count stays on the device (rowoff[H8]) and the caller synchronises / checks the
  // error flag itself (b2_superpoint_extract_dev: one synchronisation per image instead of two)
  SuperPointState* s = ctx->sp;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "superpoint weights not set");
  if (nms_radius != NR) return b2_fail(ctx, B2_ERR_ARG, "only nms_radius == 4 (the reference default) is built");
  if (H < 8 || W < 8 || (channels != 1 && channels != 3 && channels != 4)) return b2_fail(ctx, B2_ERR_ARG, "bad image shape");
  if (border < 0) return b2_fail(ctx, B2_ERR_ARG, "border < 0");
  const int H2 = H / 2, W2 = W / 2, H4 = H2 / 2, W4 = W2 / 2, Hc = H4 / 2, Wc = W4 / 2;
  const int H8 = Hc * 8, W8 = Wc * 8;
  s->H = H, s->W = W, s->Hc = Hc, s->Wc = Wc;
  s->have_dense = false;
  const size_t px = (size_t)H * W;
  B2_CUDA(ctx, s->gray.ensure(px));
  B2_CUDA(ctx, s->a0.ensure(px * 64 * sizeof(float)));
  B2_CUDA(ctx, s->a1.ensure((size_t)H2 * W2 * 64 * sizeof(float)));
  B2_CUDA(ctx, s->feat.ensure((size_t)Hc * Wc * 128 * sizeof(float)));
  B2_CUDA(ctx, s->head.ensure((size_t)Hc * Wc * 256 * sizeof(float)));
  B2_CUDA(ctx, s->heat.ensure((size_t)H8 * W8 * sizeof(float)));
  B2_CUDA(ctx, s->nms.ensure((size_t)H8 * W8 * sizeof(float)));
  B2_CUDA(ctx, s->rowcnt.ensure((size_t)(H8 + 1) * sizeof(int)));
  B2_CUDA(ctx, s->rowoff.ensure((size_t)(H8 + 2) * sizeof(int)));
  B2_CUDA(ctx, s->dense.ensure((size_t)Hc * Wc * 256 * sizeof(float)));
  float* a0 = s->a0.as<float>();
  float* a1 = s->a1.as<float>();
  float* feat = s->feat.as<float>();
  float* head = s->head.as<float>();

  const bool tcp = s->use_tc;
  if (tcp) {
    B2_CUDA(ctx, s->kpxy.ensure((size_t)Hc * Wc * 128 * sizeof(float)));
    B2_CUDA(ctx, s->logits.ensure((size_t)Hc * Wc * 68 * sizeof(float)));
  }
  B2_LAUNCH(ctx, k_to_gray, dim3(cdiv(W, 256), H), 256, 0, st, image, pitch, channels, H, W, s->gray.as<uint8_t>());
  B2_CHECK_LAUNCH(ctx);
  // OPT-IN (b2_set_option "superpoint_graph" / B2_SP_GRAPH=1): the network's ~21 launches replayed as ONE CUDA graph per (shape,
  // parameters, buffers) key, captured on a private stream the first time the key is seen.  The host
  // enqueues faster than the GPU drains, so there is no launch gap for a graph to remove.  Direct launches when one of its kernels is being profiled, on the SIMT path, with
  // B2_SP_GRAPH=0, or when the key keeps changing (caller-owned output pointers that move on every call).
  int rc;
  SuperPointState::GraphSlot* hit = nullptr;
  bool use_graph = tcp && !sp_prof_in_network(ctx->prof) && !getenv("B2_CONV_DBG");
  if (use_graph) {
    if (ctx->sp_graph >= 0) {
      use_graph = ctx->sp_graph != 0;
    } else {
      const char* e = getenv("B2_SP_GRAPH");
      use_graph = e && e[0] == '1';  // default OFF: measured slower than direct launches (the path is GPU-bound, see below)
    }
  }
  if (use_graph) {
    const uint64_t key[SuperPointState::GKEY] = {(uint64_t)H, (uint64_t)W, (uint64_t)__float_as_uint_host(thr), (uint64_t)border, (uint64_t)cap,
        (uint64_t)(uintptr_t)out_xy, (uint64_t)(uintptr_t)out_score, (uint64_t)(uintptr_t)s->gray.p, (uint64_t)(uintptr_t)s->a0.p,
        (uint64_t)(uintptr_t)s->a1.p, (uint64_t)(uintptr_t)s->feat.p, (uint64_t)(uintptr_t)s->head.p, (uint64_t)(uintptr_t)s->heat.p,
        (uint64_t)(uintptr_t)s->nms.p, (uint64_t)(uintptr_t)s->rowcnt.p, (uint64_t)(uintptr_t)s->rowoff.p, (uint64_t)(uintptr_t)s->dense.p,
        (uint64_t)(uintptr_t)s->kpxy.p, (uint64_t)(uintptr_t)s->logits.p, (uint64_t)ctx->sm_count};
    for (auto& g : s->gslot)
      if (g.exec && memcmp(key, g.key, sizeof(key)) == 0) hit = &g;
    if (!hit) {
      if (s->gcaptures >= 256) {  // keys that never repeat (caller buffers moving every call): stop paying for captures
        use_graph = false;
      } else {
        if (!s->cap_stream) B2_CUDA(ctx, cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
        const uint64_t l0 = ctx->launches;
        B2_CUDA(ctx, cudaStreamBeginCapture(s->cap_stream, cudaStreamCaptureModeThreadLocal));
        rc = sp_enqueue_network(ctx, s->cap_stream, H, W, thr, border, out_xy, out_score, cap);
        cudaGraph_t graph = nullptr;
        const cudaError_t ce = cudaStreamEndCapture(s->cap_stream, &graph);
        const uint64_t nl = ctx->launches - l0;
        ctx->launches = l0;
        if (rc || ce != cudaSuccess || !graph) {
          if (graph) cudaGraphDestroy(graph);
          cudaGetLastError();
          return rc ? rc : b2_fail(ctx, B2_ERR_CUDA, std::string("CUDA graph capture of the SuperPoint network failed: ") + cudaGetErrorString(ce));
        }
        SuperPointState::GraphSlot& g = s->gslot[s->gnext];
        s->gnext = (s->gnext + 1) % SuperPointState::GSLOTS;
        if (g.exec) cudaGraphExecDestroy(g.exec), g.exec = nullptr;
        const cudaError_t ie = cudaGraphInstantiate(&g.exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) return b2_fail(ctx, B2_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ie));
        memcpy(g.key, key, sizeof(key));
        g.launches = nl;
        s->gcaptures++;
        hit = &g;
      }
    }
  }
  if (use_graph) {
    B2_CUDA(ctx, cudaGraphLaunch(hit->exec, st));
    ctx->launches += hit->launches;
  } else if ((rc = sp_enqueue_network(ctx, st, H, W, thr, border, out_xy, out_score, cap))) {
    return rc;
  }
  int n = 0, err = 0;
  if (!defer_sync) {
    B2_CUDA(ctx, cudaMemcpyAsync(&n, s->rowoff.as<int>() + H8, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (tcp) B2_CUDA(ctx, cudaMemcpyAsync(&err, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma conv pipeline timed out on an mbarrier (kernel bug)");
  }
  s->n_kp = n;
  s->have_dense = true;
  s->map_token += 1;
  if (out_token) *out_token = s->map_token;
  *out_n = n;
  ctx->debug["heat"] = {s->heat.as<float>(), (int64_t)H8 * W8};
  ctx->debug["nms"] = {s->nms.as<float>(), (int64_t)H8 * W8};
  ctx->debug["dense_desc"] = {s->dense.as<float>(), (int64_t)Hc * Wc * 256};
  ctx->debug["conv4b"] = {s->feat.as<float>(), (int64_t)Hc * Wc * 128};
  return B2_OK;
}

extern "C" int b2_superpoint_detect_dev(b2_context* ctx, const uint8_t* image, int H, int W, int channels, size_t pitch,
                                        float thr, int nms_radius, int border, float* out_xy, float* out_score, int cap,
                                        int* out_n, uint64_t* out_map_token, void* stream) {
  if (!ctx || !image || !out_xy || !out_score || !out_n || cap < 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return sp_detect_impl(ctx, image, H, W, channels, pitch, thr, nms_radius, border, out_xy, out_score, cap, out_n,
                        (cudaStream_t)stream, out_map_token);
}

static int sp_describe_impl(b2_context* ctx, uint64_t token, const float* xy, int n, float* out_desc, cudaStream_t st,
                            const int* n_dev = nullptr) {
  SuperPointState* s = ctx->sp;
  if (!s || !s->have_dense) return b2_fail(ctx, B2_ERR_STATE, "describe called before a successful detect");
  if (token != s->map_token)
    return b2_fail(ctx, B2_ERR_STATE, "stale feature-map token: another detect ran on this context since the token was issued");
  if (n == 0) return B2_OK;
  B2_LAUNCH(ctx, k_sample_desc, cdiv(n, 8), 256, 0, st, s->dense.as<float>(), s->Hc, s->Wc, xy, n, n_dev, out_desc);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

extern "C" int b2_superpoint_describe_dev(b2_context* ctx, uint64_t map_token, const float* xy, int n, float* out_desc, void* stream) {
  if (!ctx || n < 0 || (n > 0 && (!xy || !out_desc))) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return sp_describe_impl(ctx, map_token, xy, n, out_desc, (cudaStream_t)stream);
}

extern "C" int b2_superpoint_detect_host(b2_context* ctx, const uint8_t* image, int H, int W, int channels, float thr,
                                         int nms_radius, int border, float* out_xy, float* out_score, int cap,
                                         int* out_n, uint64_t* out_map_token) {
  if (!ctx || !image || !out_xy || !out_score || !out_n || cap < 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t bytes = (size_t)H * W * channels;
  B2_CUDA(ctx, ctx->stage_d[0].ensure(bytes));
  B2_CUDA(ctx, ctx->stage_d[1].ensure((size_t)cap * 2 * sizeof(float) + 16));
  B2_CUDA(ctx, ctx->stage_d[2].ensure((size_t)cap * sizeof(float) + 16));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->stage_d[0].p, image, bytes, cudaMemcpyHostToDevice, st));
  int rc = sp_detect_impl(ctx, ctx->stage_d[0].as<uint8_t>(), H, W, channels, (size_t)W * channels, thr, nms_radius, border,
                          ctx->stage_d[1].as<float>(), ctx->stage_d[2].as<float>(), cap, out_n, st, out_map_token);
  if (rc) return rc;
  int n = *out_n < cap ? *out_n : cap;
  if (n > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(out_xy, ctx->stage_d[1].p, (size_t)n * 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(out_score, ctx->stage_d[2].p, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return B2_OK;
}

extern "C" int b2_superpoint_describe_host(b2_context* ctx, uint64_t map_token, const float* xy, int n, float* out_desc) {
  if (!ctx || n < 0 || (n > 0 && (!xy || !out_desc))) return B2_ERR_ARG;
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  B2_CUDA(ctx, ctx->stage_d[3].ensure((size_t)n * 2 * sizeof(float)));
  B2_CUDA(ctx, ctx->stage_d[4].ensure((size_t)n * 256 * sizeof(float)));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->stage_d[3].p, xy, (size_t)n * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
  int rc = sp_describe_impl(ctx, map_token, ctx->stage_d[3].as<float>(), n, ctx->stage_d[4].as<float>(), st);
  if (rc) return rc;
  B2_CUDA(ctx, cudaMemcpyAsync(out_desc, ctx->stage_d[4].p, (size_t)n * 256 * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B2_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// device top-k for the batched path: the k largest scores (ties at the k-th value -> lowest indices), kept in their
// original (row-major) order (topk.cuh).  Single CTA: n is a few 10^4.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_topk_select(const float* __restrict__ score, int n, const int* __restrict__ n_dev, int k,
                                                       int* __restrict__ out_idx, int* __restrict__ out_count) {
  if (n_dev) n = min(n, *n_dev);  // candidate count still on the device (single-sync extract): n is then the capacity bound
  b2_topk_select_cta(score, n, k, out_idx, out_count);
}

extern "C" int b2_topk_indices_dev(b2_context* ctx, const float* scores, int n, int k, int32_t* out_idx, int* out_k,
                                   void* stream) {
  if (!ctx || !out_k || n < 0 || k < 0 || (n > 0 && (!scores || !out_idx))) return B2_ERR_ARG;
  *out_k = 0;
  if (n == 0 || k == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(ctx, ctx->stage_d[7].ensure(16));
  B2_LAUNCH(ctx, k_topk_select, 1, 1024, 0, st, scores, n, (const int*)nullptr, k, (int*)out_idx, ctx->stage_d[7].as<int>());
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaMemcpyAsync(out_k, ctx->stage_d[7].p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B2_OK;
}


// ------------------------------------------------------------------------------------------------------------------
// fused device-resident extraction for the batched path: detect -> top-k (device radix select, row-major order kept) ->
// gather -> describe in ONE call, one host synchronisation (the data-dependent count).  Replaces the host-side
// Keypoints.get_top_k of the per-call plugin (gtsfm/common/keypoints.py:89-110) by its order-preserving device twin.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_gather_kp(const float* __restrict__ xy, const float* __restrict__ sc, const int* __restrict__ idx,
                                                    const int* __restrict__ cnt, float* __restrict__ oxy, float* __restrict__ osc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *cnt) return;
  const int j = idx[i];
  reinterpret_cast<float2*>(oxy)[i] = reinterpret_cast<const float2*>(xy)[j];
  osc[i] = sc[j];
}

// detect -> device top-k -> describe, enqueued on `st` with NO host synchronisation: every count stays on the device
// (rowoff[H8] = candidates, sel_cnt = selected) and the kernels after the network read them there.
static int sp_extract_enqueue(b2_context* ctx, const uint8_t* image, int H, int W, int channels, size_t pitch, float thr, int nms_radius,
                              int border, int max_keypoints, float* out_xy, float* out_score, float* out_desc, cudaStream_t st) {
  SuperPointState* s = ctx->sp;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "superpoint weights not set");
  const int Hc = H / 8, Wc = W / 8;
  const int cap = (Hc * 8 / 5 + 1) * (Wc * 8 / 5 + 1);  // radius-4 maxima are >= 5 apart (Chebyshev)
  B2_CUDA(ctx, s->kpsc.ensure((size_t)cap * 3 * sizeof(float)));
  B2_CUDA(ctx, s->sel_idx.ensure((size_t)cap * sizeof(int)));
  B2_CUDA(ctx, s->sel_cnt.ensure(16));
  float* all_xy = s->kpsc.as<float>();
  float* all_sc = all_xy + (size_t)cap * 2;
  int unused = 0;
  uint64_t token = 0;
  int rc = sp_detect_impl(ctx, image, H, W, channels, pitch, thr, nms_radius, border, all_xy, all_sc, cap, &unused, st, &token, true);
  if (rc) return rc;
  const int* n_dev = s->rowoff.as<int>() + s->Hc * 8;
  const int kmax = cap < max_keypoints ? cap : max_keypoints;
  B2_LAUNCH(ctx, k_topk_select, 1, 1024, 0, st, all_sc, cap, n_dev, max_keypoints, s->sel_idx.as<int>(), s->sel_cnt.as<int>());
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_gather_kp, cdiv(kmax, 256), 256, 0, st, all_xy, all_sc, s->sel_idx.as<int>(), s->sel_cnt.as<int>(), out_xy, out_score);
  B2_CHECK_LAUNCH(ctx);
  return sp_describe_impl(ctx, token, out_xy, kmax, out_desc, st, s->sel_cnt.as<int>());
}

extern "C" int b2_superpoint_extract_dev(b2_context* ctx, const uint8_t* image, int H, int W, int channels, size_t pitch,
                                         float thr, int nms_radius, int border, int max_keypoints, float* out_xy, float* out_score,
                                         float* out_desc, int* out_n, void* stream) {
  if (!ctx || !image || !out_xy || !out_score || !out_desc || !out_n || max_keypoints <= 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  *out_n = 0;
  int rc = sp_extract_enqueue(ctx, image, H, W, channels, pitch, thr, nms_radius, border, max_keypoints, out_xy, out_score, out_desc, st);
  if (rc) return rc;
  SuperPointState* s = ctx->sp;
  int n = 0, err = 0;  // ONE synchronisation per image: the selected count and the pipeline error flag
  B2_CUDA(ctx, cudaMemcpyAsync(&n, s->sel_cnt.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma conv pipeline timed out on an mbarrier (kernel bug)");
  *out_n = n;
  return B2_OK;
}

// The same without any synchronisation: `out_n_pinned` (page-locked host int, one per image in flight) receives the count when
// the stream gets there.  Many images can be enqueued back to back (the work buffers are reused in stream order); call
// b2_superpoint_finish_dev before reading the counts or the outputs on the host.
extern "C" int b2_superpoint_extract_async_dev(b2_context* ctx, const uint8_t* image, int H, int W, int channels, size_t pitch,
                                               float thr, int nms_radius, int border, int max_keypoints, float* out_xy,
                                               float* out_score, float* out_desc, int* out_n_pinned, void* stream) {
  if (!ctx || !image || !out_xy || !out_score || !out_desc || !out_n_pinned || max_keypoints <= 0) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = sp_extract_enqueue(ctx, image, H, W, channels, pitch, thr, nms_radius, border, max_keypoints, out_xy, out_score, out_desc, st);
  if (rc) return rc;
  B2_CUDA(ctx, cudaMemcpyAsync(out_n_pinned, ctx->sp->sel_cnt.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  return B2_OK;
}

// Synchronise `stream` and report a tensor-core pipeline fault of any extract enqueued before (the async variant cannot).
extern "C" int b2_superpoint_finish_dev(b2_context* ctx, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  SuperPointState* s = ctx->sp;
  if (!s || !s->loaded) return b2_fail(ctx, B2_ERR_STATE, "superpoint weights not set");
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&err, s->errflag.p, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  B2_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma conv pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}
