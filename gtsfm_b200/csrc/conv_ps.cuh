// 3x3 convolution (pad 1) + bias + ReLU (+ fused 2x2/2 max-pool): persistent, warp-specialised wgmma implicit GEMM with
// HALO REUSE, split-fp16 (~fp32).
//
// The SuperPoint encoder / head convolutions (thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:119-134,148-162)
// are GEMMs with M = pixels, N = output channels, K = 9 taps x Cin.  Activations live in HBM as NHWC fp16 hi / lo planes
// (x ~= hi + lo * 2^-11).
//
//   * Output tile = 16 rows x 8 columns of pixels (M = 128, m = h * 8 + w) by 64 output channels.  ONE 3-D TMA box
//     {64 ch, 10 px, 18 rows} per plane and 64-channel chunk brings the tile with its halo; out-of-image coordinates are
//     zero-filled by the TMA unit = the convolution's zero padding.  Pixels are 128-byte rows (128-byte swizzle).
//   * The 9 taps are 9 wgmma descriptors into the SAME buffer: start address + ((dy + 1) * 10 + (dx + 1)) * 128 bytes, 8-row
//     group stride 10 * 128 bytes (a group = 8 consecutive pixels of one tile row).  The start is not 1024-byte aligned and
//     the stride not a multiple of 1024: that works because the tensor core applies the 128-byte swizzle to ABSOLUTE
//     shared-memory address bits, exactly like the TMA unit that wrote the tile (descriptor base_offset = 0).
//   * Weights of the CTA's 64 output channels and the current 64-channel chunk stay resident in shared memory (9 taps x
//     [Bh (64 rows); Bl (64 rows)] x 64 K = 144 KB): loaded once per CTA when Cin = 64, once per (tile, chunk) when
//     Cin = 128 (the register accumulators hold one tile).  Stacking Bh over Bl makes  Ah x [Bh; Bl]^T  ONE N = 128 MMA
//     (columns 0-63: Ah Bh, 64-127: Ah Bl); Al x Bh^T (N = 64) goes to a third accumulator.
//   * Warp 8 = TMA producer (3 plane buffers); warpgroup w (warps 4w .. 4w + 3) owns pixels 64w .. 64w + 63: MMAs, then
//     hh + (hl + lh) * 2^-11, 2x2 max-pool (partners: row + 8 in the fragment, lane ^ 4), bias, ReLU, planes and / or fp32.
//
// DILATION (k_conv_ps<2>: D2-Net's conv4_x, 3x3 with dilation 2 and padding 2).  The template parameter D is the dilation
// and the padding.  The halo box becomes {64, 8 + 2D, 16 + 2D}, the tap offsets are D pixels apart and the 8-row group stride
// is (8 + 2D) x 128 bytes.  At D = 2 a box is 30 KiB: the 144 KiB weight block plus three of them would be 241 152 bytes, over
// the 232 448-byte per-block limit, so the dilated instance keeps TWO activation buffers (210 432 bytes).  The producer then
// runs at most one plane ahead of the consumers.  Measured effect (profiles/h100_d2net.json, H100 80GB HBM3 at a 400 W power
// limit): one 512 -> 512 layer at 282 x 189 takes 1.659 ms on k_conv_ps<2> (two buffers, 20 x 12 halo) against 1.653 ms on
// k_conv_ps<1> (three buffers, 18 x 10 halo), 151.6 vs 152.1 TFLOP/s: with Cin >= 256 every 64-channel chunk reloads its
// 144 KiB of weights, and that wait, not the third activation buffer, sets the pace.  The alternative, a smaller tile, would
// re-read more halo per output pixel.  D = 1 is the shipped SuperPoint / NetVLAD instance: every expression reduces to the
// former constants and it compiles to the same SASS.
#pragma once
#include "common.cuh"
#include "tma.cuh"

constexpr int CP_TH = 16, CP_TW = 8;  // output tile (pixels)
constexpr int CP_B_TAP = 128 * 128;   // [Bh; Bl] x 64 K halves
constexpr int CP_B_BYTES = 9 * CP_B_TAP;
constexpr int CP_THREADS = 256 + 32;

template <int D>  // dilation = padding
struct CpGeom {
  static constexpr int HH = CP_TH + 2 * D, HW = CP_TW + 2 * D;  // halo tile
  static constexpr int A_LOAD = HH * HW * 128;                  // bytes per plane box (D = 1: 23040)
  static constexpr int A_BYTES = (A_LOAD + 1023) / 1024 * 1024;  // buffer pitch (1024-aligned)
  static constexpr int NA = D == 1 ? 3 : 2;                     // activation plane buffers
  static constexpr size_t SMEM = (size_t)CP_B_BYTES + NA * A_BYTES + 1024 + 512;
};
constexpr int CP_HH = CpGeom<1>::HH, CP_HW = CpGeom<1>::HW;
constexpr int CP_A_LOAD = CpGeom<1>::A_LOAD, CP_A_BYTES = CpGeom<1>::A_BYTES, CP_NA = CpGeom<1>::NA;
constexpr size_t CP_SMEM = CpGeom<1>::SMEM;
static_assert(CP_A_BYTES == 23 * 1024 && CpGeom<2>::SMEM <= 232448, "conv_ps shared-memory plan");

struct ConvPsMaps {
  CUtensorMap ah, al;  // activations: 3-D {C, W, H}, box {64, 8 + 2D, 16 + 2D}
  CUtensorMap wh, wl;  // weights: 2-D {9 * Cin, Cout}, box {64, 64}
};
struct ConvPsArgs {
  int H, W, Cin, Cout;
  int pool;           // 1: 2x2/2 max-pool fused; output is (H/2, W/2)
  int relu;           // 1: max(., 0) after the bias (every SuperPoint / VGG layer but NetVLAD's last convolution)
  const float* bias;  // [Cout]
  __half *Oh, *Ol;    // optional output planes NHWC
  float* Of;          // optional fp32 output NHWC
  int* err_flag;
};

namespace tc {
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
}  // namespace tc

template <int D = 1>
static __global__ void __launch_bounds__(CP_THREADS, 1) k_conv_ps(const __grid_constant__ ConvPsMaps maps, ConvPsArgs g) {
  using Geo = CpGeom<D>;
  constexpr int HW = Geo::HW, A_BYTES = Geo::A_BYTES, NA = Geo::NA;
  extern __shared__ unsigned char cp_raw[];
  const uint32_t raw = tc::smem_u32(cp_raw);
  const uint32_t smem0 = (raw + 1023u) & ~1023u;
  unsigned char* sm = cp_raw + (smem0 - raw);
  const uint32_t sB = smem0, sA = smem0 + CP_B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + CP_B_BYTES + NA * A_BYTES);
  uint64_t* fullA = bars;               // [NA]
  uint64_t* emptyA = fullA + NA;        // [NA] one arrival per consumer warp
  uint64_t* fullB = emptyA + NA;        // [9]
  uint64_t* emptyB = fullB + 9;         // [9] one arrival per consumer warp

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int nblk = g.Cout / 64, nchunk = g.Cin / 64;
  const int tiles_x = (g.W + CP_TW - 1) / CP_TW, tiles_y = (g.H + CP_TH - 1) / CP_TH, ntiles = tiles_x * tiles_y;
  const int nb = blockIdx.x % nblk, lane_id = blockIdx.x / nblk, stride = gridDim.x / nblk;
  const int nt = lane_id < ntiles ? (ntiles - lane_id + stride - 1) / stride : 0;  // this CTA's tiles: lane_id + k * stride

  if (t == 0) {
    for (int i = 0; i < NA; ++i) tc::mbar_init(&fullA[i], 1), tc::mbar_init(&emptyA[i], 8);
    for (int i = 0; i < 9; ++i) tc::mbar_init(&fullB[i], 1), tc::mbar_init(&emptyB[i], 8);
    tc::fence_mbar_init();
    tc::tma_prefetch_desc(&maps.ah);
    tc::tma_prefetch_desc(&maps.al);
    tc::tma_prefetch_desc(&maps.wh);
    tc::tma_prefetch_desc(&maps.wl);
  }
  __syncthreads();
  bool ok = true;

  if (warp == 8) {
    if (lane == 0) {
      uint32_t a_cnt = 0, bver = 0;
      for (int k = 0; k < nt; ++k) {
        const int tile = lane_id + k * stride;
        const int x0 = (tile % tiles_x) * CP_TW, y0 = (tile / tiles_x) * CP_TH;
        for (int c = 0; c < nchunk; ++c) {
          if (nchunk > 1 || bver == 0) {  // (re)load the weights of (nb, c): tap slot by tap slot, as the consumers free them
            for (int tap = 0; tap < 9; ++tap) {
              if (bver > 0) ok = tc::mbar_wait(&emptyB[tap], (bver - 1) & 1) && ok;
              tc::mbar_expect_tx(&fullB[tap], CP_B_TAP);
              tc::tma_load_2d(sB + tap * CP_B_TAP, &maps.wh, &fullB[tap], (tap * nchunk + c) * 64, nb * 64);
              tc::tma_load_2d(sB + tap * CP_B_TAP + CP_B_TAP / 2, &maps.wl, &fullB[tap], (tap * nchunk + c) * 64, nb * 64);
            }
            ++bver;
          }
          for (int plane = 0; plane < 2; ++plane, ++a_cnt) {
            const uint32_t buf = a_cnt % NA, use = a_cnt / NA;
            if (use > 0) ok = tc::mbar_wait(&emptyA[buf], (use - 1) & 1) && ok;
            tc::mbar_expect_tx(&fullA[buf], Geo::A_LOAD);
            tc::tma_load_3d(sA + buf * A_BYTES, plane ? &maps.al : &maps.ah, &fullA[buf], c * 64, x0 - D, y0 - D);
          }
        }
      }
    }
  } else {
    // ---- consumer warpgroup wg: tile rows h = 8 wg .. 8 wg + 7; thread rows (h0, wc) and (h0 + 1, wc) ------------------
    const int wg = warp >> 2;
    const int h0 = wg * 8 + (warp & 3) * 2, wc = lane >> 2, c2 = (lane & 3) * 2;
    const int OH = g.pool ? g.H >> 1 : g.H, OW = g.pool ? g.W >> 1 : g.W;
    uint32_t a_cnt = 0, bver = 0;
    for (int k = 0; k < nt; ++k) {
      const int tile = lane_id + k * stride;
      const int x0 = (tile % tiles_x) * CP_TW, y0 = (tile / tiles_x) * CP_TH;
      float acc[64], accl[32];  // acc columns 0-63: Ah Bh, 64-127: Ah Bl; accl: Al Bh
      for (int c = 0; c < nchunk; ++c) {
        const bool new_b = nchunk > 1 || bver == 0;
        if (new_b) ++bver;
        {  // hi plane: Ah x [Bh; Bl]^T
          const uint32_t buf = a_cnt % NA;
          ok = tc::mbar_wait(&fullA[buf], (a_cnt / NA) & 1) && ok;
          const uint32_t base = sA + buf * A_BYTES;
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap) {
            if (new_b) ok = tc::mbar_wait(&fullB[tap], (bver - 1) & 1) && ok;
            const uint64_t dA = tc::wg_desc_sw128(base + ((D * (tap / 3) + wg * 8) * HW + D * (tap % 3)) * 128, HW * 128);
            const uint64_t dB = tc::wg_desc_sw128(sB + tap * CP_B_TAP);
            tc::wg_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)
              tc::wg_ss_n128(acc, dA + (uint64_t)(ks * 2), dB + (uint64_t)(ks * 2), (c == 0 && tap == 0 && ks == 0) ? 0u : 1u);
            tc::wg_commit();
          }
          tc::wg_wait<0>();
          if (lane == 0) tc::mbar_arrive(&emptyA[buf]);
          ++a_cnt;
        }
        {  // lo plane: Al x Bh^T into accl
          const uint32_t buf = a_cnt % NA;
          ok = tc::mbar_wait(&fullA[buf], (a_cnt / NA) & 1) && ok;
          const uint32_t base = sA + buf * A_BYTES;
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap) {
            const uint64_t dA = tc::wg_desc_sw128(base + ((D * (tap / 3) + wg * 8) * HW + D * (tap % 3)) * 128, HW * 128);
            const uint64_t dB = tc::wg_desc_sw128(sB + tap * CP_B_TAP);
            tc::wg_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) tc::wg_ss_n64(accl, dA + (uint64_t)(ks * 2), dB + (uint64_t)(ks * 2), (c == 0 && tap == 0 && ks == 0) ? 0u : 1u);
            tc::wg_commit();
            if (nchunk > 1 && tap > 0) {  // the previous tap's weights are no longer read: hand the slot back
              tc::wg_wait<1>();
              if (lane == 0) tc::mbar_arrive(&emptyB[tap - 1]);
            }
          }
          tc::wg_wait<0>();
          if (lane == 0) {
            if (nchunk > 1) tc::mbar_arrive(&emptyB[8]);
            tc::mbar_arrive(&emptyA[buf]);
          }
          ++a_cnt;
        }
      }
      // ---- epilogue: v[4j + 2i + e] = pixel (h0 + i, wc), channel 8j + c2 + e ----
      float v[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = fmaf(acc[32 + i] + accl[i], tc::LO_INV, acc[i]);
      const float* bp = g.bias + nb * 64 + c2;
      if (g.pool) {  // max over the 2x2 window; max commutes with bias (+ ReLU)
        const int oy = (y0 + h0) >> 1, ox = (x0 + wc) >> 1;
        const bool writer = (wc & 1) == 0 && oy < OH && ox < OW;
        float p[16];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float m = fmaxf(v[4 * j + e], v[4 * j + 2 + e]);
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
            p[2 * j + e] = m;
          }
        if (writer) {
          const size_t opix = ((size_t)oy * OW + ox) * g.Cout + nb * 64 + c2;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 b = make_float2(__ldg(bp + 8 * j), __ldg(bp + 8 * j + 1));
            float a0 = p[2 * j] + b.x, a1 = p[2 * j + 1] + b.y;
            if (g.relu) a0 = fmaxf(a0, 0.f), a1 = fmaxf(a1, 0.f);
            if (g.Of) *reinterpret_cast<float2*>(g.Of + opix + 8 * j) = make_float2(a0, a1);
            if (g.Oh) {
              uint32_t hi, lo;
              tc::split2(a0, a1, hi, lo);
              *reinterpret_cast<uint32_t*>(g.Oh + opix + 8 * j) = hi;
              *reinterpret_cast<uint32_t*>(g.Ol + opix + 8 * j) = lo;
            }
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int oy = y0 + h0 + i, ox = x0 + wc;
          if (oy >= OH || ox >= OW) continue;
          const size_t opix = ((size_t)oy * OW + ox) * g.Cout + nb * 64 + c2;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 b = make_float2(__ldg(bp + 8 * j), __ldg(bp + 8 * j + 1));
            float a0 = v[4 * j + 2 * i] + b.x, a1 = v[4 * j + 2 * i + 1] + b.y;
            if (g.relu) a0 = fmaxf(a0, 0.f), a1 = fmaxf(a1, 0.f);
            if (g.Of) *reinterpret_cast<float2*>(g.Of + opix + 8 * j) = make_float2(a0, a1);
            if (g.Oh) {
              uint32_t hi, lo;
              tc::split2(a0, a1, hi, lo);
              *reinterpret_cast<uint32_t*>(g.Oh + opix + 8 * j) = hi;
              *reinterpret_cast<uint32_t*>(g.Ol + opix + 8 * j) = lo;
            }
          }
        }
      }
    }
  }
  if (!ok && g.err_flag) *g.err_flag = 1;
  __syncthreads();
}

// NHWC fp16 activation plane [H][W][C] -> 3-D map {C, W, H}, box {64, 8 + 2 dil, 16 + 2 dil}, 128-byte swizzle, zero OOB fill
static inline bool tma_map_nhwc_halo(CUtensorMap* out, const __half* base, int H, int W, int C, int dil = 1) {
  PFN_encodeTiled enc = tma_encoder();
  if (!enc || !base) return false;
  cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H};
  cuuint64_t strides[2] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)(CP_TW + 2 * dil), (cuuint32_t)(CP_TH + 2 * dil)};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<__half*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// ---- host helpers shared by the networks on this kernel (SuperPoint, NetVLAD, D2-Net) --------------------------------------

// Walks n layers of (OIHW 3x3 weight, bias) from `blob`: layer 0 (3 input channels, run by a SIMT kernel) -> w0 fp32
// [tap][ci][co]; layers >= 1 -> `stage` at woff[l] as [co][tap * Cin + ci] (the implicit GEMM's K order); biases concatenated
// at boff[l].  Returns the number of floats read.
static size_t conv_ps_repack(const float* blob, int n, const int* CI, const int* CO, std::vector<float>& stage, std::vector<float>& bias,
                             std::vector<float>& w0, size_t* woff, size_t* boff) {
  size_t wtot = 0, btot = 0;
  for (int l = 0; l < n; ++l) {
    woff[l] = wtot, boff[l] = btot;
    if (l) wtot += (size_t)CO[l] * 9 * CI[l];
    btot += CO[l];
  }
  stage.assign(wtot, 0.f), bias.assign(btot, 0.f), w0.assign((size_t)27 * CO[0], 0.f);
  size_t src = 0;
  for (int l = 0; l < n; ++l) {
    const int co = CO[l], ci = CI[l];
    const float* w = blob + src;
    if (l == 0) {
      for (int o = 0; o < co; ++o)
        for (int i = 0; i < ci; ++i)
          for (int tp = 0; tp < 9; ++tp) w0[((size_t)tp * 3 + i) * co + o] = w[((size_t)o * ci + i) * 9 + tp];
    } else {
      float* d = stage.data() + woff[l];
      for (int o = 0; o < co; ++o)
        for (int tp = 0; tp < 9; ++tp)
          for (int i = 0; i < ci; ++i) d[(size_t)o * 9 * ci + (size_t)tp * ci + i] = w[((size_t)o * ci + i) * 9 + tp];
    }
    src += (size_t)co * ci * 9;
    std::copy(blob + src, blob + src + co, bias.begin() + boff[l]);
    src += co;
  }
  return src;
}

// host fp32 [n] -> device split planes h / l (k_split_f32), staged through `tmp` in pieces of `piece` floats; synchronous
static cudaError_t conv_ps_upload_planes(const float* host, size_t n, DevBuf& h, DevBuf& l, DevBuf& tmp, size_t piece) {
  cudaError_t e;
  if ((e = h.ensure(n * sizeof(__half))) != cudaSuccess || (e = l.ensure(n * sizeof(__half))) != cudaSuccess) return e;
  for (size_t o = 0; o < n; o += piece) {
    const size_t m = n - o < piece ? n - o : piece;
    if ((e = cudaMemcpy(tmp.p, host + o, m * sizeof(float), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
    k_split_f32<<<(unsigned)((m + 255) / 256), 256>>>(tmp.as<float>(), m, h.as<__half>() + o, l.as<__half>() + o);
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// k_conv_ps's grid: one CTA per (tile, 64-channel block) up to the SM count, rounded down to a multiple of the blocks (a CTA
// keeps one block of the weights resident: CTA c serves block c % (Cout / 64))
static inline int conv_ps_grid(int sm_count, int H, int W, int Cout) {
  const int nblk = Cout / 64, units = cdiv(W, CP_TW) * cdiv(H, CP_TH) * nblk;
  const int grid = sm_count < units ? sm_count : units;
  return grid - grid % nblk;
}

// One layer's tensor maps, kept by a caller that runs the same layer on the same buffers call after call (SuperPoint: four
// host-side encodes per layer and image otherwise).  The key is everything the maps depend on.
struct ConvPsMapCache {
  ConvPsMaps maps;
  const __half *ih = nullptr, *wh = nullptr, *wl = nullptr;
  int H = 0, W = 0, Cin = 0, Cout = 0, dil = 0;
};

// One layer on k_conv_ps<dil> (dil = padding, 1 or 2): input planes `ih` [H][W][Cin] with the lo plane right after the hi one,
// weight planes wh / wl [Cout][9 Cin] -> output planes `oh` (lo after hi) and / or fp32 `of`, NHWC.  ctas = 0 launches
// conv_ps_grid's grid, otherwise exactly `ctas` CTAs (a multiple of Cout / 64).  `cache` = NULL encodes the maps on every
// call, otherwise only when its key differs.  The caller has set the kernel's dynamic shared-memory attribute (CP_SMEM /
// CpGeom<2>::SMEM).
static int conv_ps_run(b2_context* ctx, cudaStream_t st, const __half* ih, int H, int W, int Cin, int Cout, int pool, int relu, int dil,
                       const __half* wh, const __half* wl, const float* bias, __half* oh, float* of, int* err_flag, const char* model,
                       int ctas = 0, ConvPsMapCache* cache = nullptr) {
  if (dil != 1 && dil != 2) return b2_fail(ctx, B2_ERR_ARG, "conv_ps: dilation must be 1 or 2");
  // the kernel walks Cin / 64 whole chunks and Cout / 64 channel blocks: a remainder would be dropped
  if (Cin <= 0 || Cout <= 0 || Cin % 64 || Cout % 64 || H <= 0 || W <= 0)
    return b2_fail(ctx, B2_ERR_ARG, "conv_ps: Cin and Cout must be positive multiples of 64, H and W positive");
  if (ctas < 0 || ctas % (Cout / 64)) return b2_fail(ctx, B2_ERR_ARG, "conv_ps: the grid must be a multiple of Cout / 64");
  const int OH = pool ? H / 2 : H, OW = pool ? W / 2 : W;
  ConvPsMapCache local;
  ConvPsMapCache& mc = cache ? *cache : local;
  if (mc.ih != ih || mc.wh != wh || mc.wl != wl || mc.H != H || mc.W != W || mc.Cin != Cin || mc.Cout != Cout || mc.dil != dil) {
    mc = ConvPsMapCache{};  // a failed encode leaves no key behind
    const __half* il = ih + (size_t)H * W * Cin;
    bool ok = tma_map_nhwc_halo(&mc.maps.ah, ih, H, W, Cin, dil) && tma_map_nhwc_halo(&mc.maps.al, il, H, W, Cin, dil) &&
              tma_map_2d(&mc.maps.wh, wh, Cout, 9 * Cin, 9 * Cin, 64) && tma_map_2d(&mc.maps.wl, wl, Cout, 9 * Cin, 9 * Cin, 64);
    if (!ok) return b2_fail(ctx, B2_ERR_CUDA, std::string("cuTensorMapEncodeTiled failed (") + model + " conv)");
    mc.ih = ih, mc.wh = wh, mc.wl = wl, mc.H = H, mc.W = W, mc.Cin = Cin, mc.Cout = Cout, mc.dil = dil;
  }
  const ConvPsMaps& maps = mc.maps;
  ConvPsArgs a{};
  a.H = H, a.W = W, a.Cin = Cin, a.Cout = Cout, a.pool = pool, a.relu = relu, a.bias = bias;
  if (oh) a.Oh = oh, a.Ol = oh + (size_t)OH * OW * Cout;
  a.Of = of, a.err_flag = err_flag;
  const int grid = ctas ? ctas : conv_ps_grid(ctx->sm_count, H, W, Cout);
  b2_prof_work(ctx, dil == 1 ? "k_conv_ps<1>" : "k_conv_ps<2>", 2.0 * 9.0 * H * W * Cin * Cout);
  if (dil == 1) B2_LAUNCH(ctx, k_conv_ps<1>, grid, CP_THREADS, CP_SMEM, st, maps, a);
  else B2_LAUNCH(ctx, k_conv_ps<2>, grid, CP_THREADS, CpGeom<2>::SMEM, st, maps, a);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}

// ---- the exact-fp32 SIMT path (SuperPoint under force_simt) ------------------------------------------------------------------

// Generic 3x3 conv, pad 1, bias + ReLU, optional fused 2x2/2 max-pool, NHWC fp32, SIMT fp32 FMA (exact-fp32 path).
// Block tile: 8 rows x 16 cols of pixels x 64 output channels; thread micro-tile 2x4 pixels x 4 channels.
constexpr int CT_H = 8, CT_W = 16, CK = 8, CKP = 12;  // CKP: padded per-pixel stride in smem (floats)
template <int POOL>
static __global__ void __launch_bounds__(256) k_conv3x3(const float* __restrict__ in, const float* __restrict__ wt,
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

// One layer on k_conv3x3<pool>: fp32 NHWC `in` [H][W][Cin] (Cin a multiple of CK), weights [tap][Cin][Cout] (Cout a multiple of
// 64), bias, ReLU -> fp32 NHWC `out`
static int conv3x3_simt_run(b2_context* ctx, cudaStream_t st, const float* in, const float* wt, const float* bias, float* out, int H, int W,
                            int Cin, int Cout, bool pool) {
  const dim3 grid(cdiv(W, CT_W), cdiv(H, CT_H), Cout / 64);
  b2_prof_work(ctx, "k_conv3x3", 2.0 * 9.0 * H * W * Cin * Cout);
  if (pool)
    B2_LAUNCH(ctx, k_conv3x3<1>, grid, 256, 0, st, in, wt, bias, out, H, W, Cin, Cout);
  else
    B2_LAUNCH(ctx, k_conv3x3<0>, grid, 256, 0, st, in, wt, bias, out, H, W, Cin, Cout);
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}
