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
#pragma once
#include "common.cuh"
#include "tma.cuh"

constexpr int CP_TH = 16, CP_TW = 8;                 // output tile (pixels)
constexpr int CP_HH = CP_TH + 2, CP_HW = CP_TW + 2;  // halo tile
constexpr int CP_A_LOAD = CP_HH * CP_HW * 128;       // 23040 bytes per plane box
constexpr int CP_A_BYTES = 23 * 1024;                // buffer pitch (1024-aligned)
constexpr int CP_NA = 3;                             // activation plane buffers
constexpr int CP_B_TAP = 128 * 128;                  // [Bh; Bl] x 64 K halves
constexpr int CP_B_BYTES = 9 * CP_B_TAP;
constexpr int CP_THREADS = 256 + 32;
constexpr size_t CP_SMEM = (size_t)CP_B_BYTES + CP_NA * CP_A_BYTES + 1024 + 512;

struct ConvPsMaps {
  CUtensorMap ah, al;  // activations: 3-D {C, W, H}, box {64, 10, 18}
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
  float* dbg;  // optional [gridDim.x][8] timestamps (globaltimer ns & 0xFFFFFF), profiling runs only
};

namespace tc {
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
}  // namespace tc

__device__ __forceinline__ void cp_stamp(float* dbg, int slot) {
  if (!dbg) return;
  unsigned long long tns;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(tns));
  dbg[blockIdx.x * 8 + slot] = (float)(tns & 0xFFFFFFull);
}

static __global__ void __launch_bounds__(CP_THREADS, 1) k_conv_ps(const __grid_constant__ ConvPsMaps maps, ConvPsArgs g) {
  extern __shared__ unsigned char cp_raw[];
  const uint32_t raw = tc::smem_u32(cp_raw);
  const uint32_t smem0 = (raw + 1023u) & ~1023u;
  unsigned char* sm = cp_raw + (smem0 - raw);
  const uint32_t sB = smem0, sA = smem0 + CP_B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + CP_B_BYTES + CP_NA * CP_A_BYTES);
  uint64_t* fullA = bars;               // [CP_NA]
  uint64_t* emptyA = fullA + CP_NA;     // [CP_NA] one arrival per consumer warp
  uint64_t* fullB = emptyA + CP_NA;     // [9]
  uint64_t* emptyB = fullB + 9;         // [9] one arrival per consumer warp

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int nblk = g.Cout / 64, nchunk = g.Cin / 64;
  const int tiles_x = (g.W + CP_TW - 1) / CP_TW, tiles_y = (g.H + CP_TH - 1) / CP_TH, ntiles = tiles_x * tiles_y;
  const int nb = blockIdx.x % nblk, lane_id = blockIdx.x / nblk, stride = gridDim.x / nblk;
  const int nt = lane_id < ntiles ? (ntiles - lane_id + stride - 1) / stride : 0;  // this CTA's tiles: lane_id + k * stride

  if (t == 0) {
    cp_stamp(g.dbg, 0);
    for (int i = 0; i < CP_NA; ++i) tc::mbar_init(&fullA[i], 1), tc::mbar_init(&emptyA[i], 8);
    for (int i = 0; i < 9; ++i) tc::mbar_init(&fullB[i], 1), tc::mbar_init(&emptyB[i], 8);
    tc::fence_mbar_init();
    tc::tma_prefetch_desc(&maps.ah);
    tc::tma_prefetch_desc(&maps.al);
    tc::tma_prefetch_desc(&maps.wh);
    tc::tma_prefetch_desc(&maps.wl);
  }
  __syncthreads();
  bool ok = true;
  if (t == 0) cp_stamp(g.dbg, 1), g.dbg ? (void)(g.dbg[blockIdx.x * 8 + 7] = (float)nt) : (void)0;

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
            const uint32_t buf = a_cnt % CP_NA, use = a_cnt / CP_NA;
            if (use > 0) ok = tc::mbar_wait(&emptyA[buf], (use - 1) & 1) && ok;
            tc::mbar_expect_tx(&fullA[buf], CP_A_LOAD);
            tc::tma_load_3d(sA + buf * CP_A_BYTES, plane ? &maps.al : &maps.ah, &fullA[buf], c * 64, x0 - 1, y0 - 1);
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
          const uint32_t buf = a_cnt % CP_NA;
          ok = tc::mbar_wait(&fullA[buf], (a_cnt / CP_NA) & 1) && ok;
          const uint32_t base = sA + buf * CP_A_BYTES;
          if (a_cnt == 0 && t == 0) cp_stamp(g.dbg, 2);
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap) {
            if (new_b) ok = tc::mbar_wait(&fullB[tap], (bver - 1) & 1) && ok;
            const uint64_t dA = tc::wg_desc_sw128(base + ((tap / 3 + wg * 8) * CP_HW + tap % 3) * 128, CP_HW * 128);
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
          const uint32_t buf = a_cnt % CP_NA;
          ok = tc::mbar_wait(&fullA[buf], (a_cnt / CP_NA) & 1) && ok;
          const uint32_t base = sA + buf * CP_A_BYTES;
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap) {
            const uint64_t dA = tc::wg_desc_sw128(base + ((tap / 3 + wg * 8) * CP_HW + tap % 3) * 128, CP_HW * 128);
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
      if (k == 0 && t == 0) cp_stamp(g.dbg, 3);
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
      if (k == nt - 1 && t == 0) cp_stamp(g.dbg, 5);
    }
  }
  if (!ok && g.err_flag) *g.err_flag = 1;
  __syncthreads();
  if (t == 0) cp_stamp(g.dbg, 6);
}

// NHWC fp16 activation plane [H][W][C] -> 3-D map {C, W, H}, box {64, CP_HW, CP_HH}, 128-byte swizzle, zero OOB fill
static inline bool tma_map_nhwc_halo(CUtensorMap* out, const __half* base, int H, int W, int C) {
  PFN_encodeTiled enc = tma_encoder();
  if (!enc || !base) return false;
  cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H};
  cuuint64_t strides[2] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2};
  cuuint32_t box[3] = {64, CP_HW, CP_HH};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<__half*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
