// Persistent, warp-specialised wgmma + TMA split-fp16 "NT" GEMM over a BATCH of problems that share one weight matrix:
//     C_z[M_z, N] = [A1_z | A2_z][M_z, K] * B[N, K]^T        z = 0 .. nprob-1  (images of a batch of pairs)
// or, with `b_per_problem`, one (A_z, B_z, N_z) triple per problem (the assignment similarity of every pair of a batch).
//
// Arithmetic: every fp32 value travels as two fp16 planes, x ~= hi + lo * 2^-11 (the producing kernel's epilogue writes
// them); three MMAs per K step,  acc0 += Ah Bh ; acc1 += Ah Bl + Al Bh ; result = acc0 + acc1 * 2^-11, both fp32
// accumulators in registers.  The dropped Al * Bl term is 2^-22 relative.
//
// Schedule: one CTA per SM walks output tiles `blockIdx.x + i * gridDim.x` of the whole batch (problem-major, then row
// tile, then column tile - concurrently running CTAs share the A row tile through L2):
//   warp 8 (lane 0)  TMA producer: a 3-stage ring (3 x 64 KB) that keeps loading the next tile during the epilogue
//   warps 0-7        warpgroup w: rows 64w .. 64w + 63 of the 128 x 128 tile, wgmma m64n128k16 into two register
//                    accumulators, then bias / scale / ReLU / residual / split-plane stores from the fragment.
#pragma once
#include "tma.cuh"

constexpr int GW_MAXP = 16;  // problems per launch (2 images x 8 pairs)
constexpr int GW_M = 128, GW_N = 128, GW_K = 64;
constexpr int GW_A_BYTES = GW_M * GW_K * 2;  // 16 KB per plane
constexpr int GW_B_BYTES = GW_N * GW_K * 2;  // 16 KB per plane
constexpr int GW_STAGE_BYTES = 2 * GW_A_BYTES + 2 * GW_B_BYTES;  // 64 KB
constexpr int GW_STAGES = 3;
constexpr int GW_THREADS = 256 + 32;  // two consumer warpgroups + the TMA producer warp
constexpr size_t GW_SMEM = GW_STAGES * GW_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;

struct GemmProblem {
  const float* resid;  // [M][ldr] fp32 or null, added after bias / scale
  float* C;            // optional fp32 output, row-major [M][ldc]
  __half *Ch, *Cl;     // optional split output planes
  int M, N, ldc;
  int vec4;      // outputs / residual may be accessed in pairs (8-byte fp32, 4-byte plane accesses; host checks 16-byte alignment)
  int tiles_n;   // ceil(N / 128)
  int tile_end;  // running total of tiles up to and including this problem
};
struct GemmWsMaps {  // 128-byte TMA descriptors, passed as a __grid_constant__ kernel parameter
  CUtensorMap a1h[GW_MAXP], a1l[GW_MAXP];  // per problem: first K segment
  CUtensorMap a2h[GW_MAXP], a2l[GW_MAXP];  // optional second K segment (torch.cat([x, msg], -1) without the concat)
  CUtensorMap bh[GW_MAXP], bl[GW_MAXP];    // [0] when every problem shares the weight matrix
};
struct GemmWsArgs {
  GemmProblem p[GW_MAXP];
  int nprob, tiles;
  int K1, K2;
  int b_per_problem;
  const float* bias;  // [N] or null
  int ldr;
  float scale;
  int ldch;        // row-major leading dimension of Ch / Cl (ignored when head_major)
  int head_major;  // 1: Ch / Cl (and C) are written as [N/64][M][64] (attention head layout)
  int relu;        // max(., 0) after bias / scale, before the residual
  int lo_unscaled; // split outputs keep lo = fp16(x - hi) (attention operands)
  int* err_flag;   // set to 1 if an mbarrier wait timed out (pipeline bug): results are then invalid
};

static __global__ void __launch_bounds__(GW_THREADS, 1) k_gemm_ws(const __grid_constant__ GemmWsMaps maps, const __grid_constant__ GemmWsArgs g) {
  extern __shared__ unsigned char gw_raw[];
  const uint32_t raw = tc::smem_u32(gw_raw);
  const uint32_t smem0 = (raw + 1023u) & ~1023u;
  unsigned char* sm = gw_raw + (smem0 - raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + GW_STAGES * GW_STAGE_BYTES);
  uint64_t* empty = full + GW_STAGES;  // one arrival per consumer warp

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int nk = (g.K1 + g.K2) / GW_K;

  if (t == 0) {
    for (int s = 0; s < GW_STAGES; ++s) tc::mbar_init(&full[s], 1), tc::mbar_init(&empty[s], 8);
    tc::fence_mbar_init();
    tc::tma_prefetch_desc(&maps.bh[0]);
    tc::tma_prefetch_desc(&maps.bl[0]);
  }
  __syncthreads();
  bool ok = true;

  auto decode = [&](int tile, int& z, int& m0, int& n0) {
    z = 0;
    while (z + 1 < g.nprob && tile >= g.p[z].tile_end) ++z;
    const int local = tile - (z ? g.p[z - 1].tile_end : 0);
    const int mt = local / g.p[z].tiles_n;
    n0 = (local - mt * g.p[z].tiles_n) * GW_N;
    m0 = mt * GW_M;
  };

  if (warp == 8) {
    if (lane == 0) {
      // ===== TMA producer =====
      int gk = 0;
      for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
        int z, m0, n0;
        decode(tile, z, m0, n0);
        const int zb = g.b_per_problem ? z : 0;
        for (int kc = 0; kc < nk; ++kc, ++gk) {
          const int s = gk % GW_STAGES;
          if (gk >= GW_STAGES) ok = tc::mbar_wait(&empty[s], ((gk / GW_STAGES) - 1) & 1) && ok;
          const int k0 = kc * GW_K;
          const bool seg2 = k0 >= g.K1;
          const CUtensorMap* ah = seg2 ? &maps.a2h[z] : &maps.a1h[z];
          const CUtensorMap* al = seg2 ? &maps.a2l[z] : &maps.a1l[z];
          const int ka = seg2 ? k0 - g.K1 : k0;
          const uint32_t sA = smem0 + s * GW_STAGE_BYTES, sB = sA + 2 * GW_A_BYTES;
          tc::mbar_expect_tx(&full[s], GW_STAGE_BYTES);
          tc::tma_load_2d(sA, ah, &full[s], ka, m0);
          tc::tma_load_2d(sA + GW_A_BYTES, al, &full[s], ka, m0);
          tc::tma_load_2d(sB, &maps.bh[zb], &full[s], k0, n0);
          tc::tma_load_2d(sB + GW_B_BYTES, &maps.bl[zb], &full[s], k0, n0);
        }
      }
    }
  } else {
    // ===== consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of every tile =====
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment rows r0, r0 + 8
    const int c2 = (lane & 3) * 2;                           // fragment columns 8j + c2, + 1
    const float scale = g.scale;
    const int relu = g.relu;
    int gk = 0;
    for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
      int z, m0, n0;
      decode(tile, z, m0, n0);
      float acc0[64], acc1[64];
      for (int kc = 0; kc < nk; ++kc, ++gk) {
        const int s = gk % GW_STAGES;
        ok = tc::mbar_wait(&full[s], (gk / GW_STAGES) & 1) && ok;
        const uint32_t aH = smem0 + s * GW_STAGE_BYTES + wg * (64 * 128), aL = aH + GW_A_BYTES;
        const uint32_t bH = smem0 + s * GW_STAGE_BYTES + 2 * GW_A_BYTES, bL = bH + GW_B_BYTES;
        const uint64_t dAh = tc::wg_desc_sw128(aH), dAl = tc::wg_desc_sw128(aL), dBh = tc::wg_desc_sw128(bH), dBl = tc::wg_desc_sw128(bL);
        tc::wg_fence();
#pragma unroll
        for (int ks = 0; ks < GW_K / 16; ++ks) {
          const uint64_t adv = (uint64_t)(ks * 2);  // 32 bytes per K step, in 16-byte units of the start-address field
          const uint32_t first = (kc == 0 && ks == 0) ? 0u : 1u;
          tc::wg_ss_n128(acc0, dAh + adv, dBh + adv, first);  // acc0 (+)= Ah Bh
          tc::wg_ss_n128(acc1, dAh + adv, dBl + adv, first);  // acc1 (+)= Ah Bl
          tc::wg_ss_n128(acc1, dAl + adv, dBh + adv, 1u);     // acc1  += Al Bh
        }
        tc::wg_commit();
        if (kc > 0) {  // the previous chunk's MMAs have completed: release its stage
          tc::wg_wait<1>();
          if (lane == 0) tc::mbar_arrive(&empty[(gk - 1) % GW_STAGES]);
        }
      }
      tc::wg_wait<0>();
      if (lane == 0) tc::mbar_arrive(&empty[(gk - 1) % GW_STAGES]);

      // ===== epilogue from the accumulator fragment =====
      const GemmProblem& pb = g.p[z];
      const int M = pb.M, N = pb.N;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int n = n0 + 8 * j + c2;  // first of this thread's 2 columns
        if (n >= N) continue;
        const bool pair = n + 1 < N;
        const bool vec = pb.vec4 && pair;  // 8-byte fp32 and 4-byte plane accesses allowed
        float b2[2] = {0.f, 0.f};
        if (g.bias) {
          b2[0] = __ldg(g.bias + n);
          if (pair) b2[1] = __ldg(g.bias + n + 1);
        }
        const size_t hm_col = (size_t)(n >> 6) * M * 64 + (n & 63);  // head-major: [N / 64][M][64]
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + r0 + 8 * h;
          if (row >= M) continue;
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * j + 2 * h + e;
            v[e] = (fmaf(acc1[i], tc::LO_INV, acc0[i]) + b2[e]) * scale;
            if (relu) v[e] = fmaxf(v[e], 0.f);
          }
          if (pb.resid) {
            const float* rp = pb.resid + (size_t)row * g.ldr + n;
            if (vec) {
              const float2 rr = *reinterpret_cast<const float2*>(rp);
              v[0] += rr.x, v[1] += rr.y;
            } else {
              v[0] += rp[0];
              if (pair) v[1] += rp[1];
            }
          }
          const size_t off_c = g.head_major ? hm_col + (size_t)row * 64 : (size_t)row * pb.ldc + n;
          const size_t off_s = g.head_major ? hm_col + (size_t)row * 64 : (size_t)row * g.ldch + n;
          if (pb.C) {
            if (vec) {
              *reinterpret_cast<float2*>(pb.C + off_c) = make_float2(v[0], v[1]);
            } else {
              pb.C[off_c] = v[0];
              if (pair) pb.C[off_c + 1] = v[1];
            }
          }
          if (pb.Ch) {
            if (vec) {
              uint32_t h01, l01;
              if (g.lo_unscaled) tc::split2_unscaled_clamped(v[0], v[1], h01, l01);
              else tc::split2(v[0], v[1], h01, l01);
              *reinterpret_cast<uint32_t*>(pb.Ch + off_s) = h01;
              *reinterpret_cast<uint32_t*>(pb.Cl + off_s) = l01;
            } else {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (e == 0 || pair) {
                  __half hh, ll;
                  if (g.lo_unscaled) tc::split_h_unscaled(v[e], hh, ll);
                  else tc::split_h(v[e], hh, ll);
                  pb.Ch[off_s + e] = hh;
                  pb.Cl[off_s + e] = ll;
                }
              }
            }
          }
        }
      }
    }
  }
  if (!ok && g.err_flag) *g.err_flag = 1;
}
