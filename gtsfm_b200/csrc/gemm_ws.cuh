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
//   warps 0-7        consumer warpgroup w: rows 64w .. 64w + 63 of the 128 x 128 tile, wgmma m64n128k16 into two register
//                    accumulators; at the end of the tile they write fmaf(acc1, 2^-11, acc0) as fp32 into a shared
//                    staging tile and go straight on to the next tile's MMAs
//   warps 8-11       epilogue warpgroup: reads the staging tile row by row and applies bias / scale / ReLU / residual,
//                    then writes fp32 and / or split planes with 16-byte (fp32) and 8-byte (plane) coalesced stores
//   warp 12 (lane 0) TMA producer: a 2-stage ring (2 x 64 KB) that runs ahead into the next tile's K chunks; warps 13-15
//                    only exist so that the producer has a warpgroup of its own for setmaxnreg
// With K = 256 or 512 a tile is only 6 k - 12 k tensor cycles while its epilogue writes 64 - 192 KB, so the epilogue, not
// the operand traffic, paces the linears: running it in the consumers left the tensor cores idle for the whole of it.
// Here the epilogue of tile t overlaps the MMAs of tile t + 1; the single staging buffer is handed over with two
// mbarriers (sfull: 256 consumer arrivals, sempty: 128 epilogue arrivals).
// Registers: 512 threads start at 128 each; setmaxnreg moves them to the consumers (184), leaving the epilogue 104 and the
// producer 40 (ptxas: no spills, no serialised wgmma).  Without the rebalance, a fourth epilogue warp (416 threads) made
// ptxas cap the kernel at 128 registers and spill the accumulators; with 3 epilogue warps and no rebalance the family took
// 91-93 ms per vga_lightglue step against 85 ms with 4 (H100 80GB HBM3, three alternated runs each).
// Shared memory: 2 x 64 KB ring + 68 KB staging (a third ring stage no longer fits).  The epilogue computes exactly what
// the consumers used to: (fmaf(acc1, 2^-11, acc0) + bias) * scale, ReLU or GELU, + residual, then the same split helpers.  Its
// mode flags (relu, gelu, head-major, unscaled lo, which outputs) are read once per tile and are warp-uniform; they are not
// compile-time specialisations.
// Column segments (seg_n > 0): output columns s * seg_n .. (s + 1) * seg_n - 1 go to their own head-major planes Ch[s] / Cl[s],
// so one launch can write several attention operands (LightGlue's q | k | v, or the cross block's q | v).  A segment whose
// bit is set in rot_mask gets the rotary encoding of lightglue.py:58-65 from the problem's cos / sin table [M][32] before
// the split: an epilogue lane's 4 columns are two whole (2p, 2p + 1) pairs, and the product / sum sequence is the one of
// k_lg_split_rotary, so the planes are bit-identical to an fp32 GEMM output rotated and split in a second kernel.
#pragma once
#include "tma.cuh"

constexpr int GW_MAXP = 16;  // problems per launch (2 images x 8 pairs)
constexpr int GW_M = 128, GW_N = 128, GW_K = 64;
constexpr int GW_A_BYTES = GW_M * GW_K * 2;  // 16 KB per plane
constexpr int GW_B_BYTES = GW_N * GW_K * 2;  // 16 KB per plane
constexpr int GW_STAGE_BYTES = 2 * GW_A_BYTES + 2 * GW_B_BYTES;  // 64 KB
constexpr int GW_STAGES = 2;
// staging pitch in floats: 136 = 8 (mod 32) puts the 4 rows of a half-warp's 8-byte fragment stores on disjoint banks
constexpr int GW_PITCH = GW_N + 8;
constexpr int GW_STG_BYTES = GW_M * GW_PITCH * 4;  // 68 KB
constexpr int GW_RB = 8;  // epilogue rows per warp whose residual loads are in flight together
constexpr int GW_EW = 4;  // epilogue warps
constexpr int GW_THREADS = 512;  // two consumer warpgroups, the epilogue warpgroup, the producer warpgroup (one thread works)
constexpr size_t GW_SMEM = GW_STAGES * GW_STAGE_BYTES + GW_STG_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int GW_SEGS = 3;  // column segments per problem

struct GemmProblem {
  const float* resid;  // [M][ldr] fp32 or null, added after bias / scale
  float* C;            // optional fp32 output, row-major [M][ldc]
  __half *Ch[GW_SEGS], *Cl[GW_SEGS];  // optional split output planes; [0] unless the launch has column segments
  const float *cs, *sn;               // rotary table [M][32] (segments with a rot_mask bit)
  int M, N, ldc;
  int vec4;      // outputs / residual may be accessed 4 columns at a time (host checks 16-byte alignment of bases and lds)
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
  int gelu;        // exact (erf) GELU after bias / scale, before the residual
  int lo_unscaled; // split outputs keep lo = fp16(x - hi) (attention operands)
  int seg_n;       // > 0: columns per segment (a multiple of GW_N; head_major, plane outputs only, every access 4-wide)
  int rot_mask;    // bit s: rotary on segment s
  int* err_flag;   // set to 1 if an mbarrier wait timed out (pipeline bug): results are then invalid
};

// exact (erf) GELU; out of line, so that the epilogue's unrolled row loop does not carry eight inlined copies of erff
static __device__ __noinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

static __global__ void __launch_bounds__(GW_THREADS, 1) k_gemm_ws(const __grid_constant__ GemmWsMaps maps, const __grid_constant__ GemmWsArgs g) {
  extern __shared__ unsigned char gw_raw[];
  const uint32_t raw = tc::smem_u32(gw_raw);
  const uint32_t smem0 = (raw + 1023u) & ~1023u;
  unsigned char* sm = gw_raw + (smem0 - raw);
  float* stg = reinterpret_cast<float*>(sm + GW_STAGES * GW_STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + GW_STAGES * GW_STAGE_BYTES + GW_STG_BYTES);
  uint64_t* empty = full + GW_STAGES;  // one arrival per consumer warp
  uint64_t* sfull = empty + GW_STAGES;  // staging tile written: every consumer thread arrives
  uint64_t* sempty = sfull + 1;         // staging tile read: every epilogue thread arrives

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int nk = (g.K1 + g.K2) / GW_K;

  if (t == 0) {
    for (int s = 0; s < GW_STAGES; ++s) tc::mbar_init(&full[s], 1), tc::mbar_init(&empty[s], 8);
    tc::mbar_init(sfull, 256);
    tc::mbar_init(sempty, 32 * GW_EW);
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

  if (warp >= 12) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 12 && lane == 0) {
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
  } else if (warp < 8) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 184;\n" ::: "memory");
    // ===== consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of every tile =====
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment rows r0, r0 + 8
    const int c2 = (lane & 3) * 2;                           // fragment columns 8j + c2, + 1
    int gk = 0, it = 0;
    for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x, ++it) {
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

      // ===== hand the combined accumulators to the epilogue warps =====
      if (it > 0) ok = tc::mbar_wait(sempty, (it - 1) & 1) && ok;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 4 * j + 2 * h;
          *reinterpret_cast<float2*>(stg + (r0 + 8 * h) * GW_PITCH + 8 * j + c2) =
              make_float2(fmaf(acc1[i], tc::LO_INV, acc0[i]), fmaf(acc1[i + 1], tc::LO_INV, acc0[i + 1]));
        }
      tc::mbar_arrive(sfull);
    }
  } else {
    // ===== epilogue: warp 8 + ew takes rows ew, ew + 4, ...; lane takes columns 4 lane .. 4 lane + 3 =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 104;\n" ::: "memory");
    const int ew = warp - 8;
    const int c = 4 * lane;
    const float scale = g.scale;
    const int relu = g.relu, gelu = g.gelu, hm = g.head_major, lo_unscaled = g.lo_unscaled, ldr = g.ldr, ldch = g.ldch;
    int it = 0;
    for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x, ++it) {
      int z, m0, n0;
      decode(tile, z, m0, n0);
      const GemmProblem& pb = g.p[z];
      const float* resid = pb.resid;
      float* C = pb.C;
      const int sg = g.seg_n ? n0 / g.seg_n : 0;  // column segment of this tile
      __half *Ch = pb.Ch[sg], *Cl = pb.Cl[sg];
      const bool rot = (g.rot_mask >> sg) & 1;
      const int M = pb.M, ldc = pb.ldc;
      const int n = n0 + c;
      const int ncols = min(4, pb.N - n);  // this thread's valid columns (<= 0 past the end)
      const bool vec = pb.vec4 && ncols == 4;
      const int rows = min(GW_M, M - m0);
      float b4[4] = {0.f, 0.f, 0.f, 0.f};
      if (g.bias)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (e < ncols) b4[e] = __ldg(g.bias + n + e);
      const int ns = n - sg * g.seg_n;  // column inside the segment
      const size_t hm_col = (size_t)(ns >> 6) * M * 64 + (ns & 63);  // head-major: [N / 64][M][64] (4 columns stay in one head)
      // Rows go in batches of GW_RB per warp with the batch's residual loads issued together (the first batch's before the
      // staging wait), so the residual's DRAM latency is paid once per batch rather than once per row.  In-place use
      // (resid == C) stays safe: every element is read and then written by this thread alone.  A rotary segment has no
      // residual and loads its rows' (cos, cos, sin, sin) of pairs p, p + 1 into the same registers.
      const bool vres = resid && vec;
      const int rp = (ns & 63) >> 1;  // first rotary pair of this thread's columns
      float4 rr[GW_RB];
      auto load_rows = [&](int rb) {  // the branch stays outside the loops: each batch's loads go out back to back
        if (rot) {
#pragma unroll
          for (int i = 0; i < GW_RB; ++i)
            if (rb + GW_EW * i < rows) {
              const size_t o = (size_t)(m0 + rb + GW_EW * i) * 32 + rp;
              const float2 cc = __ldg(reinterpret_cast<const float2*>(pb.cs + o)), ss = __ldg(reinterpret_cast<const float2*>(pb.sn + o));
              rr[i] = make_float4(cc.x, cc.y, ss.x, ss.y);
            }
        } else {
#pragma unroll
          for (int i = 0; i < GW_RB; ++i)
            if (rb + GW_EW * i < rows) rr[i] = *reinterpret_cast<const float4*>(resid + (size_t)(m0 + rb + GW_EW * i) * ldr + n);
        }
      };
      if (vres || rot) load_rows(ew);
      ok = tc::mbar_wait(sfull, it & 1) && ok;
      auto pre = [&](int r, float* v) {  // staged accumulators -> (. + bias) * scale, ReLU / GELU
        const float4 a = *reinterpret_cast<const float4*>(stg + r * GW_PITCH + c);
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[e] = (v[e] + b4[e]) * scale;
          if (relu) v[e] = fmaxf(v[e], 0.f);
          if (gelu) v[e] = gelu_erf(v[e]);
        }
      };
      if (ncols > 0 && vec) {
        for (int rb = ew; rb < rows; rb += GW_EW * GW_RB) {
          if ((vres || rot) && rb != ew) load_rows(rb);
#pragma unroll
          for (int i = 0; i < GW_RB; ++i) {
            const int r = rb + GW_EW * i;
            if (r >= rows) break;
            const int row = m0 + r;
            float v[4];
            pre(r, v);
            if (resid) v[0] += rr[i].x, v[1] += rr[i].y, v[2] += rr[i].z, v[3] += rr[i].w;
            if (rot) {  // (t * cos) + (rotate_half(t) * sin), rotate_half: (x1, x2) -> (-x2, x1)
              const float c0 = rr[i].x, c1 = rr[i].y, s0 = rr[i].z, s1 = rr[i].w;
              const float a0 = __fadd_rn(__fmul_rn(v[0], c0), __fmul_rn(-v[1], s0)), a1 = __fadd_rn(__fmul_rn(v[1], c0), __fmul_rn(v[0], s0));
              const float a2 = __fadd_rn(__fmul_rn(v[2], c1), __fmul_rn(-v[3], s1)), a3 = __fadd_rn(__fmul_rn(v[3], c1), __fmul_rn(v[2], s1));
              v[0] = a0, v[1] = a1, v[2] = a2, v[3] = a3;
            }
            const size_t off = hm ? hm_col + (size_t)row * 64 : (size_t)row * ldc + n;
            if (C) *reinterpret_cast<float4*>(C + off) = make_float4(v[0], v[1], v[2], v[3]);
            if (Ch) {
              const size_t off_s = hm ? off : (size_t)row * ldch + n;
              uint32_t h01, l01, h23, l23;
              if (lo_unscaled) {
                tc::split2_unscaled_clamped(v[0], v[1], h01, l01);
                tc::split2_unscaled_clamped(v[2], v[3], h23, l23);
              } else {
                tc::split2(v[0], v[1], h01, l01);
                tc::split2(v[2], v[3], h23, l23);
              }
              *reinterpret_cast<uint2*>(Ch + off_s) = make_uint2(h01, h23);
              *reinterpret_cast<uint2*>(Cl + off_s) = make_uint2(l01, l23);
            }
          }
        }
      } else if (ncols > 0) {
        // the cold path (a ragged last column tile, or outputs without 16-byte alignment): element by element, one row at a
        // time, kept out of the unrolled loop above so that the hot loop's code stays small
#pragma unroll 1
        for (int r = ew; r < rows; r += GW_EW) {
          const int row = m0 + r;
          float v[4];
          pre(r, v);
          const size_t off_c = hm ? hm_col + (size_t)row * 64 : (size_t)row * ldc + n;
          const size_t off_s = hm ? hm_col + (size_t)row * 64 : (size_t)row * ldch + n;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (e >= ncols) break;
            if (resid) v[e] += resid[(size_t)row * ldr + n + e];
            if (C) C[off_c + e] = v[e];
            if (Ch) {
              __half hh, ll;
              if (lo_unscaled) tc::split_h_unscaled(v[e], hh, ll);
              else tc::split_h(v[e], hh, ll);
              Ch[off_s + e] = hh;
              Cl[off_s + e] = ll;
            }
          }
        }
      }
      tc::mbar_arrive(sempty);
    }
  }
  if (!ok && g.err_flag) *g.err_flag = 1;
}
