// Persistent warp-specialised wgmma + TMA flash attention over a BATCH of problems, split-fp16 operands (~fp32 accuracy).
//
//   O[Nq][ldo], columns 64 h .. 64 h + 63 = softmax(scale * Q_h K_h^T) V_h per head h (LightGlue / SuperGlue: 4 heads into
//   [Nq][256]; MegaLoc's DINOv2: 12 heads into [Nq][768]); q / k / v arrive as head-major [heads][N][64] fp16 hi / lo planes
//   with UNSCALED lo (x ~= hi + lo, lo = fp16(x - hi)), the output leaves as hi / lo planes with the usual 2^11-scaled lo.
//
// One CTA (384 threads, one per SM) owns TWO 128-query tiles of one head at a time and streams 64-key tiles.
//   warp 8 lane 0 : TMA producer - K and V tiles through one 4-entry ring (128-byte swizzled, zero OOB fill); warps 9-11
//                   only exist so that the producer has a warpgroup of its own for setmaxnreg
//   warps 0-3 / 4-7: consumer warpgroup of query tile 0 / 1, Q lo in shared memory and Q hi in registers.  Per key tile
//                   and 64-row slab: S = Qh Kh^T + Qh Kl^T + Ql Kh^T (the Qh products take A from registers, so they read
//                   only K from shared memory: with 64-wide tiles these MMAs are paced by shared-memory reads, and this
//                   removes a third of the QK traffic); base-2 online softmax on the fragment with a
//                   LAZY reference maximum (rescale only when the row maximum grew by more than 2^8: P <= 256 stays exact
//                   in the hi / lo split); O += Ph Vh + Ph Vl + Pl Vh (P from registers, V MN-major), O kept in registers.
// Software pipeline inside a consumer warpgroup: the softmax of one slab runs while the tensor core works on the other
// slab's MMAs.  Per key tile i:
//     QK(i, 0) QK(i, 1) | wait QK(i, 0) | softmax 0 | PV(i, 0) | wait QK(i, 1) | softmax 1 | PV(i, 1) | wait PV(i, *)
// While one warpgroup waits for its last PV, the other warpgroup's MMAs keep the tensor core busy.
// Every accumulator still receives the same MMAs in the same order, so the result is bit-identical to running the slabs one
// after the other.  Registers: 384 threads start at 168 each; setmaxnreg moves them to the consumers (240) and leaves the
// producer 24, which holds both O accumulators, Q hi of both slabs, one S being produced while the other is softmaxed, and
// the P planes that an in-flight PV MMA still reads, without spilling.
//
// Schedule ("stream-K" over the key dimension): the whole launch - every problem of the batch, i.e. the self- or
// cross-attention of all images of up to 8 pairs - is ONE linear space of (item, key tile) units, item = (problem, head,
// 256-query block), cut into equal contiguous ranges, one per SM.  A CTA therefore runs a few SEGMENTS (item, key-tile
// range) back to back: the barriers keep running phase counters and the TMA producer streams the next segment's K / V
// tiles while the current one drains.  A segment that covers its item completely writes the normalised output planes;
// otherwise it writes an un-normalised partial (O, m, l), and the LAST segment of an item to arrive (device-scope counter,
// stream-K "fix-up") combines the partials in the same kernel.  All barrier parities are functions of the running ring
// counter `ge` that every role advances identically.
#pragma once
#include "tma.cuh"

constexpr int AW_Q = 128, AW_KV = 64, AW_D = 64;
constexpr int AW_KV_BYTES = AW_KV * AW_D * 2;  // 8 KB per plane
constexpr int AS_NS = 4;                     // ring depth; entry e holds K tile e and V tile e - 2 (consumed together)
constexpr int AS_HALF = 2 * AW_KV_BYTES;     // hi + lo plane of one 64 x 64 tile = 16 KB
constexpr int AS_STAGE = 2 * AS_HALF;        // K part at +0, V part at +AS_HALF
constexpr int AS_TILE_BYTES = AS_NS * AS_STAGE;
constexpr int AS_Q_PLANE = AW_Q * AW_D * 2;  // 16 KB: one plane of a 128-query tile
constexpr int AS_Q_BYTES = 2 * AS_Q_PLANE;  // lo plane of both query tiles (Q hi is read into registers)
constexpr size_t AS_SMEM = AS_TILE_BYTES + AS_Q_BYTES + 1024 + 512;
constexpr int AS_THREADS = 256 + 128;  // 2 consumer warpgroups + TMA producer warpgroup (one thread works)
constexpr float AS_RESCALE = 8.0f;  // log2 of the largest P allowed before the reference maximum is refreshed
constexpr int AP_MAXP = 16;         // problems per launch (2 images x 8 pairs)

struct AttnPsMaps {
  CUtensorMap kh[AP_MAXP], kl[AP_MAXP], vh[AP_MAXP], vl[AP_MAXP];  // per problem; 2-D views [heads * N rows][64] of the head-major planes
};

struct AttnPsProblem {
  const __half *Qh, *Ql;  // head-major planes [heads][Nq][64]
  __half *Oh, *Ol;        // final output planes [Nq][ldo]
  int Nq, Nk;
  int ldo;                // output row pitch in halves (64 x heads when the heads fill the row)
  int qt, tiles;          // 256-query blocks, 64-key tiles
  int w_end;              // running total of (item, key tile) units up to and including this problem
  int item0;              // items (head x query block) of the problems before this one
};
struct AttnPsArgs {
  AttnPsProblem p[AP_MAXP];
  int nprob;
  float* Opart;  // [item][max_splits][256][64] fp32, un-normalised
  float* ml;     // [item][max_splits][256][2]
  int* arrivals; // [item][2] zero on entry; counts the partials of (item, query tile) written so far, reset by the merger
  int W;         // total units
  int quota;     // units per CTA
  int max_splits;
  float scale;
  int* err_flag;
};

struct AttnPsSeg {
  int z, item, h, q0, tile0, T, split, nsplits, itemg;
};
// segment starting at unit w (clipped to w_end)
__device__ __forceinline__ AttnPsSeg attn_ps_decode(const AttnPsArgs& a, int w, int w_end) {
  AttnPsSeg s;
  s.z = 0;
  while (s.z + 1 < a.nprob && w >= a.p[s.z].w_end) ++s.z;
  const AttnPsProblem& p = a.p[s.z];
  const int base = s.z ? a.p[s.z - 1].w_end : 0;
  const int wl = w - base;
  s.item = wl / p.tiles;
  s.tile0 = wl - s.item * p.tiles;
  s.T = min(p.tiles - s.tile0, w_end - w);
  s.h = s.item / p.qt;
  s.q0 = (s.item - s.h * p.qt) * (2 * AW_Q);
  const int wi0 = base + s.item * p.tiles, wi1 = wi0 + p.tiles;
  const int c_first = wi0 / a.quota;
  s.split = w / a.quota - c_first;
  s.nsplits = (wi1 - 1) / a.quota - c_first + 1;
  s.itemg = p.item0 + s.item;
  return s;
}

// SINGLE = the reference's CUDA numerics (lightglue.py:116-121: q, k, v cast to half, fp16 flash SDPA, result cast back):
// only the hi planes take part - ONE wgmma per product instead of three - and the output is rounded to fp16.  Opt-in
// (b2_lightglue_params.fp16_attention); the default exact path reproduces the fp32 CPU front-end.
template <bool SINGLE>
static __global__ void __launch_bounds__(AS_THREADS, 1) k_flash_ps(const __grid_constant__ AttnPsMaps maps, const __grid_constant__ AttnPsArgs args) {
  extern __shared__ unsigned char ap_raw[];
  const uint32_t raw = tc::smem_u32(ap_raw);
  const uint32_t smem0 = (raw + 1023u) & ~1023u;
  unsigned char* sm = ap_raw + (smem0 - raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + AS_TILE_BYTES + AS_Q_BYTES);
  uint64_t* kv_full = bars;                 // [AS_NS]
  uint64_t* kv_empty = kv_full + AS_NS;     // [AS_NS] one arrival per consumer warp
  volatile int* last_flag = reinterpret_cast<volatile int*>(kv_empty + AS_NS);  // [2] per consumer warpgroup

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int w_begin = blockIdx.x * args.quota;
  const int w_end = min(args.W, w_begin + args.quota);

  if (t == 0) {
    for (int i = 0; i < AS_NS; ++i) tc::mbar_init(&kv_full[i], 1), tc::mbar_init(&kv_empty[i], 8);
    tc::fence_mbar_init();
  }
  __syncthreads();
  bool ok = true;

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (warp == 8 && lane == 0) {
      // ===== TMA producer: ring entry e of a segment = K tile e (if any) + V tile e - 2 (if any) =====
      int ge = 0;
      for (int w = w_begin; w < w_end;) {
        const AttnPsSeg sg = attn_ps_decode(args, w, w_end);
        const int Nk = args.p[sg.z].Nk;
        for (int e = 0; e < sg.T + 2; ++e) {
          const int g = ge + e, s = g % AS_NS;
          if (g >= AS_NS) ok = tc::mbar_wait(&kv_empty[s], ((g / AS_NS) - 1) & 1) && ok;
          const bool hk = e < sg.T, hv = e >= 2;
          constexpr int PART = SINGLE ? AW_KV_BYTES : AS_HALF;  // bytes of one operand tile that are really fetched
          tc::mbar_expect_tx(&kv_full[s], (hk ? PART : 0) + (hv ? PART : 0));
          const uint32_t dst = smem0 + s * AS_STAGE;
          if (hk) {
            const int row = sg.h * Nk + (sg.tile0 + e) * AW_KV;
            tc::tma_load_2d(dst, &maps.kh[sg.z], &kv_full[s], 0, row);
            if (!SINGLE) tc::tma_load_2d(dst + AW_KV_BYTES, &maps.kl[sg.z], &kv_full[s], 0, row);
          }
          if (hv) {
            const int row = sg.h * Nk + (sg.tile0 + e - 2) * AW_KV;
            tc::tma_load_2d(dst + AS_HALF, &maps.vh[sg.z], &kv_full[s], 0, row);
            if (!SINGLE) tc::tma_load_2d(dst + AS_HALF + AW_KV_BYTES, &maps.vl[sg.z], &kv_full[s], 0, row);
          }
        }
        ge += sg.T + 2;
        w += sg.T;
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
    // ===== consumer warpgroup q: query rows q * 128 + slab * 64 + rq (+ 8) =====
    const int q = warp >> 2;
    const int r = t & 127;
    const int rq = (warp & 3) * 16 + (lane >> 2);  // fragment rows rq, rq + 8 of a slab
    const int c2 = (lane & 3) * 2;                 // fragment columns 8j + c2, + 1
    const uint32_t sQl = smem0 + AS_TILE_BYTES + q * AS_Q_PLANE;
    const float c2s = args.scale * 1.4426950408889634f;
    auto wg_bar = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + q) : "memory"); };
    auto release = [&](int g) { if (lane == 0) tc::mbar_arrive(&kv_empty[g % AS_NS]); };

    int ge = 0;
    for (int w = w_begin; w < w_end;) {
      const AttnPsSeg sg = attn_ps_decode(args, w, w_end);
      const AttnPsProblem& pr = args.p[sg.z];
      const int T = sg.T, Nk = pr.Nk;
      if (!SINGLE) {  // this thread's query row of the lo plane -> shared memory, 128-byte swizzled (zero rows past the end)
        const int qrow = sg.q0 + q * AW_Q + r;
        wg_bar();  // the previous segment's MMAs of every warp of the group have read Q lo
        const __half* src = pr.Ql + ((size_t)sg.h * pr.Nq + qrow) * 64;
        unsigned char* dst = sm + AS_TILE_BYTES + q * AS_Q_PLANE + r * 128;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          uint4 v = make_uint4(0u, 0u, 0u, 0u);
          if (qrow < pr.Nq) v = __ldg(reinterpret_cast<const uint4*>(src) + c);
          *reinterpret_cast<uint4*>(dst + ((c ^ (r & 7)) << 4)) = v;
        }
        tc::fence_proxy_async();  // generic-proxy stores -> visible to the tensor core
        wg_bar();
      }
      // Q hi of slab 0 / 1 also as register A fragments (k step ks: registers 4 ks .. 4 ks + 3): the QK products with Qh
      // then read only K from shared memory
      uint32_t qf[2][16];
#pragma unroll
      for (int sl = 0; sl < 2; ++sl)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int qrow = sg.q0 + q * AW_Q + sl * 64 + rq + 8 * h;
          const uint32_t* src = reinterpret_cast<const uint32_t*>(pr.Qh + ((size_t)sg.h * pr.Nq + qrow) * 64 + c2);
#pragma unroll
          for (int j = 0; j < 8; ++j) qf[sl][4 * (j >> 1) + 2 * (j & 1) + h] = qrow < pr.Nq ? __ldg(src + 4 * j) : 0u;
        }
      float o[2][32];
      float m_ref[2][2], l_i[2][2];
#pragma unroll
      for (int sl = 0; sl < 2; ++sl)
#pragma unroll
        for (int h = 0; h < 2; ++h) m_ref[sl][h] = -INFINITY, l_i[sl][h] = 0.f;
      float s[2][32];                 // S of slab 0 / 1
      uint32_t ph[2][16], pl[2][16];  // P hi / lo planes of slab 0 / 1: register A operands of the PV MMAs
      // S(sl) = Q(sl) K(i)^T: one commit group
      auto qk = [&](int i, int sl) {
        const uint32_t sK = smem0 + ((ge + i) % AS_NS) * AS_STAGE;
        const uint64_t dKh = tc::wg_desc_sw128(sK), dKl = tc::wg_desc_sw128(sK + AW_KV_BYTES);
        const uint64_t dQl = tc::wg_desc_sw128(sQl + sl * (64 * 128));
        tc::wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t adv = (uint64_t)(ks * 2);
          tc::wg_rs_n64(s[sl], qf[sl] + 4 * ks, dKh + adv, ks ? 1u : 0u);
          if (!SINGLE) {
            tc::wg_rs_n64(s[sl], qf[sl] + 4 * ks, dKl + adv, 1u);
            tc::wg_ss_n64(s[sl], dQl + adv, dKh + adv, 1u);
          }
        }
        tc::wg_commit();
      };
      // online softmax of S(sl) of key tile i -> P(sl), rescaling O(sl) when the reference maximum moves
      auto softmax = [&](int i, int sl) {
        float* a = s[sl];
        const int k0 = (sg.tile0 + i) * AW_KV;
        if (k0 + AW_KV > Nk) {
#pragma unroll
          for (int jj = 0; jj < 32; ++jj)
            if (k0 + 8 * (jj >> 2) + c2 + (jj & 1) >= Nk) a[jj] = -INFINITY;  // 2^(-inf) = 0
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {  // fragment row rq + 8h: a[4j + 2h + e]
          float mx = a[2 * h];
#pragma unroll
          for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(a[4 * j + 2 * h], a[4 * j + 2 * h + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m_ref[sl][h], mx * c2s);
          if (m_new - m_ref[sl][h] > AS_RESCALE) {  // also true on the first tile (m_ref = -inf); uniform over the quad
            const float corr = tc::ex2(m_ref[sl][h] - m_new);
            l_i[sl][h] *= corr;
            if (i > 0) {
#pragma unroll
              for (int j = 0; j < 8; ++j) o[sl][4 * j + 2 * h] *= corr, o[sl][4 * j + 2 * h + 1] *= corr;
            }
            m_ref[sl][h] = m_new;
          }
          float rs = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float p0 = tc::ex2(fmaf(a[4 * j + 2 * h], c2s, -m_ref[sl][h]));
            const float p1 = tc::ex2(fmaf(a[4 * j + 2 * h + 1], c2s, -m_ref[sl][h]));
            rs += p0 + p1;
            const __half2 hh = __floats2half2_rn(p0, p1);
            // A fragment of k step j / 2: registers (row rq, k 2c), (row rq + 8, k 2c), (row rq, k 2c + 8), (row rq + 8, ...)
            const int ri = 4 * (j >> 1) + 2 * (j & 1) + h;
            ph[sl][ri] = *reinterpret_cast<const uint32_t*>(&hh);
            if (!SINGLE) {
              const float2 hf = __half22float2(hh);
              const __half2 ll = __floats2half2_rn(p0 - hf.x, p1 - hf.y);  // p - hi, exact
              pl[sl][ri] = *reinterpret_cast<const uint32_t*>(&ll);
            }
          }
          l_i[sl][h] += rs;
        }
      };
      // O(sl) += P(sl) V(i): one commit group
      auto pv = [&](int i, int sl) {
        const uint32_t sV = smem0 + ((ge + i + 2) % AS_NS) * AS_STAGE + AS_HALF;
        const uint64_t dVh = tc::wg_desc_sw128(sV), dVl = tc::wg_desc_sw128(sV + AW_KV_BYTES);
        tc::wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t advV = (uint64_t)(ks * 128);  // 16 key rows of 128 bytes
          tc::wg_rs_n64_bt(o[sl], ph[sl] + 4 * ks, dVh + advV, (i | ks) ? 1u : 0u);
          if (!SINGLE) {
            tc::wg_rs_n64_bt(o[sl], ph[sl] + 4 * ks, dVl + advV, 1u);
            tc::wg_rs_n64_bt(o[sl], pl[sl] + 4 * ks, dVh + advV, 1u);
          }
        }
        tc::wg_commit();
      };

      // Ring entry ge + e holds K tile e (e < T) and V tile e - 2 (e >= 2); every entry is released exactly once, after all
      // MMAs that read it have completed.  Key tiles i - 1 and i share no MMA in flight: ptxas cannot count commit groups
      // across the loop's back edge and, if any were left in flight there, would serialise every MMA of the loop.
      for (int j = 0; j < 2; ++j) ok = tc::mbar_wait(&kv_full[(ge + j) % AS_NS], ((ge + j) / AS_NS) & 1) && ok;
      if (T == 1) release(ge + 1);  // ring entry 1 of a one-tile segment is empty but still cycles through the ring
      for (int i = 0; i < T; ++i) {
        // K tile i sits in an entry already waited for (the prologue, or V tile i - 2's entry)
        qk(i, 0);
        qk(i, 1);
        tc::wg_wait<1>();  // QK(i, 0) has completed; softmax 0 overlaps QK(i, 1)
        tc::fence_regs(s[0]);
        softmax(i, 0);
        const int gv = ge + i + 2;  // ring entry: V tile i and (if any) K tile i + 2
        ok = tc::mbar_wait(&kv_full[gv % AS_NS], (gv / AS_NS) & 1) && ok;
        pv(i, 0);
        tc::wg_wait<1>();  // QK(i, 1) has completed; softmax 1 overlaps PV(i, 0)
        tc::fence_regs(s[1]);
        release(ge + i);  // K tile i (and V tile i - 2)
        softmax(i, 1);
        pv(i, 1);
        tc::wg_wait<0>();
        tc::fence_regs(o[0]), tc::fence_regs(o[1]);
        if (i + 2 >= T) release(gv);  // an entry without a K tile: V tile i was its only content
      }
      ge += T + 2;
      w += T;
      // ---- this segment's result: row sums over the quad ----
#pragma unroll
      for (int sl = 0; sl < 2; ++sl)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          l_i[sl][h] += __shfl_xor_sync(0xffffffffu, l_i[sl][h], 1);
          l_i[sl][h] += __shfl_xor_sync(0xffffffffu, l_i[sl][h], 2);
        }
      auto write_row = [&](const float* v, float inv, int qrow) {  // v[4j + e] scaled by inv -> output dims 8j + c2 + e
        uint32_t* dh = reinterpret_cast<uint32_t*>(pr.Oh + (size_t)qrow * pr.ldo + sg.h * 64 + c2);
        uint32_t* dl = reinterpret_cast<uint32_t*>(pr.Ol + (size_t)qrow * pr.ldo + sg.h * 64 + c2);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          uint32_t hi, lo;
          if (SINGLE) {  // SDPA returns half: the message is the fp16 rounding of the fp32 accumulator
            const __half2 hh = __floats2half2_rn(tc::clamp_h(v[4 * j] * inv), tc::clamp_h(v[4 * j + 1] * inv));
            hi = *reinterpret_cast<const uint32_t*>(&hh), lo = 0u;
          } else {
            tc::split2(v[4 * j] * inv, v[4 * j + 1] * inv, hi, lo);
          }
          dh[4 * j] = hi;
          dl[4 * j] = lo;
        }
      };
      if (sg.nsplits == 1) {
#pragma unroll
        for (int sl = 0; sl < 2; ++sl)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int qrow = sg.q0 + q * AW_Q + sl * 64 + rq + 8 * h;
            if (qrow >= pr.Nq) continue;
            float v[32];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[4 * j] = o[sl][4 * j + 2 * h], v[4 * j + 1] = o[sl][4 * j + 2 * h + 1];
            write_row(v, 1.0f / l_i[sl][h], qrow);
          }
      } else {
        // partial of a cut item; the warpgroup that completes the item (last to arrive) merges all of them
        const size_t slot0 = (size_t)sg.itemg * args.max_splits;
#pragma unroll
        for (int sl = 0; sl < 2; ++sl)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int rl = q * AW_Q + sl * 64 + rq + 8 * h;
            if (sg.q0 + rl >= pr.Nq) continue;
            const size_t rowi = (slot0 + sg.split) * 256 + rl;
            float* dst = args.Opart + rowi * 64 + c2;
#pragma unroll
            for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[sl][4 * j + 2 * h], o[sl][4 * j + 2 * h + 1]);
            if (c2 == 0) *reinterpret_cast<float2*>(args.ml + rowi * 2) = make_float2(m_ref[sl][h], l_i[sl][h]);
          }
        __threadfence();  // partial visible device-wide before this warpgroup is counted
        wg_bar();
        if (r == 0) {
          int* cnt = args.arrivals + sg.itemg * 2 + q;
          const int old = atomicAdd(cnt, 1);
          const int last = old == sg.nsplits - 1;
          if (last) atomicExch(cnt, 0);  // nobody else touches it in this launch; zero again for the next one
          last_flag[q] = last;
        }
        wg_bar();
        if (last_flag[q]) {
          __threadfence();
#pragma unroll 1
          for (int sl = 0; sl < 2; ++sl)
#pragma unroll 1
            for (int h = 0; h < 2; ++h) {
              const int rl = q * AW_Q + sl * 64 + rq + 8 * h;
              const int qrow = sg.q0 + rl;
              if (qrow >= pr.Nq) continue;
              float m = -INFINITY;
              for (int sp = 0; sp < sg.nsplits; ++sp) m = fmaxf(m, __ldcg(args.ml + ((slot0 + sp) * 256 + rl) * 2));
              float l = 0.f, v[32];
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = 0.f;
              for (int sp = 0; sp < sg.nsplits; ++sp) {
                const size_t ri = (slot0 + sp) * 256 + rl;
                const float2 mlv = __ldcg(reinterpret_cast<const float2*>(args.ml + ri * 2));
                const float wgt = tc::ex2(mlv.x - m);
                l = fmaf(mlv.y, wgt, l);
                const float* src = args.Opart + ri * 64 + c2;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  const float2 x = __ldcg(reinterpret_cast<const float2*>(src + 8 * j));
                  v[4 * j] = fmaf(x.x, wgt, v[4 * j]), v[4 * j + 1] = fmaf(x.y, wgt, v[4 * j + 1]);
                }
              }
              write_row(v, 1.0f / l, qrow);
            }
        }
      }
    }
  }
  if (!ok && args.err_flag) *args.err_flag = 1;
}
