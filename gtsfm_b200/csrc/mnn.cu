// Two-way (mutual nearest neighbour) descriptor matching, gtsfm/frontend/matcher/twoway_matcher.py (`TwoWayMatcher`):
// cv2.BFMatcher(NORM_L2) knnMatch(k = 2) / match in both directions, optional ratio test, mutual check, rows ordered by
// the 1 -> 2 distance.  The n0 x n1 distance matrix is never written: k_mnn_top2 keeps each query row's best and second-best
// train rows in registers while it walks the train tiles.
//
// Arithmetic.  d^2 = |a|^2 + |b|^2 - 2 a.b, distance = sqrtf(d^2), candidates ordered by (float distance, train index), which
// is cv2's insertion rule in batchDistance (an equal distance keeps the lower index).
//   u8 path   (uint8 input, or float32 input holding integers in [0, 255] with D <= 258): wgmma u8 x u8 -> s32, d^2 in
//             int32, distance = sqrtf((float)d^2).  cv2 sums (a - b)^2 in float for both input types, which is exact while
//             D * 255^2 < 2^24 (D <= 258): there the result is bit-identical to cv2.  For uint8 with larger D the integer
//             d^2 is exact and cv2's float sum may round, so distances can differ from cv2's in the last bits.  The float
//             distance, not d^2, is the key: near d^2 ~ 2^23 distinct integers share one sqrtf and cv2 then keeps the lower
//             index.
//   fp16 path (everything else): split-fp16 operands, three MMAs into two fp32 accumulators (as k_gemm_ws), d^2 in fp32
//             clamped at 0.  Not bit-exact: cv2 sums (a - b)^2 directly in its own SIMD order.
// The path is a per-pair property of the input.  The prep kernel clears a per-image flag when a float32 row is not
// integer-valued in [0, 255]; both kernels are launched and each skips the pairs of the other, so the device path needs no
// host round trip before the one synchronisation at the end of the batch.
//
// Layout.  Every image of the batch (two per pair, no de-duplication) is one segment of a shared operand buffer, padded to
// a multiple of 128 rows, so one TMA map serves the whole launch and a problem is (query row offset, n, train row offset,
// n).  Each pair is two problems, (A, B) and (B, A), like the reference's two one-way matches.
//
// Schedule of k_mnn_top2 (one CTA per SM, persistent over work items = 128-row query tiles of all problems):
//   warps 0-7  consumer warpgroup w: query rows 64 w .. 64 w + 63 of the tile; per 128-column train tile, wgmma m64n128 over
//              the K chunks, then the selection epilogue on the register accumulators: a per-thread top 2 for each of its
//              two rows; the u8 path takes the sqrtf only for candidates whose integer d^2 is below the second-best's
//   warp 8     (lane 0) TMA producer: ring of (query chunk, train chunk) stages running ahead across train tiles and items
// At the end of an item the four lanes that share a row merge their lists (the merge keyed on (key, index) is associative).
#include "common.cuh"
#include "tma.cuh"

constexpr int MN_T = 128;        // rows per query tile and per train tile
constexpr int MN_THREADS = 384;  // two consumer warpgroups + the producer warpgroup (one thread works)
constexpr int MN_MAXN = 32768;   // rows per image
constexpr int MN_MAXD = 32768;   // |a|^2 of a u8 row stays below 2^31
constexpr int MN_U8_FLOAT_MAXD = 258;  // D * 255^2 < 2^24: cv2's float32 sums of integer-valued rows are exact
constexpr int MN_SORT_SMEM = 4096;     // finish kernel: survivors sorted in shared memory up to this count
constexpr int MN_FIN_THREADS = 1024;
constexpr int MN_PLANE = MN_T * 128;   // one operand tile: 128 rows x 128 bytes

template <bool U8>
struct MnCfg;
template <>
struct MnCfg<true> {
  static constexpr int KC = 128, PLANES = 1, STAGES = 4;  // 128 u8 per chunk
};
template <>
struct MnCfg<false> {
  static constexpr int KC = 64, PLANES = 2, STAGES = 3;  // 64 halves per chunk, hi and lo planes
};
template <bool U8>
constexpr int mn_stage_bytes() { return 2 * MnCfg<U8>::PLANES * MN_PLANE; }
template <bool U8>
constexpr size_t mn_smem() { return (size_t)MnCfg<U8>::STAGES * mn_stage_bytes<U8>() + 1024 + 256; }

struct MnnProb {  // one direction of one pair
  int q_off, nq, t_off, nt;  // query / train rows in the batch operand buffers
  int pair;
  int item_end;  // running total of 128-row query tiles up to and including this problem
};
struct MnnMaps {
  CUtensorMap a, b;  // u8: a = the u8 operands; fp16: a = hi plane, b = lo plane
};
struct MnnArgs {
  const MnnProb* probs;
  int nprob, items, nk;
  const int* seg_ok;  // per segment: nonzero = u8 path possible; a pair takes it when both of its segments allow it
  const int* norm_i;  // per buffer row: |a|^2 from the u8 values
  const float* norm_f;
  int* best;  // per buffer row (as query): best train index, its distance, the second-best distance
  float* d1;
  float* d2;
  int* err_flag;
};

struct MnnState {
  DevBuf u8, hi, lo, norm_i, norm_f, best, d1, d2, seg_ok, table, out_k, sort, err;
  DevBuf in0, in1, om, od;  // host entry point: inputs and outputs
};

void mn_destroy(b2_context* ctx) {
  delete ctx->mn;
  ctx->mn = nullptr;
}

struct MnnSeg {
  const void* src;
  int n, row0;  // rows row0 .. row0 + roundup(n, 128) of the operand buffers
};

// One warp per operand-buffer row (padding rows included, written as zeros): u8 and / or split-fp16 operands, both norms,
// and the per-segment integer-value flag.
__global__ void __launch_bounds__(256) k_mnn_prep(const MnnSeg* __restrict__ segs, int nseg, int rows, int dim, int dtype, int dp8,
                                                 int dp16, uint8_t* __restrict__ u8, __half* __restrict__ hi, __half* __restrict__ lo,
                                                 int* __restrict__ norm_i, float* __restrict__ norm_f, int* __restrict__ seg_ok) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  int lo_s = 0, hi_s = nseg - 1;  // last segment with row0 <= r
  while (lo_s < hi_s) {
    const int mid = (lo_s + hi_s + 1) >> 1;
    if (segs[mid].row0 <= r) lo_s = mid;
    else hi_s = mid - 1;
  }
  const MnnSeg sg = segs[lo_s];
  const int local = r - sg.row0;
  const bool valid = local < sg.n;
  const int width = dp8 > dp16 ? dp8 : dp16;
  int si = 0;
  double sf = 0.0;
  bool integral = true;
  for (int c = lane; c < width; c += 32) {
    float v = 0.f;
    if (valid && c < dim) {
      if (dtype == 1) v = (float)reinterpret_cast<const uint8_t*>(sg.src)[(size_t)local * dim + c];
      else v = reinterpret_cast<const float*>(sg.src)[(size_t)local * dim + c];
    }
    const bool vi = v >= 0.f && v <= 255.f && v == rintf(v);
    integral = integral && vi;
    const int q = vi ? (int)v : 0;
    si += q * q;
    sf += (double)v * (double)v;
    if (u8 && c < dp8) u8[(size_t)r * dp8 + c] = (uint8_t)q;
    if (hi && c < dp16) {
      __half h, l;
      tc::split_h(v, h, l);
      hi[(size_t)r * dp16 + c] = h;
      lo[(size_t)r * dp16 + c] = l;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    si += __shfl_xor_sync(0xffffffffu, si, o);
    sf += __shfl_xor_sync(0xffffffffu, sf, o);
  }
  if (!__all_sync(0xffffffffu, integral) && lane == 0) seg_ok[lo_s] = 0;
  if (lane == 0) norm_i[r] = si, norm_f[r] = (float)sf;
}

__device__ __forceinline__ bool mn_less(float ka, int ia, float kb, int ib) { return ka < kb || (ka == kb && ia < ib); }

template <bool U8>
static __global__ void __launch_bounds__(MN_THREADS, 1) k_mnn_top2(const __grid_constant__ MnnMaps maps, const __grid_constant__ MnnArgs g) {
  using Cfg = MnCfg<U8>;
  constexpr int STAGES = Cfg::STAGES, STAGE = mn_stage_bytes<U8>();
  extern __shared__ unsigned char mn_raw[];
  const uint32_t raw = tc::smem_u32(mn_raw);
  const uint32_t smem0 = (raw + 1023u) & ~1023u;
  unsigned char* sm = mn_raw + (smem0 - raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + STAGES * STAGE);
  uint64_t* empty = full + STAGES;  // one arrival per consumer warp

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  if (t == 0) {
    for (int s = 0; s < STAGES; ++s) tc::mbar_init(&full[s], 1), tc::mbar_init(&empty[s], 8);
    tc::fence_mbar_init();
    tc::tma_prefetch_desc(&maps.a);
    if (!U8) tc::tma_prefetch_desc(&maps.b);
  }
  __syncthreads();
  bool ok = true;

  // item -> (problem, first query row); `mine`: the pair takes this kernel's arithmetic (same answer in every role)
  auto decode = [&](int item, int& z, int& m0) {
    int lo = 0, hi = g.nprob - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (item < g.probs[mid].item_end) hi = mid;
      else lo = mid + 1;
    }
    z = lo;
    m0 = (item - (z ? g.probs[z - 1].item_end : 0)) * MN_T;
  };
  auto mine = [&](int z) {
    const int p = g.probs[z].pair;
    return ((g.seg_ok[2 * p] != 0) && (g.seg_ok[2 * p + 1] != 0)) == U8;
  };

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 8 && lane == 0) {
      // ===== TMA producer =====
      int gk = 0;
      for (int item = blockIdx.x; item < g.items; item += gridDim.x) {
        int z, m0;
        decode(item, z, m0);
        if (!mine(z)) continue;
        const MnnProb p = g.probs[z];
        for (int n0 = 0; n0 < p.nt; n0 += MN_T)
          for (int kc = 0; kc < g.nk; ++kc, ++gk) {
            const int s = gk % STAGES;
            if (gk >= STAGES) ok = tc::mbar_wait(&empty[s], ((gk / STAGES) - 1) & 1) && ok;
            const uint32_t sA = smem0 + s * STAGE, sB = sA + Cfg::PLANES * MN_PLANE;
            const int x = kc * Cfg::KC;
            tc::mbar_expect_tx(&full[s], STAGE);
            tc::tma_load_2d(sA, &maps.a, &full[s], x, p.q_off + m0);
            tc::tma_load_2d(sB, &maps.a, &full[s], x, p.t_off + n0);
            if (!U8) {
              tc::tma_load_2d(sA + MN_PLANE, &maps.b, &full[s], x, p.q_off + m0);
              tc::tma_load_2d(sB + MN_PLANE, &maps.b, &full[s], x, p.t_off + n0);
            }
          }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    // ===== consumer warpgroup wg =====
    const int wg = warp >> 2;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment rows rl, rl + 8 of the query tile
    const int c2 = (lane & 3) * 2;                           // fragment columns 8j + c2, + 1
    int gk = 0;
    for (int item = blockIdx.x; item < g.items; item += gridDim.x) {
      int z, m0;
      decode(item, z, m0);
      if (!mine(z)) continue;
      const MnnProb p = g.probs[z];
      // per row h: (key, index) of the best and second-best; key = float distance (u8) or fp32 d^2 (fp16); x1, x2: their
      // integer d^2 (u8)
      float k1[2], k2[2];
      int i1[2], i2[2], x1[2], x2[2], nai[2];
      float naf[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        k1[h] = k2[h] = INFINITY;
        i1[h] = i2[h] = x1[h] = x2[h] = 0x7fffffff;
        nai[h] = g.norm_i[p.q_off + m0 + rl + 8 * h];  // padding rows of the segment are zeros
        naf[h] = g.norm_f[p.q_off + m0 + rl + 8 * h];
      }
      for (int n0 = 0; n0 < p.nt; n0 += MN_T) {
        uint32_t acc[U8 ? 64 : 1];
        float acc0[U8 ? 1 : 64], acc1[U8 ? 1 : 64];
        for (int kc = 0; kc < g.nk; ++kc, ++gk) {
          const int s = gk % STAGES;
          ok = tc::mbar_wait(&full[s], (gk / STAGES) & 1) && ok;
          const uint32_t aS = smem0 + s * STAGE + wg * (64 * 128), bS = smem0 + s * STAGE + Cfg::PLANES * MN_PLANE;
          const uint64_t dA = tc::wg_desc_sw128(aS), dB = tc::wg_desc_sw128(bS);
          tc::wg_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint64_t adv = (uint64_t)(ks * 2);  // 32 bytes per K step, in 16-byte units of the start-address field
            const uint32_t first = (kc == 0 && ks == 0) ? 0u : 1u;
            if constexpr (U8) {
              tc::wg_ss_u8_n128(acc, dA + adv, dB + adv, first);
            } else {
              const uint64_t dAl = tc::wg_desc_sw128(aS + MN_PLANE), dBl = tc::wg_desc_sw128(bS + MN_PLANE);
              tc::wg_ss_n128(acc0, dA + adv, dB + adv, first);   // acc0 (+)= Ah Bh
              tc::wg_ss_n128(acc1, dA + adv, dBl + adv, first);  // acc1 (+)= Ah Bl
              tc::wg_ss_n128(acc1, dAl + adv, dB + adv, 1u);     // acc1  += Al Bh
            }
          }
          tc::wg_commit();
          if (kc > 0) {  // the previous chunk's MMAs have completed: release its stage
            tc::wg_wait<1>();
            if (lane == 0) tc::mbar_arrive(&empty[(gk - 1) % STAGES]);
          }
        }
        tc::wg_wait<0>();
        if (lane == 0) tc::mbar_arrive(&empty[(gk - 1) % STAGES]);

        // ===== selection epilogue =====
        // A thread visits its columns in increasing index order (n0, then j, then e), so a candidate has a higher index than
        // both entries it holds and enters only if its key is strictly below the second's.  With sqrtf monotone, u8 keys
        // below the second's need d^2 < x2: that integer test skips the sqrtf for all other candidates.
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = n0 + 8 * j + c2;  // even; the segment is padded to 128 rows, so col + 1 is inside it
          int2 nbi;
          float2 nbf;
          if (U8) nbi = *reinterpret_cast<const int2*>(g.norm_i + p.t_off + col);
          else nbf = *reinterpret_cast<const float2*>(g.norm_f + p.t_off + col);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = col + e;
            if (c >= p.nt) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * j + 2 * h + e;
              if constexpr (U8) {
                // sum (a - b)^2 < 2^31; the intermediate |a|^2 + |b|^2 may not be, so it wraps in unsigned arithmetic
                const int d2 = (int)((uint32_t)nai[h] + (uint32_t)(e ? nbi.y : nbi.x) - 2u * acc[i]);
                if (d2 >= x2[h]) continue;
                const float f = __fsqrt_rn((float)d2);
                if (f < k1[h]) {
                  k2[h] = k1[h], i2[h] = i1[h], x2[h] = x1[h];
                  k1[h] = f, i1[h] = c, x1[h] = d2;
                } else if (f < k2[h]) {
                  k2[h] = f, i2[h] = c, x2[h] = d2;
                }
              } else {
                const float dot = fmaf(acc1[i], tc::LO_INV, acc0[i]);
                const float d2 = fmaf(-2.f, dot, naf[h] + (e ? nbf.y : nbf.x));
                if (d2 < k1[h]) {
                  k2[h] = k1[h], i2[h] = i1[h];
                  k1[h] = d2, i1[h] = c;
                } else if (d2 < k2[h]) {
                  k2[h] = d2, i2[h] = c;
                }
              }
            }
          }
        }
      }
      // ===== merge the four lanes of each row, write =====
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float ok1 = __shfl_xor_sync(0xffffffffu, k1[h], o), ok2 = __shfl_xor_sync(0xffffffffu, k2[h], o);
          const int oi1 = __shfl_xor_sync(0xffffffffu, i1[h], o), oi2 = __shfl_xor_sync(0xffffffffu, i2[h], o);
          if (mn_less(ok1, oi1, k1[h], i1[h])) {
            if (mn_less(ok2, oi2, k1[h], i1[h])) k2[h] = ok2, i2[h] = oi2;
            else k2[h] = k1[h], i2[h] = i1[h];
            k1[h] = ok1, i1[h] = oi1;
          } else if (mn_less(ok1, oi1, k2[h], i2[h])) {
            k2[h] = ok1, i2[h] = oi1;
          }
        }
        const int row = m0 + rl + 8 * h;
        if ((lane & 3) == 0 && row < p.nq) {
          const size_t o = (size_t)p.q_off + row;
          g.best[o] = i1[h];
          g.d1[o] = U8 ? k1[h] : sqrtf(fmaxf(k1[h], 0.f));
          g.d2[o] = U8 ? k2[h] : sqrtf(fmaxf(k2[h], 0.f));
        }
      }
    }
  }
  if (!ok && g.err_flag) *g.err_flag = 1;
}

struct MnnPairOut {
  int64_t* matches;
  float* dist;
  int a_off, n0, b_off, n1;
  long long sort_off;  // this pair's global sort scratch (survivors beyond MN_SORT_SMEM)
};

// One CTA per pair: ratio test in double (the reference compares Python floats), mutual check, compaction, then a bitonic
// sort on the unique keys (distance bits, i0) - non-negative floats order like their bit patterns - and the int64 rows.
__global__ void __launch_bounds__(MN_FIN_THREADS) k_mnn_finish(const MnnPairOut* __restrict__ pairs, const int* __restrict__ best,
                                                              const float* __restrict__ d1, const float* __restrict__ d2, double ratio,
                                                              unsigned long long* __restrict__ gsort, int* __restrict__ out_k) {
  __shared__ unsigned long long skeys[MN_SORT_SMEM];
  __shared__ int cnt;
  const MnnPairOut po = pairs[blockIdx.x];
  const int tid = threadIdx.x;
  if (po.n0 == 0 || po.n1 == 0) {
    if (tid == 0) out_k[blockIdx.x] = 0;
    return;
  }
  const int cap = po.n0 < po.n1 ? po.n0 : po.n1;
  int cap2 = 1;
  while (cap2 < cap) cap2 <<= 1;
  unsigned long long* keys = cap2 <= MN_SORT_SMEM ? skeys : gsort + po.sort_off;
  if (tid == 0) cnt = 0;
  __syncthreads();
  for (int i = tid; i < po.n0; i += blockDim.x) {
    const int j = best[po.a_off + i];
    bool pass = best[po.b_off + j] == i;
    if (ratio >= 0.0)
      pass = pass && (double)d1[po.a_off + i] <= ratio * (double)d2[po.a_off + i] &&
             (double)d1[po.b_off + j] <= ratio * (double)d2[po.b_off + j];
    if (pass) keys[atomicAdd(&cnt, 1)] = ((unsigned long long)__float_as_uint(d1[po.a_off + i]) << 32) | (unsigned)i;
  }
  __syncthreads();
  const int K = cnt;
  int P = 1;
  while (P < K) P <<= 1;
  for (int i = K + tid; i < P; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          if ((a > b) == ((i & k) == 0)) keys[i] = b, keys[ixj] = a;
        }
      }
      __syncthreads();
    }
  for (int r = tid; r < K; r += blockDim.x) {
    const unsigned long long key = keys[r];
    const int i = (int)(key & 0xffffffffu);
    po.matches[2 * r] = i;
    po.matches[2 * r + 1] = best[po.a_off + i];
    if (po.dist) po.dist[r] = __uint_as_float((unsigned)(key >> 32));
  }
  if (tid == 0) out_k[blockIdx.x] = K;
}

static bool mn_map_u8(CUtensorMap* out, const uint8_t* base, uint64_t rows, uint64_t cols) {
  PFN_encodeTiled enc = tma_encoder();
  if (!enc || !base) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols};
  cuuint32_t box[2] = {128, (cuuint32_t)MN_T};
  cuuint32_t estr[2] = {1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int pad_rows(int n) { return cdiv(n, MN_T) * MN_T; }

// The batch: caller holds ctx->mu; device pointers in `pairs`; out_k written on the host structs.
static int mnn_run(b2_context* ctx, b2_mnn_pair* pairs, int n_pairs, int dim, int dtype, double ratio, cudaStream_t st) {
  if (n_pairs <= 0 || !pairs) return b2_fail(ctx, B2_ERR_ARG, "mnn: no pairs");
  if (dim < 1 || dim > MN_MAXD) return b2_fail(ctx, B2_ERR_ARG, "mnn: descriptor dimension must be in [1, 32768]");
  if (dtype != 0 && dtype != 1) return b2_fail(ctx, B2_ERR_ARG, "mnn: dtype must be 0 (float32) or 1 (uint8)");
  for (int p = 0; p < n_pairs; ++p) {
    const b2_mnn_pair& q = pairs[p];
    if (q.n0 < 0 || q.n1 < 0 || q.n0 > MN_MAXN || q.n1 > MN_MAXN)
      return b2_fail(ctx, B2_ERR_ARG, "mnn: at most 32768 descriptors per image");
    if ((q.n0 && !q.desc0) || (q.n1 && !q.desc1) || (q.n0 && q.n1 && !q.out_matches)) return b2_fail(ctx, B2_ERR_ARG, "mnn: null pointer");
    if (ratio >= 0.0 && q.n0 > 0 && q.n1 > 0 && (q.n0 < 2 || q.n1 < 2))
      return b2_fail(ctx, B2_ERR_MNN_RATIO, "mnn: the ratio test needs at least 2 descriptors on each side");
  }
  if (!ctx->mn) ctx->mn = new MnnState();
  MnnState* s = ctx->mn;
  const bool can_u8 = dtype == 1 || dim <= MN_U8_FLOAT_MAXD;
  const bool need_f16 = dtype == 0;
  const int dp8 = cdiv(dim, 128) * 128, dp16 = cdiv(dim, 64) * 64;

  // host tables: segments, problems, pair outputs
  std::vector<MnnSeg> segs(2 * n_pairs);
  std::vector<MnnProb> probs;
  std::vector<MnnPairOut> outs(n_pairs);
  int rows = 0, items = 0;
  long long sort_total = 0;
  for (int p = 0; p < n_pairs; ++p) {
    const b2_mnn_pair& q = pairs[p];
    segs[2 * p] = {q.desc0, q.n0, rows};
    rows += pad_rows(q.n0);
    segs[2 * p + 1] = {q.desc1, q.n1, rows};
    rows += pad_rows(q.n1);
    MnnPairOut& o = outs[p];
    o = {q.out_matches, q.out_dist, segs[2 * p].row0, q.n0, segs[2 * p + 1].row0, q.n1, sort_total};
    if (q.n0 == 0 || q.n1 == 0) continue;
    int cap = q.n0 < q.n1 ? q.n0 : q.n1, cap2 = 1;
    while (cap2 < cap) cap2 <<= 1;
    if (cap2 > MN_SORT_SMEM) sort_total += cap2;
    for (int d = 0; d < 2; ++d) {
      MnnProb pr;
      pr.q_off = d ? o.b_off : o.a_off, pr.nq = d ? q.n1 : q.n0;
      pr.t_off = d ? o.a_off : o.b_off, pr.nt = d ? q.n0 : q.n1;
      pr.pair = p;
      items += cdiv(pr.nq, MN_T);
      pr.item_end = items;
      probs.push_back(pr);
    }
  }
  const size_t seg_b = segs.size() * sizeof(MnnSeg), prob_b = probs.size() * sizeof(MnnProb), out_b = outs.size() * sizeof(MnnPairOut);
  std::vector<unsigned char> table(seg_b + prob_b + out_b);
  memcpy(table.data(), segs.data(), seg_b);
  if (prob_b) memcpy(table.data() + seg_b, probs.data(), prob_b);
  memcpy(table.data() + seg_b + prob_b, outs.data(), out_b);
  const size_t ro = (size_t)(rows > 0 ? rows : 1);
  B2_CUDA(ctx, s->table.ensure(table.size()));
  B2_CUDA(ctx, s->norm_i.ensure(ro * 4));
  B2_CUDA(ctx, s->norm_f.ensure(ro * 4));
  B2_CUDA(ctx, s->best.ensure(ro * 4));
  B2_CUDA(ctx, s->d1.ensure(ro * 4));
  B2_CUDA(ctx, s->d2.ensure(ro * 4));
  B2_CUDA(ctx, s->seg_ok.ensure(segs.size() * 4));
  B2_CUDA(ctx, s->out_k.ensure((size_t)n_pairs * 4));
  B2_CUDA(ctx, s->sort.ensure((size_t)(sort_total > 0 ? sort_total : 1) * 8));
  B2_CUDA(ctx, s->err.ensure(16));
  if (can_u8) B2_CUDA(ctx, s->u8.ensure(ro * dp8));
  if (need_f16) {
    B2_CUDA(ctx, s->hi.ensure(ro * dp16 * 2));
    B2_CUDA(ctx, s->lo.ensure(ro * dp16 * 2));
  }
  unsigned char* tab = s->table.as<unsigned char>();
  B2_CUDA(ctx, cudaMemcpyAsync(tab, table.data(), table.size(), cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(s->seg_ok.p, can_u8 ? 1 : 0, segs.size() * 4, st));  // nonzero = u8 path allowed
  B2_CUDA(ctx, cudaMemsetAsync(s->err.p, 0, 16, st));
  if (rows > 0) {
    B2_LAUNCH(ctx, k_mnn_prep, cdiv(rows, 8), 256, 0, st, reinterpret_cast<const MnnSeg*>(tab), (int)segs.size(), rows, dim, dtype, dp8,
              dp16, can_u8 ? s->u8.as<uint8_t>() : nullptr, need_f16 ? s->hi.as<__half>() : nullptr, need_f16 ? s->lo.as<__half>() : nullptr,
              s->norm_i.as<int>(), s->norm_f.as<float>(), s->seg_ok.as<int>());
    B2_CHECK_LAUNCH(ctx);
  }
  if (items > 0) {
    MnnArgs a;
    a.probs = reinterpret_cast<const MnnProb*>(tab + seg_b);
    a.nprob = (int)probs.size(), a.items = items;
    a.seg_ok = s->seg_ok.as<int>();
    a.norm_i = s->norm_i.as<int>(), a.norm_f = s->norm_f.as<float>();
    a.best = s->best.as<int>(), a.d1 = s->d1.as<float>(), a.d2 = s->d2.as<float>();
    a.err_flag = s->err.as<int>();
    const int sms = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
    const int grid = items < sms ? items : sms;
    if (can_u8) {
      MnnMaps m;
      memset(&m, 0, sizeof(m));
      if (!mn_map_u8(&m.a, s->u8.as<uint8_t>(), rows, dp8)) return b2_fail(ctx, B2_ERR_CUDA, "mnn: TMA map (u8) failed");
      m.b = m.a;
      a.nk = dp8 / 128;
      B2_CUDA(ctx, cudaFuncSetAttribute(k_mnn_top2<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mn_smem<true>()));
      B2_LAUNCH(ctx, k_mnn_top2<true>, grid, MN_THREADS, mn_smem<true>(), st, m, a);
      B2_CHECK_LAUNCH(ctx);
    }
    if (need_f16) {
      MnnMaps m;
      if (!tma_map_2d(&m.a, s->hi.as<__half>(), rows, dp16, dp16, MN_T) || !tma_map_2d(&m.b, s->lo.as<__half>(), rows, dp16, dp16, MN_T))
        return b2_fail(ctx, B2_ERR_CUDA, "mnn: TMA map (fp16) failed");
      a.nk = dp16 / 64;
      B2_CUDA(ctx, cudaFuncSetAttribute(k_mnn_top2<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mn_smem<false>()));
      B2_LAUNCH(ctx, k_mnn_top2<false>, grid, MN_THREADS, mn_smem<false>(), st, m, a);
      B2_CHECK_LAUNCH(ctx);
    }
  }
  B2_LAUNCH(ctx, k_mnn_finish, n_pairs, MN_FIN_THREADS, 0, st, reinterpret_cast<const MnnPairOut*>(tab + seg_b + prob_b), s->best.as<int>(),
            s->d1.as<float>(), s->d2.as<float>(), ratio, s->sort.as<unsigned long long>(), s->out_k.as<int>());
  B2_CHECK_LAUNCH(ctx);
  // counts, the pipeline fault flag and the per-image path flags come back in the batch's one synchronisation
  std::vector<int> ks(n_pairs + 1 + segs.size());
  int* seg_ok = ks.data() + n_pairs + 1;
  B2_CUDA(ctx, cudaMemcpyAsync(ks.data(), s->out_k.p, (size_t)n_pairs * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(ks.data() + n_pairs, s->err.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(seg_ok, s->seg_ok.p, segs.size() * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (ks[n_pairs]) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  for (int p = 0; p < n_pairs; ++p) {
    pairs[p].out_k = ks[p];
    // profiler work, 2 n0 n1 Dpad per direction, credited to the instance that ran the pair (b2_profile_start("k_mnn_top2")
    // times both instances, "k_mnn_top2<true>" / "k_mnn_top2<false>" one of them)
    const bool u8 = seg_ok[2 * p] && seg_ok[2 * p + 1];
    b2_prof_work(ctx, u8 ? "k_mnn_top2<true>" : "k_mnn_top2<false>", 2.0 * 2.0 * pairs[p].n0 * (double)pairs[p].n1 * (u8 ? dp8 : dp16));
  }
  return B2_OK;
}

extern "C" int b2_mnn_match_batched_dev(b2_context* ctx, b2_mnn_pair* pairs, int n_pairs, int dim, int dtype, double ratio, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  return mnn_run(ctx, pairs, n_pairs, dim, dtype, ratio, (cudaStream_t)stream);
}

// float32 rows that all hold integers in [0, 255] (cv2 SIFT) travel as uint8: the u8 path's input, a quarter of the bytes
static bool mn_integral(const float* x, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (!(x[i] >= 0.f && x[i] <= 255.f && x[i] == rintf(x[i]))) return false;
  return true;
}

extern "C" int b2_mnn_match_host(b2_context* ctx, const void* desc0, int n0, const void* desc1, int n1, int dim, int dtype, double ratio,
                                 int64_t* out_matches, float* out_dist, int* out_k) {
  if (!ctx || !out_k || (n0 > 0 && !desc0) || (n1 > 0 && !desc1) || (n0 > 0 && n1 > 0 && !out_matches)) return B2_ERR_ARG;
  if (dim < 1 || dim > MN_MAXD || (dtype != 0 && dtype != 1) || n0 < 0 || n1 < 0 || n0 > MN_MAXN || n1 > MN_MAXN)
    return b2_fail(ctx, B2_ERR_ARG, "mnn: bad sizes or dtype");
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->mn) ctx->mn = new MnnState();
  MnnState* s = ctx->mn;
  cudaStream_t st = ctx->stream;
  std::vector<uint8_t> c0, c1;
  if (dtype == 0 && dim <= MN_U8_FLOAT_MAXD && mn_integral((const float*)desc0, (size_t)n0 * dim) &&
      mn_integral((const float*)desc1, (size_t)n1 * dim)) {
    c0.resize((size_t)n0 * dim + 1), c1.resize((size_t)n1 * dim + 1);
    for (size_t i = 0; i < (size_t)n0 * dim; ++i) c0[i] = (uint8_t)((const float*)desc0)[i];
    for (size_t i = 0; i < (size_t)n1 * dim; ++i) c1[i] = (uint8_t)((const float*)desc1)[i];
    desc0 = c0.data(), desc1 = c1.data(), dtype = 1;
  }
  const size_t es = dtype == 1 ? 1 : 4, b0 = (size_t)n0 * dim * es, b1 = (size_t)n1 * dim * es;
  const int cap = n0 < n1 ? n0 : n1;
  B2_CUDA(ctx, s->in0.ensure(b0 + 16));
  B2_CUDA(ctx, s->in1.ensure(b1 + 16));
  B2_CUDA(ctx, s->om.ensure((size_t)(cap > 0 ? cap : 1) * 16));
  B2_CUDA(ctx, s->od.ensure((size_t)(cap > 0 ? cap : 1) * 4));
  if (b0) B2_CUDA(ctx, cudaMemcpyAsync(s->in0.p, desc0, b0, cudaMemcpyHostToDevice, st));
  if (b1) B2_CUDA(ctx, cudaMemcpyAsync(s->in1.p, desc1, b1, cudaMemcpyHostToDevice, st));
  ctx->h2d_bytes += b0 + b1;
  b2_mnn_pair pr{s->in0.p, n0, s->in1.p, n1, s->om.as<int64_t>(), out_dist ? s->od.as<float>() : nullptr, 0};
  const int rc = mnn_run(ctx, &pr, 1, dim, dtype, ratio, st);
  if (rc) return rc;
  *out_k = pr.out_k;
  if (pr.out_k > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(out_matches, s->om.p, (size_t)pr.out_k * 16, cudaMemcpyDeviceToHost, st));
    if (out_dist) B2_CUDA(ctx, cudaMemcpyAsync(out_dist, s->od.p, (size_t)pr.out_k * 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return B2_OK;
}
