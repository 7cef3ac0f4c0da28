// Order-preserving top-k of one score array in one 1024-thread CTA (superpoint.cu's k_topk_select, sift.cu's k_sift_topk).
#pragma once

// The k largest scores (ties at the k-th value -> lowest indices), kept in their original order: 4-pass 8-bit radix select
// on the float bit patterns (scores are non-negative), then an ordered compaction.  Writes the selected indices (ascending)
// to out_idx and their number to *out_count.  Must be called by all 1024 threads of the block.
__device__ __forceinline__ void b2_topk_select_cta(const float* __restrict__ score, int n, int k, int* __restrict__ out_idx,
                                                   int* __restrict__ out_count) {
  __shared__ unsigned hist[256];
  __shared__ unsigned prefix, need;
  __shared__ int wtot[32];
  __shared__ int carry, eq_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (k >= n) {
    for (int i = threadIdx.x; i < n; i += 1024) out_idx[i] = i;
    if (threadIdx.x == 0) *out_count = n;
    return;
  }
  if (threadIdx.x == 0) prefix = 0, need = (unsigned)k;
  __syncthreads();
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const unsigned himask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = threadIdx.x; i < 256; i += 1024) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += 1024) {
      unsigned key = __float_as_uint(score[i]);
      if ((key & himask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned acc = 0;
      int b = 255;
      for (; b > 0; --b) {
        if (acc + hist[b] >= need) break;
        acc += hist[b];
      }
      need -= acc;  // how many still have to come from bin b
      prefix |= ((unsigned)b) << shift;
    }
    __syncthreads();
  }
  // prefix = bit pattern of the k-th largest score; take everything above it and the first `need` equal to it
  const unsigned T = prefix;
  if (threadIdx.x == 0) carry = 0, eq_carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    int i = base + threadIdx.x;
    unsigned key = i < n ? __float_as_uint(score[i]) : 0u;
    bool gt = i < n && key > T, eq = i < n && key == T;
    // rank among equals, in index order
    unsigned em = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) wtot[warp] = __popc(em);
    __syncthreads();
    if (warp == 0) {
      int w = wtot[lane], ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int u = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += u;
      }
      wtot[lane] = ws - w;
    }
    __syncthreads();
    int eq_rank = eq_carry + wtot[warp] + __popc(em & ((1u << lane) - 1));
    bool take = gt || (eq && (unsigned)eq_rank < need);
    __syncthreads();
    if (threadIdx.x == 1023) eq_carry = eq_rank + (eq ? 1 : 0);
    unsigned tm = __ballot_sync(0xffffffffu, take);
    if (lane == 0) wtot[warp] = __popc(tm);
    __syncthreads();
    if (warp == 0) {
      int w = wtot[lane], ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int u = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += u;
      }
      wtot[lane] = ws - w;
    }
    __syncthreads();
    int pos = carry + wtot[warp] + __popc(tm & ((1u << lane) - 1));
    if (take) out_idx[pos] = i;
    __syncthreads();
    if (threadIdx.x == 1023) carry = pos + (take ? 1 : 0);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out_count = carry;
}
