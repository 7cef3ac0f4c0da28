// Tensor Memory Accelerator helpers shared by the wgmma kernels: TMA tile loads signalled on mbarriers (complete_tx),
// host-side tensor-map construction, and the fp32 -> split-fp16 plane kernel.
//
// Shared-memory tile = [rows][64 halves] with 128-byte rows, XOR-swizzled in 8-row x 128-byte atoms: the wgmma descriptor
// is layout SWIZZLE_128B, SBO = 1024 B (one atom), and one MMA K step (16 halves) advances the start address by 32 B.
// Tiles are 1024-byte aligned.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc.cuh"

namespace tc {
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* map, uint64_t* bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
}  // namespace tc

// ---- host: tensor-map construction (driver entry point resolved at run time: the library does not link libcuda) ------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline PFN_encodeTiled tma_encoder() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 2-D fp16 matrix [rows][ld] (K contiguous), box = 64 K-elements x box_rows rows (<= 256), 128-byte swizzle, zero OOB fill.
static inline bool tma_map_2d(CUtensorMap* out, const __half* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  PFN_encodeTiled enc = tma_encoder();
  if (!enc || !base) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(__half)};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// fp32 -> fp16 hi / lo * 2^11 planes (weights once at load time; network inputs once per call)
static __global__ void k_split_f32(const float* __restrict__ x, size_t n, __half* __restrict__ hi, __half* __restrict__ lo) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  __half h, l;
  tc::split_h(x[i], h, l);
  hi[i] = h;
  lo[i] = l;
}
