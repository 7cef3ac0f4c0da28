// Test-only entry points: run one GEMM through the SIMT fp32 kernel or the wgmma split-fp16 kernel (parity tests), the
// wgmma kernel's column-segment / rotary epilogue, and one batched launch of the split-fp16 flash attention kernel.
#include <stdlib.h>

#include <vector>

#include "common.cuh"
#include "linear.cuh"

// fp32 -> fp16 hi plane and UNSCALED lo plane (the operand format of the attention kernel)
static __global__ void k_split_unscaled_f32(const float* __restrict__ x, size_t n, __half* __restrict__ hi, __half* __restrict__ lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) tc::split_h_unscaled(x[i], hi[i], lo[i]);
}

extern "C" int b2_debug_gemm_host(b2_context* ctx, int mode, const float* A, const float* B, const float* bias, float* C,
                                  int M, int N, int K) {
  if (!ctx || !A || !B || !C || M <= 0 || N <= 0 || K <= 0 || (K % 64)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  DevBuf dA, dB, dC, dBias, dErr;
  B2_CUDA(ctx, dA.ensure((size_t)M * K * 4));
  B2_CUDA(ctx, dB.ensure((size_t)N * K * 4));
  B2_CUDA(ctx, dC.ensure((size_t)M * N * 4));
  B2_CUDA(ctx, dBias.ensure((size_t)N * 4));
  B2_CUDA(ctx, dErr.ensure(16));
  B2_CUDA(ctx, cudaMemcpyAsync(dA.p, A, (size_t)M * K * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dB.p, B, (size_t)N * K * 4, cudaMemcpyHostToDevice, st));
  if (bias) B2_CUDA(ctx, cudaMemcpyAsync(dBias.p, bias, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  if (mode == 0) {
    const int rc = launch_gemm(ctx, st, gemm_linear(dA.as<float>(), K, K, dB.as<float>(), bias ? dBias.as<float>() : nullptr, dC.as<float>(), N, M, N));
    if (rc != B2_OK) return rc;
  } else {
    // modes 1 and 2 both run the wgmma kernel on operands split here (A and B as fp16 hi / lo planes)
    DevBuf dAh, dAl, dBh, dBl;
    B2_CUDA(ctx, dAh.ensure((size_t)M * K * 2));
    B2_CUDA(ctx, dAl.ensure((size_t)M * K * 2));
    B2_CUDA(ctx, dBh.ensure((size_t)N * K * 2));
    B2_CUDA(ctx, dBl.ensure((size_t)N * K * 2));
    B2_LAUNCH(ctx, k_split_f32, (unsigned)(((size_t)M * K + 255) / 256), 256, 0, st, dA.as<float>(), (size_t)M * K, dAh.as<__half>(), dAl.as<__half>());
    B2_LAUNCH(ctx, k_split_f32, (unsigned)(((size_t)N * K + 255) / 256), 256, 0, st, dB.as<float>(), (size_t)N * K, dBh.as<__half>(), dBl.as<__half>());
    B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
    TcWeights tw{nullptr, nullptr, nullptr, dErr.as<int>(), true};
    tw.sm_count = ctx->sm_count;
    LinArgs a;
    a.a1p = {dAh.as<__half>(), dAl.as<__half>()}, a.lda1 = K, a.K1 = K, a.bp = {dBh.as<__half>(), dBl.as<__half>()}, a.ldb = K;
    a.bias = bias ? dBias.as<float>() : nullptr, a.cf = dC.as<float>(), a.ldc = N, a.tc_want_f32 = true, a.M = M, a.N = N;
    const int rc = run_linear(ctx, st, tw, &a, 1);
    if (rc != B2_OK) return rc;
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(C, dC.p, (size_t)M * N * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

extern "C" int b2_debug_gemm_segments_host(b2_context* ctx, const float* A, const float* B, const float* bias, int M, int K, int nseg,
                                           int rot_mask, const float* cs, const float* sn, int separate, uint16_t* out_hi, uint16_t* out_lo) {
  if (!ctx || !A || !B || !bias || !out_hi || !out_lo || M <= 0 || K <= 0 || (K % 64) || nseg < 1 || nseg > GW_SEGS ||
      (rot_mask && (!cs || !sn || separate)))
    return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int N = 256 * nseg;
  const size_t ep = (size_t)M * 256;  // halves of one segment's plane
  DevBuf dA, dB, dBias, dCs, dSn, dErr, dAh, dAl, dBh, dBl, dH, dL;
  B2_CUDA(ctx, dA.ensure((size_t)M * K * 4));
  B2_CUDA(ctx, dB.ensure((size_t)N * K * 4));
  B2_CUDA(ctx, dBias.ensure((size_t)N * 4));
  B2_CUDA(ctx, dCs.ensure((size_t)M * 32 * 4));
  B2_CUDA(ctx, dSn.ensure((size_t)M * 32 * 4));
  B2_CUDA(ctx, dErr.ensure(16));
  B2_CUDA(ctx, dAh.ensure((size_t)M * K * 2));
  B2_CUDA(ctx, dAl.ensure((size_t)M * K * 2));
  B2_CUDA(ctx, dBh.ensure((size_t)N * K * 2));
  B2_CUDA(ctx, dBl.ensure((size_t)N * K * 2));
  B2_CUDA(ctx, dH.ensure(nseg * ep * 2));
  B2_CUDA(ctx, dL.ensure(nseg * ep * 2));
  B2_CUDA(ctx, cudaMemcpyAsync(dA.p, A, (size_t)M * K * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dB.p, B, (size_t)N * K * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dBias.p, bias, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  if (rot_mask) {
    B2_CUDA(ctx, cudaMemcpyAsync(dCs.p, cs, (size_t)M * 32 * 4, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(dSn.p, sn, (size_t)M * 32 * 4, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  B2_LAUNCH(ctx, k_split_f32, (unsigned)(((size_t)M * K + 255) / 256), 256, 0, st, dA.as<float>(), (size_t)M * K, dAh.as<__half>(), dAl.as<__half>());
  B2_LAUNCH(ctx, k_split_f32, (unsigned)(((size_t)N * K + 255) / 256), 256, 0, st, dB.as<float>(), (size_t)N * K, dBh.as<__half>(), dBl.as<__half>());
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  TcWeights tw{nullptr, nullptr, nullptr, dErr.as<int>(), true};
  tw.sm_count = ctx->sm_count;
  __half *H = dH.as<__half>(), *L = dL.as<__half>(), *Bh = dBh.as<__half>(), *Bl = dBl.as<__half>();
  LinArgs a;
  a.a1p = {dAh.as<__half>(), dAl.as<__half>()}, a.lda1 = K, a.K1 = K, a.ldb = K, a.M = M, a.head_major = 1, a.lo_unscaled = 1;
  for (int s = 0; s < (separate ? nseg : 1); ++s) {
    if (separate) {  // segment s as a linear of its own: its 256 rows of B and of the bias
      a.bp = {Bh + (size_t)s * 256 * K, Bl + (size_t)s * 256 * K}, a.bias = dBias.as<float>() + s * 256, a.N = 256;
      a.cp = {H + s * ep, L + s * ep};
    } else {
      a.bp = {Bh, Bl}, a.bias = dBias.as<float>(), a.N = N, a.seg_n = 256;
      for (int j = 0; j < nseg; ++j) a.seg_p[j] = {H + j * ep, L + j * ep};
      a.rot_mask = rot_mask, a.cs = dCs.as<float>(), a.sn = dSn.as<float>();
    }
    const int rc = run_linear(ctx, st, tw, &a, 1);
    if (rc != B2_OK) return rc;
  }
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(out_hi, H, nseg * ep * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(out_lo, L, nseg * ep * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

extern "C" int b2_debug_attention_host(b2_context* ctx, int np, const int* nq, const int* nk, int heads, float scale, int single,
                                       const float* q, const float* k, const float* v, float* o) {
  if (!ctx || !nq || !nk || !q || !k || !v || !o || np <= 0 || np > AP_MAXP || heads <= 0) return B2_ERR_ARG;
  size_t eq = 0, ek = 0;  // elements of q (and o), of k (and v)
  for (int z = 0; z < np; ++z) {
    if (nq[z] <= 0 || nk[z] <= 0) return B2_ERR_ARG;
    eq += (size_t)nq[z] * heads * 64, ek += (size_t)nk[z] * heads * 64;
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t n = eq + 2 * ek;  // q, k, v back to back
  DevBuf dIn, dPl, dO, dErr, part, ml, cnt;
  B2_CUDA(ctx, dIn.ensure(n * 4));
  B2_CUDA(ctx, dPl.ensure(n * 2 * 2));
  B2_CUDA(ctx, dO.ensure(eq * 2 * 2));
  B2_CUDA(ctx, dErr.ensure(16));
  float* in = dIn.as<float>();
  B2_CUDA(ctx, cudaMemcpyAsync(in, q, eq * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + eq, k, ek * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + eq + ek, v, ek * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  __half *hi = dPl.as<__half>(), *lo = hi + n, *oh = dO.as<__half>(), *ol = oh + eq;
  B2_LAUNCH(ctx, k_split_unscaled_f32, (unsigned)((n + 255) / 256), 256, 0, st, in, n, hi, lo);
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  FlashPlanes fp[AP_MAXP];
  size_t qo = 0, ko = eq;
  for (int z = 0; z < np; ++z) {
    const size_t vo = ko + ek;
    fp[z] = {{hi + qo, lo + qo}, {hi + ko, lo + ko}, {hi + vo, lo + vo}, {oh + qo, ol + qo}, nq[z], nk[z], heads, 64 * heads};
    qo += (size_t)nq[z] * heads * 64, ko += (size_t)nk[z] * heads * 64;
  }
  TcWeights tw{nullptr, nullptr, nullptr, dErr.as<int>(), true};
  tw.attn_part = &part, tw.attn_ml = &ml, tw.attn_cnt = &cnt, tw.sm_count = ctx->sm_count;
  const int rc = run_flash_planes(ctx, st, tw, fp, np, scale, single != 0);
  if (rc != B2_OK) return rc;
  std::vector<__half> ho(2 * eq);
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(ho.data(), oh, eq * 2 * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  // o = hi + lo * 2^-11 (the SINGLE variant writes lo = 0)
  for (size_t i = 0; i < eq; ++i) o[i] = __half2float(ho[i]) + __half2float(ho[eq + i]) * tc::LO_INV;
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma attention timed out on an mbarrier (kernel bug)");
  return B2_OK;
}
