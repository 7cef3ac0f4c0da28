// Test-only entry points: run one GEMM through the SIMT fp32 kernel or the wgmma split-fp16 kernel (parity tests).
#include <stdlib.h>

#include "common.cuh"
#include "linear.cuh"

extern "C" int b2_debug_gemm_host(b2_context* ctx, int mode, const float* A, const float* B, const float* bias, float* C,
                                  int M, int N, int K) {
  if (!ctx || !A || !B || !C || M <= 0 || N <= 0 || K <= 0 || (K % 64)) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  DevBuf dA, dB, dC, dBias, dBh, dBl, dErr;
  B2_CUDA(ctx, dA.ensure((size_t)M * K * 4));
  B2_CUDA(ctx, dB.ensure((size_t)N * K * 4));
  B2_CUDA(ctx, dC.ensure((size_t)M * N * 4));
  B2_CUDA(ctx, dBias.ensure((size_t)N * 4));
  B2_CUDA(ctx, dErr.ensure(16));
  B2_CUDA(ctx, cudaMemcpyAsync(dA.p, A, (size_t)M * K * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dB.p, B, (size_t)N * K * 4, cudaMemcpyHostToDevice, st));
  if (bias) B2_CUDA(ctx, cudaMemcpyAsync(dBias.p, bias, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  int rc = B2_OK;
  if (mode == 0) {
    rc = launch_gemm(ctx, st, gemm_linear(dA.as<float>(), K, K, dB.as<float>(), bias ? dBias.as<float>() : nullptr, dC.as<float>(), N, M, N));
  } else {
    // modes 1 and 2 both run the wgmma kernel on operands split here (A and B as fp16 hi / lo planes)
    DevBuf dAh, dAl;
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
    rc = run_linear(ctx, st, tw, &a, 1);
    if (rc == B2_OK) {
      cudaError_t e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) rc = b2_fail(ctx, B2_ERR_CUDA, std::string("debug gemm: ") + cudaGetErrorString(e));
    }
    dAh.release(), dAl.release();
  }
  int err = 0;
  if (rc == B2_OK) {
    cudaError_t e = cudaMemcpyAsync(C, dC.p, (size_t)M * N * 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = b2_fail(ctx, B2_ERR_CUDA, std::string("debug gemm: ") + cudaGetErrorString(e));
  }
  dA.release(), dB.release(), dC.release(), dBias.release(), dBh.release(), dBl.release(), dErr.release();
  if (rc == B2_OK && err) rc = b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return rc;
}
