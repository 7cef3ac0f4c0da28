// Retrieval front (SURVEY.md section 8f rank 4): the pair-selection step that precedes the hot path,
// gtsfm/retriever/similarity_retriever.py:86-260 (`SimilarityRetriever.get_image_pairs`): similarity matrix
// sim = G G^T of the global image descriptors (:93-157, torch.einsum on blocks of 50), then per query image the
// `num_matched` best-scoring partners among j > i with score >= min_score (`pairs_from_score_matrix`, :232-260: invalid =
// lower triangle + diagonal + below min_score -> -inf, torch.topk per row, finite entries kept in (row, rank) order).
// The global descriptors come from netvlad.cu (NetVLAD) or from the reference's own networks (MegaLoc).
//
// sim runs on the shared split-fp16 wgmma GEMM (fp32-equivalent); the selection is one warp per query row: `num_matched`
// rounds of a warp arg-max over the row's valid entries strictly "after" the previous pick in (score desc, index asc) order.
#include "common.cuh"
#include "linear.cuh"

constexpr int RT_KC = 256;

struct RetrievalState {
  DevBuf g, gh, gl, sim, pairs, count, err;
};

void rt_destroy(b2_context* ctx) {
  delete ctx->rt;
  ctx->rt = nullptr;
}

// out[i][r] = index of the r-th best valid partner of row i, or -1
__global__ void __launch_bounds__(256) k_rt_topk(const float* __restrict__ sim, int n, int k, float min_score, int* __restrict__ out) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const float* row = sim + (size_t)i * n;
  float pv = INFINITY;  // previous pick (value, index): strictly later entries only
  int pi = -1;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = i + 1 + lane; j < n; j += 32) {  // j > i: upper triangle without the diagonal
      const float v = row[j];
      if (!(v >= min_score)) continue;
      if (!(v < pv || (v == pv && j > pi))) continue;
      if (v > bv || (v == bv && j < bi)) bv = v, bi = j;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
    }
    if (lane == 0) out[(size_t)i * k + r] = bi == 0x7fffffff ? -1 : bi;
    if (bi == 0x7fffffff) {  // row exhausted: the remaining ranks are empty
      for (int rr = r + 1 + lane; rr < k; rr += 32) out[(size_t)i * k + rr] = -1;
      break;
    }
    pv = bv, pi = bi;
  }
}

extern "C" int b2_similarity_pairs_host(b2_context* ctx, const float* desc, int n, int dim, int num_matched, float min_score,
                                        int32_t* out_partners, float* out_sim) {
  if (!ctx || !desc || !out_partners || n <= 0 || dim <= 0 || num_matched <= 0) return B2_ERR_ARG;
  if (dim % 64) return b2_fail(ctx, B2_ERR_ARG, "descriptor dimension must be a multiple of 64");
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->rt) ctx->rt = new RetrievalState();
  RetrievalState* s = ctx->rt;
  cudaStream_t st = ctx->stream;
  const int k = num_matched < n ? num_matched : n;  // similarity_retriever.py:249
  const size_t ne = (size_t)n * dim;
  B2_CUDA(ctx, s->g.ensure(ne * 4));
  B2_CUDA(ctx, s->gh.ensure(ne * 2));
  B2_CUDA(ctx, s->gl.ensure(ne * 2));
  B2_CUDA(ctx, s->sim.ensure((size_t)n * n * 4));
  B2_CUDA(ctx, s->pairs.ensure((size_t)n * k * 4));
  B2_CUDA(ctx, s->err.ensure(16));
  B2_CUDA(ctx, cudaMemsetAsync(s->err.p, 0, 16, st));
  B2_CUDA(ctx, cudaMemcpyAsync(s->g.p, desc, ne * 4, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, k_split_f32, (unsigned)((ne + 255) / 256), 256, 0, st, s->g.as<float>(), ne, s->gh.as<__half>(), s->gl.as<__half>());
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  TcWeights tw{nullptr, nullptr, nullptr, s->err.as<int>(), !b2_force_simt(ctx)};
  tw.sm_count = ctx->sm_count - ctx->reserve_sms > 0 ? ctx->sm_count - ctx->reserve_sms : 1;
  // The tensor core's fp32 accumulation truncates instead of rounding: over K = 4096 .. 8448 positive products that is a
  // systematic -4e-5 (measured), where the hot path's K <= 512 stays below 1e-6.  So K is walked in chunks of RT_KC whose
  // partial products are added by the epilogue's CUDA-core fp32 add (the residual input, in place).
  for (int kc = 0; kc < dim; kc += RT_KC) {
    LinArgs a;
    a.a1f = s->g.as<float>() + kc, a.a1p = {s->gh.as<__half>() + kc, s->gl.as<__half>() + kc}, a.lda1 = dim, a.K1 = dim - kc < RT_KC ? dim - kc : RT_KC;
    a.bf = a.a1f, a.bp = a.a1p, a.ldb = dim, a.cf = s->sim.as<float>(), a.ldc = n, a.tc_want_f32 = true, a.M = n, a.N = n;
    if (kc) a.resid = s->sim.as<float>(), a.ldr = n;
    int rc = run_linear(ctx, st, tw, &a, 1);
    if (rc) return rc;
  }
  B2_LAUNCH(ctx, k_rt_topk, cdiv(n, 8), 256, 0, st, s->sim.as<float>(), n, k, min_score, s->pairs.as<int>());
  B2_CHECK_LAUNCH(ctx);
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(out_partners, s->pairs.p, (size_t)n * k * 4, cudaMemcpyDeviceToHost, st));
  if (out_sim) B2_CUDA(ctx, cudaMemcpyAsync(out_sim, s->sim.p, (size_t)n * n * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, s->err.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}
