// Context lifecycle and shared C-ABI entry points.
#include <string.h>

#include "common.cuh"

extern "C" int b2_version(void) { return 100; }

extern "C" int b2_create(int device, b2_context** out) {
  if (!out) return B2_ERR_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return B2_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return B2_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) return B2_ERR_STATE;  // sm_90a cubins only: fail loudly on anything else
  if (cudaSetDevice(device) != cudaSuccess) return B2_ERR_CUDA;
  b2_context* ctx = new b2_context();
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return B2_ERR_CUDA;
  }
  *out = ctx;
  return B2_OK;
}

extern "C" void b2_destroy(b2_context* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  sp_destroy(ctx);
  lg_destroy(ctx);
  sg_destroy(ctx);
  rs_destroy(ctx);
  lm_destroy(ctx);
  tv_destroy(ctx);
  te_destroy(ctx);
  vg_destroy(ctx);
  da_destroy(ctx);
  mf_destroy(ctx);
  gb_destroy(ctx);
  tr_destroy(ctx);
  rt_destroy(ctx);
  nv_destroy(ctx);
  mn_destroy(ctx);
  sf_destroy(ctx);
  ml_destroy(ctx);
  d2_destroy(ctx);
  jp_destroy(ctx);
  ob_destroy(ctx);
  for (cudaEvent_t e : ctx->prof.ev) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

extern "C" const char* b2_last_error(const b2_context* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

extern "C" uint64_t b2_launch_count(const b2_context* ctx) { return ctx ? ctx->launches : 0; }
extern "C" int b2_set_option(b2_context* ctx, const char* name, int64_t value) {
  if (!ctx || !name) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!strcmp(name, "reserve_sms")) {
    if (value < 0 || value >= ctx->sm_count) return b2_fail(ctx, B2_ERR_ARG, "reserve_sms out of range");
    ctx->reserve_sms = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "lightglue_batch")) {  // pairs walked in lock-step by b2_lightglue_match_batched_dev (1..8; 0 = maximum)
    if (value < 0 || value > 8) return b2_fail(ctx, B2_ERR_ARG, "lightglue_batch takes 0..8");
    ctx->lg_batch = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "ransac_workspace_mb")) {  // budget of one sub-batch of b2_ransac_verify_batched_dev
    if (value < 1 || value > (1 << 20)) return b2_fail(ctx, B2_ERR_ARG, "ransac_workspace_mb takes 1..1048576");
    ctx->rs_workspace_mb = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "viewgraph_workspace_mb")) {  // segment window of one chunk of b2_viewgraph_cycle_filter_host
    if (value < 1 || value > (1 << 20)) return b2_fail(ctx, B2_ERR_ARG, "viewgraph_workspace_mb takes 1..1048576");
    ctx->vg_workspace_mb = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "data_assoc_workspace_mb")) {  // device workspace of one chunk of b2_triangulate_tracks_host
    if (value < 1 || value > (1 << 20)) return b2_fail(ctx, B2_ERR_ARG, "data_assoc_workspace_mb takes 1..1048576");
    ctx->da_workspace_mb = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "mfas_workspace_mb")) {  // device workspace of one chunk of directions of b2_mfas_outlier_weights_host
    if (value < 1 || value > (1 << 20)) return b2_fail(ctx, B2_ERR_ARG, "mfas_workspace_mb takes 1..1048576");
    ctx->mf_workspace_mb = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "ba_workspace_mb")) {  // bound on the device workspace of one b2_bundle_adjust_host or b2_translation_recovery_host call
    if (value < 1 || value > (1 << 20)) return b2_fail(ctx, B2_ERR_ARG, "ba_workspace_mb takes 1..1048576");
    ctx->ba_workspace_mb = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "force_simt")) {  // takes effect for models whose weights are set AFTER this call
    ctx->force_simt = value ? 1 : 0;
    return B2_OK;
  }
  if (!strcmp(name, "lightglue_trace")) {  // 1: per-layer LightGlue state copied to host memory (a test aid: it synchronises)
    if (value != 0 && value != 1) return b2_fail(ctx, B2_ERR_ARG, "lightglue_trace takes 0 or 1");
    ctx->lg_trace = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "superglue_trace")) {  // 1: per-layer SuperGlue state copied to host memory (a test aid: it synchronises)
    if (value != 0 && value != 1) return b2_fail(ctx, B2_ERR_ARG, "superglue_trace takes 0 or 1");
    ctx->sg_trace = (int)value;
    return B2_OK;
  }
  if (!strcmp(name, "feature_cache")) {  // 0 (default): forget every cached upload and copy on every call; 1: cache
    if (value != 0 && value != 1) return b2_fail(ctx, B2_ERR_ARG, "feature_cache takes 0 or 1");
    ctx->fcache_on = (int)value;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (auto& e : ctx->fcache) {
      e.buf.release();
      e.host = nullptr, e.bytes = 0, e.sig = 0, e.stamp = 0;
    }
    return B2_OK;
  }
  return b2_fail(ctx, B2_ERR_ARG, std::string("unknown option ") + name);
}
extern "C" uint64_t b2_h2d_bytes(const b2_context* ctx) { return ctx ? ctx->h2d_bytes : 0; }

extern "C" int64_t b2_debug_fetch(b2_context* ctx, const char* name, float* host_out, int64_t max_floats) {
  if (!ctx || !name || !host_out) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = ctx->debug.find(name);
  if (it == ctx->debug.end()) return b2_fail(ctx, B2_ERR_ARG, std::string("no debug buffer named ") + name);
  int64_t n = it->second.n < max_floats ? it->second.n : max_floats;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (cudaMemcpy(host_out, it->second.p, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess)
    return b2_fail(ctx, B2_ERR_CUDA, "debug fetch copy failed");
  return n;
}

extern "C" int b2_profile_start(b2_context* ctx, const char* kernel_prefix) {
  if (!ctx || !kernel_prefix) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->prof.on = true;
  ctx->prof.name = kernel_prefix;
  ctx->prof.used = 0;
  ctx->prof.work = 0.0;
  return B2_OK;
}

extern "C" int b2_profile_stop(b2_context* ctx, double* total_ms, uint64_t* launches, double* work) {
  if (!ctx) return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  B2_CUDA(ctx, cudaDeviceSynchronize());
  double ms = 0.0;
  for (size_t i = 0; i + 1 < ctx->prof.used; i += 2) {
    float t = 0.f;
    B2_CUDA(ctx, cudaEventElapsedTime(&t, ctx->prof.ev[i], ctx->prof.ev[i + 1]));
    ms += t;
  }
  if (total_ms) *total_ms = ms;
  if (launches) *launches = ctx->prof.used / 2;
  if (work) *work = ctx->prof.work;
  ctx->prof.on = false;
  ctx->prof.used = 0;
  return B2_OK;
}
