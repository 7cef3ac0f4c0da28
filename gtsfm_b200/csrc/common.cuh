// Shared context / helpers for libgtsfm_b200.so.  sm_90a only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/gtsfm_b200.h"

#define B2_OK 0
#define B2_ERR_CUDA -1
#define B2_ERR_ARG -2
#define B2_ERR_STATE -3
#define B2_ERR_MNN_RATIO -4  // ratio test requested with fewer than 2 descriptors on one side (include/gtsfm_b200.h)
#define B2_SIFT_CAPACITY -5  // b2_sift_detect_host / b2_orb_detect_host: more keypoints than the caller's capacity, *out_n = the count needed

// DevBuf / HostBuf own their allocation: the destructor frees it, so a buffer in a model state is freed when the state is
// deleted and a local one on every return path.  Not copyable (two owners would free twice).
struct DevBuf {  // grow-only device allocation
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

struct HostBuf {  // grow-only pinned host allocation
  void* p = nullptr;
  size_t cap = 0;
  HostBuf() = default;
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  ~HostBuf() { release(); }
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMallocHost(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

struct DebugView {
  const float* p;
  int64_t n;
};

// live per-kernel timing for bench.py's roofline line: CUDA events recorded on the launching stream around every
// launch whose kernel name starts with `name`, plus the algorithmic work (FLOP or bytes) those launches did.
struct ProfState {
  bool on = false;
  std::string name;
  std::vector<cudaEvent_t> ev;
  size_t used = 0;
  double work = 0.0;
  bool match(const char* kernel) const { return on && strncmp(kernel, name.c_str(), name.size()) == 0; }
};

struct SuperPointState;
struct LightGlueState;
struct SuperGlueState;
struct RansacState;
struct LmedsState;
struct RetrievalState;
struct NetVladState;
struct MnnState;
struct SiftState;
struct MegaLocState;
struct D2NetState;
struct JpegState;
struct OrbState;
struct TwoViewState;
struct TwoViewEvalState;
struct ViewGraphState;
struct DataAssocState;
struct MfasState;
struct GlobalBaState;
struct TranslationRecoveryState;

// Device copies of host feature arrays handed to the *_host matcher entry points.  GTSfM matches one image's (keypoints,
// descriptors) against ~20-40 partners, always passing the same host arrays, so re-uploading 5 MB per image per pair is
// most of the plugin path's PCIe traffic.  OPT-IN (b2_set_option("feature_cache", 1) / B2_FEATURE_CACHE=1; the default copies
// on every call like the reference does).  An entry is keyed by (host pointer, size) and validated by a hash over the FULL
// contents, so a freed-and-reused address or an array edited in place anywhere is re-uploaded.
struct FeatCacheEntry {
  const void* host = nullptr;
  size_t bytes = 0;
  uint64_t sig = 0;
  uint64_t stamp = 0;
  DevBuf buf;
};
constexpr int B2_FEAT_CACHE_SLOTS = 96;

struct b2_context {
  int device = 0;
  int sm_count = 132;
  int reserve_sms = 0;  // SMs the persistent kernels of this context leave free (b2_set_option "reserve_sms")
  int lg_batch = 0;     // pairs per LightGlue batch (0 = the library maximum, 8); b2_set_option "lightglue_batch"
  int rs_workspace_mb = 1024;  // RANSAC workspace budget per sub-batch of a batched call; b2_set_option "ransac_workspace_mb"
  int vg_workspace_mb = 1024;  // view-graph filter: segment window of one chunk; b2_set_option "viewgraph_workspace_mb"
  int da_workspace_mb = 256;   // data association: device workspace of one chunk of tracks; "data_assoc_workspace_mb"
  int mf_workspace_mb = 1024;  // 1DSfM's MFAS: device workspace of one chunk of projection directions; "mfas_workspace_mb"
  int ba_workspace_mb = 4096;  // global BA and translation recovery: bound on one call's device workspace; "ba_workspace_mb"
  int force_simt = -1;  // 1: models loaded afterwards run the exact-fp32 SIMT kernels (no tensor cores); -1 = B2_FORCE_SIMT env
  int lg_trace = 0;     // 1: b2_lightglue_match_* record each side's state after every layer (b2_lightglue_trace_get)
  int sg_trace = 0;     // 1: b2_superglue_match_* record each side's state after every layer (b2_superglue_trace_get)
  std::string err;
  std::mutex mu;
  uint64_t launches = 0;
  uint64_t rs_syncs = 0;  // stream synchronisations performed by the RANSAC entry points (b2_ransac_sync_count)
  ProfState prof;
  cudaStream_t stream = nullptr;  // owned; used by *_host entry points
  std::map<std::string, DebugView> debug;
  SuperPointState* sp = nullptr;
  LightGlueState* lg = nullptr;
  SuperGlueState* sg = nullptr;
  RansacState* rs = nullptr;
  LmedsState* lm = nullptr;
  RetrievalState* rt = nullptr;
  NetVladState* nv = nullptr;
  MnnState* mn = nullptr;
  SiftState* sf = nullptr;
  MegaLocState* ml = nullptr;
  D2NetState* d2 = nullptr;
  JpegState* jp = nullptr;
  OrbState* ob = nullptr;
  TwoViewState* tv = nullptr;
  TwoViewEvalState* te = nullptr;
  ViewGraphState* vg = nullptr;
  DataAssocState* da = nullptr;
  MfasState* mf = nullptr;
  GlobalBaState* gb = nullptr;
  TranslationRecoveryState* tr = nullptr;
  // staging shared by the *_host entry points
  DevBuf stage_d[8];
  HostBuf stage_h[4];
  FeatCacheEntry fcache[B2_FEAT_CACHE_SLOTS];
  DevBuf resize_taps;  // b2_image_resize_dev: x then y cubic tap tables of the call in flight
  uint64_t fstamp = 0;
  int fcache_on = -1;          // -1 = read B2_FEATURE_CACHE on first use
  uint64_t h2d_bytes = 0;      // bytes the *_host entry points that track them actually copied
};

inline bool b2_force_simt(const b2_context* ctx) {
  if (ctx->force_simt >= 0) return ctx->force_simt != 0;
  const char* e = getenv("B2_FORCE_SIMT");
  return e && e[0] == '1';
}

inline int b2_fail(b2_context* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  return code;
}

#define B2_CUDA(ctx, expr)                                                                        \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      return b2_fail(ctx, B2_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) +       \
                                           " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
    }                                                                                             \
  } while (0)

// launch bookkeeping: every kernel launch of the library goes through this macro
inline void b2_prof_mark(b2_context* ctx, cudaStream_t st) {
  ProfState& p = ctx->prof;
  if (p.used == p.ev.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    p.ev.push_back(e);
  }
  cudaEventRecord(p.ev[p.used++], st);
}
inline void b2_prof_work(b2_context* ctx, const char* kernel, double work) {
  if (ctx->prof.match(kernel)) ctx->prof.work += work;
}

// `name` is what the profiler matches against: the kernel's own name, or that name followed by a call-site label
// ("k_gemm_ws/lg_self_qkv") so that one call site of a shared kernel can be timed on its own
#define B2_LAUNCH_NAMED(ctx, name, kernel, grid, block, smem, stream, ...) \
  do {                                                                     \
    const bool _prof = (ctx)->prof.match(name);                            \
    if (_prof) b2_prof_mark((ctx), (stream));                              \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);            \
    if (_prof) b2_prof_mark((ctx), (stream));                              \
    (ctx)->launches++;                                                     \
  } while (0)
#define B2_LAUNCH(ctx, kernel, grid, block, smem, stream, ...) B2_LAUNCH_NAMED(ctx, #kernel, kernel, grid, block, smem, stream, __VA_ARGS__)

#define B2_CHECK_LAUNCH(ctx) B2_CUDA(ctx, cudaGetLastError())

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// Test-only entry points (debug.cu, lightglue.cu): a host buffer that the call copies to the device and back whole, so that values outside the written region return as
// they went in, followed on the device by `guard` bytes of 0xFF (NaN in fp32 and fp16) that the kernel must leave alone.
inline int dbg_upload(b2_context* ctx, cudaStream_t st, const void* host, size_t bytes, size_t guard, DevBuf& d) {
  if (bytes == 0 && guard == 0) return B2_OK;
  B2_CUDA(ctx, d.ensure(bytes + guard));
  B2_CUDA(ctx, cudaMemcpyAsync(d.p, host, bytes, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(static_cast<unsigned char*>(d.p) + bytes, 0xFF, guard, st));
  return B2_OK;
}
inline int dbg_download(b2_context* ctx, cudaStream_t st, void* host, size_t bytes, size_t guard, const DevBuf& d, bool& guard_ok) {
  std::vector<unsigned char> g(guard);
  B2_CUDA(ctx, cudaMemcpyAsync(host, d.p, bytes, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(g.data(), static_cast<const unsigned char*>(d.p) + bytes, guard, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (unsigned char v : g) guard_ok = guard_ok && v == 0xFF;
  return B2_OK;
}

// model state lifecycle (defined in the respective .cu files)
void sp_destroy(b2_context* ctx);
void lg_destroy(b2_context* ctx);
void sg_destroy(b2_context* ctx);
void rs_destroy(b2_context* ctx);
void lm_destroy(b2_context* ctx);
void rt_destroy(b2_context* ctx);
void nv_destroy(b2_context* ctx);
void mn_destroy(b2_context* ctx);
void sf_destroy(b2_context* ctx);
void ml_destroy(b2_context* ctx);
void d2_destroy(b2_context* ctx);
void jp_destroy(b2_context* ctx);
void ob_destroy(b2_context* ctx);
void tv_destroy(b2_context* ctx);
void te_destroy(b2_context* ctx);
void vg_destroy(b2_context* ctx);
void da_destroy(b2_context* ctx);
void mf_destroy(b2_context* ctx);
void gb_destroy(b2_context* ctx);
void tr_destroy(b2_context* ctx);

// shared device helpers -------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
