/*
 * gtsfm_b200 — C ABI of the H100-native pairwise deep front-end (SuperPoint -> LightGlue/SuperGlue -> RANSAC).
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point is plain C: opaque handle, raw pointers, sizes,
 * an `int` status (0 = ok, <0 = error; text via b2_last_error).  No torch / C++ types cross it.  `*_dev` entry points
 * take DEVICE pointers plus a CUDA stream (passed as void*, i.e. a cudaStream_t / CUstream; NULL = legacy default
 * stream) so PyTorch tensors go in and out through `tensor.data_ptr()`; the `*_host` entry points take HOST pointers
 * and do the H2D / D2H copies themselves (this is what the per-call GTSfM plugins use, mirroring the reference's
 * `.to(device)` / `.cpu().numpy()` inside each call).
 *
 * Reference interface each group replaces (paths relative to the reference repo):
 *   b2_superpoint_*  : gtsfm/frontend/detector_descriptor/superpoint.py:63-93 (detect_and_describe) and the model
 *                      thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:145-202
 *   b2_lightglue_*   : gtsfm/frontend/matcher/lightglue_matcher.py:43-112 and
 *                      thirdparty/LightGlue/lightglue/lightglue.py:474-629
 *   b2_superglue_*   : gtsfm/frontend/matcher/superglue_matcher.py:47-115 and
 *                      thirdparty/SuperGluePretrainedNetwork/models/superglue.py:226-283
 *   b2_ransac_*      : gtsfm/frontend/verifier/ransac.py:52-111 (cv2.findEssentialMat / findFundamentalMat) and
 *                      gtsfm/utils/verification.py:54-96 (cv2.recoverPose)
 *
 * Threading: a handle serialises its own calls with an internal mutex (Dask workers run one thread per process,
 * gtsfm/runner.py:153-155); use one handle per thread/stream for concurrency.
 */
#ifndef GTSFM_B200_H
#define GTSFM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2_context b2_context;

/* ---- lifecycle -------------------------------------------------------------------------------------------------- */
int b2_version(void);
/* Creates a context on CUDA device `device`.  Fails (returns <0, *out = NULL) when no sm_90 device is present. */
int b2_create(int device, b2_context** out);
void b2_destroy(b2_context* ctx);
const char* b2_last_error(const b2_context* ctx);
/* Number of kernels this library has launched through `ctx` since creation (bench.py's "gpu_launches"). */
uint64_t b2_launch_count(const b2_context* ctx);
/* Host-to-device bytes actually copied so far by the entry points that keep device copies of their host inputs
 * (b2_lightglue_match_host: feature arrays already uploaded for an earlier pair are not sent again). */
uint64_t b2_h2d_bytes(const b2_context* ctx);
/* Tuning knobs.  "reserve_sms" = n: the persistent kernels (attention, GEMM, two-way matcher) launch sm_count - n CTAs, leaving n SMs to
 * kernels of OTHER contexts / streams running concurrently (the batched front-end overlaps pair k's RANSAC with pair
 * k+1's matching; a one-CTA-per-SM kernel that finds an SM busy would otherwise wait for a whole CTA lifetime).
 * "lightglue_batch" = 0..8: pairs per lock-step batch of b2_lightglue_match_batched_dev (0 = 8, the maximum).
 * "force_simt" = 0 | 1: models whose weights are set afterwards run the exact-fp32 SIMT kernels instead of the wgmma
 * split-fp16 ones (the on-device cross-check of the tensor-core path; tests only).
 * "superpoint_graph" = 0 (default) | 1: launch every kernel of the SuperPoint network directly / replay the ~21 launches as one
 * CUDA graph per (image shape, parameters, buffers) key (the path is GPU-bound, not launch-bound).
 * "feature_cache" = 0 | 1: drop every cached device copy of host feature arrays and (0, default) copy on every call like the
 * reference / (1) keep device copies keyed by (host pointer, size) and validated by a hash of the FULL contents, so arrays
 * edited in place are re-sent.  Only pays off for callers that pass the same numpy buffers repeatedly (it does nothing for
 * Dask tasks, which unpickle fresh arrays per call). */
int b2_set_option(b2_context* ctx, const char* name, int64_t value);
/* Live kernel timing for roofline reporting: CUDA events on the launching stream around every launch whose kernel name
 * starts with `kernel_prefix` (e.g. "k_flash_attn"), until b2_profile_stop, which returns the summed device time, the
 * number of such launches and the algorithmic work (FLOP) they performed. */
int b2_profile_start(b2_context* ctx, const char* kernel_prefix);
int b2_profile_stop(b2_context* ctx, double* total_ms, uint64_t* launches, double* work);
/* Copies a named intermediate device buffer of the last call to host (tests only). Returns #floats written or <0. */
int64_t b2_debug_fetch(b2_context* ctx, const char* name, float* host_out, int64_t max_floats);

/* Test-only: C[M,N] = A[M,K] * B[N,K]^T (+ bias) on HOST fp32 buffers.  mode 0 = SIMT fp32 kernel, 1 = wgmma split-fp16
 * kernel with fp32 B converted in-kernel, 2 = wgmma split-fp16 kernel with pre-split fp16 B.  K must be a multiple of 64. */
int b2_debug_gemm_host(b2_context* ctx, int mode, const float* A, const float* B, const float* bias, float* C, int M, int N,
                       int K);
/* Test-only: one batched launch of the wgmma flash attention on HOST fp32 buffers.  Problem z (0 <= z < np <= 16) has
 * nq[z] queries, nk[z] keys and `heads` heads of 64: q as [heads][nq[z]][64], k and v as [heads][nk[z]][64] (head-major),
 * each concatenated over z; o receives softmax(scale * q k^T) v as [nq[z]][64 * heads] per problem, concatenated over z.
 * The operands are split into fp16 hi / lo planes on the device; single = 1 runs the fp16 variant (hi planes only). */
int b2_debug_attention_host(b2_context* ctx, int np, const int* nq, const int* nk, int heads, float scale, int single,
                            const float* q, const float* k, const float* v, float* o);

/* ---- SuperPoint -------------------------------------------------------------------------------------------------- */
/* `blob`: the 24 state-dict tensors in reference order (conv1a.weight, conv1a.bias, conv1b.weight, ... convDb.bias;
 * SURVEY.md Appendix A), OIHW fp32, concatenated.  n_floats must equal 1300865. */
int b2_superpoint_set_weights(b2_context* ctx, const float* host_blob, size_t n_floats);

/* Detect stage on a device image.  `image`: uint8, `channels` in {1,3,4} interleaved (RGB/RGBA are converted with
 * cv2's fixed-point COLOR_RGB2GRAY), row pitch in bytes.  Runs encoder + both heads + NMS + threshold + border
 * removal + ordered compaction.  Keypoints come out in row-major (y, then x) order like torch.nonzero.
 * out_xy: [cap][2] float (x, y); out_score: [cap] float; *out_n (HOST int) = number found (may exceed cap: only the
 * first cap are written).  *out_map_token (HOST, may be NULL) identifies the dense descriptor map this call left in the
 * context.  Synchronises `stream` before returning (the count is data dependent). */
int b2_superpoint_detect_dev(b2_context* ctx, const uint8_t* image, int height, int width, int channels, size_t pitch,
                             float keypoint_threshold, int nms_radius, int border, float* out_xy, float* out_score,
                             int cap, int* out_n, uint64_t* out_map_token, void* stream);
/* Describe stage: bilinear-samples the dense descriptor map identified by `map_token` at `n` (x, y) positions and
 * L2-normalises.  Fails with a "stale feature-map token" error if another detect has run on the context since the token
 * was issued (two images interleaved on one handle can therefore never get each other's descriptors).
 * out_desc: [n][256] float row-major.  Asynchronous on `stream`. */
int b2_superpoint_describe_dev(b2_context* ctx, uint64_t map_token, const float* xy, int n, float* out_desc, void* stream);
/* Fused, self-contained extraction for the batched path: detect -> device top-k (the `max_keypoints` largest responses,
 * ties by lower index, row-major order kept) -> describe, under one lock, one host synchronisation.  out_xy [max_keypoints][2],
 * out_score [max_keypoints], out_desc [max_keypoints][256] are DEVICE buffers; *out_n (HOST) = keypoints written. */
int b2_superpoint_extract_dev(b2_context* ctx, const uint8_t* image, int height, int width, int channels, size_t pitch,
                              float keypoint_threshold, int nms_radius, int border, int max_keypoints, float* out_xy,
                              float* out_score, float* out_desc, int* out_n, void* stream);
/* The same with NO host synchronisation, for callers that keep many images in flight: `out_n_pinned` (page-locked host int,
 * one per image in flight) receives the keypoint count when `stream` gets there; the library's work buffers are reused in
 * stream order.  Call b2_superpoint_finish_dev (stream synchronisation + tensor-core pipeline fault check) before reading the
 * counts or the outputs on the host. */
int b2_superpoint_extract_async_dev(b2_context* ctx, const uint8_t* image, int height, int width, int channels, size_t pitch,
                                    float threshold, int nms_radius, int border, int max_keypoints, float* out_xy,
                                    float* out_score, float* out_desc, int* out_n_pinned, void* stream);
int b2_superpoint_finish_dev(b2_context* ctx, void* stream);
/* Device top-k by score (k largest, ties broken by lower index), result kept in row-major order; writes the selected
 * indices (int32, ascending) and returns count in *out_k (HOST).  For the batched path; the per-call plugin uses the
 * reference's host argpartition to keep its index order. */
int b2_topk_indices_dev(b2_context* ctx, const float* scores, int n, int k, int32_t* out_idx, int* out_k, void* stream);

/* Host-pointer variants (H2D / D2H inside). */
int b2_superpoint_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels,
                              float keypoint_threshold, int nms_radius, int border, float* out_xy, float* out_score,
                              int cap, int* out_n, uint64_t* out_map_token);
int b2_superpoint_describe_host(b2_context* ctx, uint64_t map_token, const float* xy, int n, float* out_desc);

/* ---- image ingest (SURVEY.md section 8f rank 2) ------------------------------------------------------------------- */
/* The loader's cubic resize (gtsfm/utils/images.py:102-129: cv2.resize(INTER_CUBIC) to the size picked by
 * get_downsampling_factor_per_axis, :150-220) on the device: src / dst are DEVICE uint8 images, `channels` interleaved,
 * src row pitch in bytes, dst dense.  OpenCV's 11-bit fixed-point arithmetic as restated in oracle/images_ref.py.
 * Asynchronous on `stream`; feed dst straight into b2_superpoint_detect_dev / b2_superpoint_extract_dev. */
int b2_image_resize_dev(b2_context* ctx, const uint8_t* src, int height, int width, int channels, size_t pitch, uint8_t* dst,
                        int new_height, int new_width, void* stream);

/* ---- LightGlue --------------------------------------------------------------------------------------------------- */
/* `blob`: packed fp32 tensors in the order documented in gtsfm_b200/weights.py::LIGHTGLUE_ORDER (nn.Linear layout
 * (out,in) row-major as in the checkpoint).  n_floats must equal 11851601 (the 251 parameter tensors; the
 * confidence_thresholds buffer is recomputed). */
int b2_lightglue_set_weights(b2_context* ctx, const float* host_blob, size_t n_floats);

typedef struct b2_lightglue_params {
  /* doubles on purpose: the reference holds these as Python floats and rounds the DERIVED value to float32 at the
   * comparison (e.g. scores > float32(1 - 0.99)), which a float32 field could not reproduce bit-exactly. */
  double depth_confidence; /* 0.95; <= 0 disables early exit   (lightglue.py:330)            */
  double width_confidence; /* 0.99; <= 0 disables pruning      (lightglue.py:331)            */
  double filter_threshold; /* 0.1                              (lightglue.py:332)            */
  int prune_min_kpts;      /* -1 = reference CPU semantics (prune at every layer); 1536 = its CUDA+flash value */
  int fp16_attention;      /* 0 (default): fp32-equivalent attention, what the reference's CPU front-end computes and the fixtures
                            * pin.  1: the reference's CUDA numerics (lightglue.py:116-121: q, k, v cast to half, fp16 flash SDPA,
                            * half result cast back) - one tensor-core product instead of three; descriptors then agree with the
                            * fp32 path to ~1e-3 and match indices are no longer guaranteed bit-identical to the CPU reference. */
} b2_lightglue_params;

/* kp: [n][2] float (x, y) pixels; desc: [n][256] float.  out_matches: [min(n0,n1)][2] int64 rows (idx0, idx1)
 * ascending in idx0; out_scores: [min(n0,n1)] float (exp of the log assignment) or NULL.  *out_k, *out_stop_layer are
 * HOST ints (stop layer is 1-based like the reference's "stop").  Synchronises `stream`. */
int b2_lightglue_match_dev(b2_context* ctx, const float* kp0, const float* desc0, int n0, const float* kp1,
                           const float* desc1, int n1, const b2_lightglue_params* params, int64_t* out_matches,
                           float* out_scores, int* out_k, int* out_stop_layer, void* stream);
int b2_lightglue_match_host(b2_context* ctx, const float* kp0, const float* desc0, int n0, const float* kp1,
                            const float* desc1, int n1, const b2_lightglue_params* params, int64_t* out_matches,
                            float* out_scores, int* out_k, int* out_stop_layer);

/* Batched variant (SURVEY.md 8b "_batched variants taking arrays of pairs"; the seam is
 * gtsfm/frontend/correspondence_generator/det_desc_correspondence_generator.py:65-85, one matcher task per pair).  Up to 8
 * pairs at a time are walked in lock-step: every linear layer, attention call and pruning step is ONE launch over all
 * images of the batch, the per-layer early-exit / pruning counters of all pairs come back in one 128-byte read, pairs
 * that stop early drop out of the later launches.  Results are identical to n_pairs calls of b2_lightglue_match_dev.
 * All pointers inside `pairs` are DEVICE pointers; out_k / out_stop_layer are written on the HOST struct. */
typedef struct b2_lightglue_pair {
  const float* kp0;   /* [n0][2] (x, y) pixels */
  const float* desc0; /* [n0][256] */
  int n0;
  const float* kp1;
  const float* desc1;
  int n1;
  int64_t* out_matches; /* [min(n0, n1)][2] rows (idx0, idx1) ascending in idx0 */
  float* out_scores;    /* [min(n0, n1)] or NULL */
  int out_k;            /* written: number of matches */
  int out_stop_layer;   /* written: 1-based stopping layer */
} b2_lightglue_pair;
int b2_lightglue_match_batched_dev(b2_context* ctx, b2_lightglue_pair* pairs, int n_pairs, const b2_lightglue_params* params,
                                   void* stream);

/* ---- SuperGlue --------------------------------------------------------------------------------------------------- */
/* `blob`: packed fp32 tensors in gtsfm_b200/weights.py::SUPERGLUE_ORDER with eval-mode BatchNorm already folded
 * into the preceding Conv1d by the host loader. */
int b2_superglue_set_weights(b2_context* ctx, const float* host_blob, size_t n_floats);
/* score: [n] keypoint responses; (h, w): image sizes used for keypoint normalisation (superglue.py:63-70).
 * out_matches: [min(n0,n1)][2] uint32 rows (i, matches0[i]) ascending in i. */
int b2_superglue_match_dev(b2_context* ctx, const float* kp0, const float* score0, const float* desc0, int n0, int h0,
                           int w0, const float* kp1, const float* score1, const float* desc1, int n1, int h1, int w1,
                           int sinkhorn_iters, float match_threshold, uint32_t* out_matches, float* out_scores,
                           int* out_k, void* stream);
int b2_superglue_match_host(b2_context* ctx, const float* kp0, const float* score0, const float* desc0, int n0, int h0,
                            int w0, const float* kp1, const float* score1, const float* desc1, int n1, int h1, int w1,
                            int sinkhorn_iters, float match_threshold, uint32_t* out_matches, float* out_scores,
                            int* out_k);

/* ---- RANSAC verifier --------------------------------------------------------------------------------------------- */
typedef struct b2_ransac_params {
  double threshold;   /* inlier threshold: max point-to-epipolar-line style distance (same unit as the points):      */
                      /* thr_px / fx for E on normalised points, thr_px for F on pixels (ransac.py:79,107)           */
  double confidence;  /* 0.999999 (ransac.py:22)                                                                     */
  int max_iters;      /* hypothesis budget (cv2 maxIters): E 1000 (cv2 default, ransac.py:74-81), clamped to 65 536; F: the       */
                      /* reference passes 10^6, the library clamps to 262 144 and stops earlier through the standard        */
                      /* confidence bound.  E only: when the bound says max_iters (<= 4096) samples were NOT enough for      */
                      /* `confidence`, up to 4 x max_iters further samples are drawn (decided on the device).                */
  uint64_t seed;      /* fixed per call => run-to-run identical results (repro test, SURVEY.md Appendix B)           */
} b2_ransac_params;

/* x1, x2: [k][2] double matched points (normalised coordinates for E, pixels for F).
 * out_model: 9 doubles row-major (E or F, x2^T M x1 = 0); out_mask: [k] uint8; *out_num_inliers HOST int.
 * For E also recovers the pose by the cheirality vote (cv2.recoverPose semantics): out_R 9 doubles row-major (i2Ri1),
 * out_t 3 doubles (unit i2ti1); may be NULL.  Returns 1 when no model could be estimated (mask all zero). */
int b2_ransac_essential_host(b2_context* ctx, const double* x1, const double* x2, int k, const b2_ransac_params* params,
                             double* out_model, uint8_t* out_mask, int* out_num_inliers, double* out_R, double* out_t);
int b2_ransac_fundamental_host(b2_context* ctx, const double* x1, const double* x2, int k,
                               const b2_ransac_params* params, double* out_model, uint8_t* out_mask,
                               int* out_num_inliers);
/* Device-resident variant for the batched path: kp1 / kp2 are DEVICE [n][2] float pixel coordinates, matches DEVICE
 * [k][2] int64 rows; cal1 / cal2 are HOST {f, u0, v0} of distortion-free pinhole cameras (Cal3Bundler with k1 = k2 = 0,
 * gtsfm/utils/features.py:41-51).  The threshold in `params` is in calibrated units (thr_px / max(f)).  out_mask_dev is a
 * DEVICE [k] uint8 buffer (or NULL); the small outputs are HOST.  Synchronises `stream`. */
int b2_ransac_essential_dev(b2_context* ctx, const float* kp1, const float* kp2, const int64_t* matches, int k,
                            const double* cal1, const double* cal2, const b2_ransac_params* params, double* out_model,
                            uint8_t* out_mask_dev, int* out_num_inliers, double* out_R, double* out_t, void* stream);
/* cv2.recoverPose restated: decompose E, pick (R, t) with most points in front of both cameras. */
int b2_recover_pose_host(b2_context* ctx, const double* E, const double* x1, const double* x2, int k, double* out_R,
                         double* out_t, int* out_num_good);

/* ---- NetVLAD global descriptor (SURVEY.md section 8f rank 4; gtsfm/frontend/global_descriptor/netvlad_global_descriptor.py:53-71,
 * thirdparty/hloc/netvlad.py:52-75,163-193) ------------------------------------------------------------------------------------- */
/* blob = 13 x (conv weight OIHW, bias) of VGG16 features[:-2], score_proj [64][512], centers [512][64], whitening weight
 * [4096][32768] and bias [4096], mean [3] (the checkpoint's averageImage): b2_netvlad_blob_floats() floats. */
size_t b2_netvlad_blob_floats(void);
int b2_netvlad_set_weights(b2_context* ctx, const float* blob, size_t n_floats);
/* images: [B][3][H][W] fp32 in [0, 1] (what the reference's batch transform produces), H, W >= 16; out: [B][4096] unit-norm
 * descriptors.  _dev: device pointers, synchronises `stream` before returning; _host: host pointers. */
int b2_netvlad_describe_dev(b2_context* ctx, const float* images, int batch, int height, int width, float* out, void* stream);
int b2_netvlad_describe_host(b2_context* ctx, const float* images, int batch, int height, int width, float* out);

/* ---- MegaLoc global descriptor (gtsfm/frontend/global_descriptor/megaloc_global_descriptor.py:18-77,
 * thirdparty/megaloc/megaloc.py:25-257: DINOv2 ViT-B/14 + SALAD + Linear(16640 -> 8448)) ------------------------------------ */
/* blob = cls_token [768], pos_embed [1370][768], patch_embed.proj weight [768][3][14][14] and bias; 12 x (norm1 weight, bias,
 * attn.qkv weight [2304][768], bias, attn.proj weight [768][768], bias, ls1.gamma, norm2 weight, bias, mlp.fc1 weight
 * [3072][768], bias, mlp.fc2 weight [768][3072], bias, ls2.gamma); norm weight, bias; SALAD cluster_features.0 weight
 * [512][768], bias, .3 weight [256][512], bias; score.0 weight [512][768], bias, .3 weight [64][512], bias; token_features.0
 * weight [512][768], bias, .2 weight [256][512], bias; dust_bin; aggregator.linear weight [8448][16640], bias:
 * b2_megaloc_blob_floats() floats (the checkpoint's tensors without mask_token, in gtsfm_b200.weights.MEGALOC_ORDER).
 * MegaLoc runs on the tensor-core path only: with the "force_simt" option set every b2_megaloc_* call returns -3. */
size_t b2_megaloc_blob_floats(void);
int b2_megaloc_set_weights(b2_context* ctx, const float* blob, size_t n_floats);
/* images: DEVICE [B][3][H][W] fp32, normalised as the plugin's batch transform does ((x / 255 - mean) / std, ImageNet); H and W
 * multiples of 14 with more than 64 patches (H / 14) (W / 14), otherwise -2.  out: DEVICE [B][8448] unit-norm descriptors.
 * Any B: the backbone runs in chunks of 16 images, the final Linear over all B at once.  Synchronises `stream`. */
int b2_megaloc_describe_dev(b2_context* ctx, const float* images, int batch, int height, int width, float* out, void* stream);
int b2_megaloc_describe_host(b2_context* ctx, const float* images, int batch, int height, int width, float* out);
/* The plugin's whole preprocessing on the device: images = HOST array of n DEVICE pointers to uint8 H x W x 3 (RGB) images of
 * one shape and row pitch (bytes), e.g. the frames already uploaded for b2_sift_detect_batched_dev.  torchvision's
 * Resize((322, 322), antialias=True) on uint8 (torch's integer path, bit for bit), then / 255 and the ImageNet normalisation,
 * then the network.  out: DEVICE [n][8448].  Synchronises `stream`. */
int b2_megaloc_describe_u8_dev(b2_context* ctx, const uint8_t* const* images, int n, int height, int width, size_t pitch, float* out,
                               void* stream);
/* The resize alone: out = DEVICE uint8 [n][3][322][322] (what the plugin's resize transform returns).  Synchronises `stream`. */
int b2_megaloc_resize_u8_dev(b2_context* ctx, const uint8_t* const* images, int n, int height, int width, size_t pitch, uint8_t* out,
                             void* stream);

/* ---- retrieval front (SURVEY.md section 8f rank 4) ---------------------------------------------------------------- */
/* gtsfm/retriever/similarity_retriever.py:86-260: sim = G G^T of the global image descriptors (desc: HOST [n][dim] fp32,
 * dim a multiple of 64), then per query image i its `num_matched` best partners among j > i with sim >= min_score, best
 * first.  out_partners: HOST [n][min(num_matched, n)] int32, -1 = no (further) partner; out_sim: HOST [n][n] or NULL.
 * (Descriptors: b2_netvlad_describe_* above, or any other unit-norm global descriptor.) */
int b2_similarity_pairs_host(b2_context* ctx, const float* desc, int n, int dim, int num_matched, float min_score,
                             int32_t* out_partners, float* out_sim);

/* ---- two-way (mutual nearest neighbour) descriptor matcher (gtsfm/frontend/matcher/twoway_matcher.py) -------------------- */
/* cv2.BFMatcher(NORM_L2) in both directions (knnMatch k = 2 with the ratio test `d1 <= ratio * d2` compared in double, or
 * match without it), mutual check, rows ordered by (0 -> 1 distance, i0).  Descriptors are [n][dim] row-major, dtype 0 =
 * float32, 1 = uint8; 1 <= dim <= 32768, n <= 32768 per image.  uint8 input, and float32 input whose values are all integers
 * in [0, 255] with dim <= 258, is matched in exact integer arithmetic (|a|^2 + |b|^2 - 2 a.b in int32, then sqrtf).  cv2 sums
 * (a - b)^2 in float for both types, exactly while dim * 255^2 < 2^24, so for dim <= 258 (cv2 SIFT, ORB, BRISK) indices,
 * order and distances equal cv2's bit for bit; for uint8 with a larger dim cv2's distances may differ in the last bits.
 * Other float32 input uses split-fp16 products; d^2 = |a|^2 + |b|^2 - 2 a.b cancels for near-duplicate rows, so distances and
 * the resolution of near-ties can differ from cv2's.  The choice is made per pair from the data.  ratio < 0: no ratio test
 * (the reference's None).  With a ratio test, a pair with a non-empty side of fewer than 2 rows fails with -4 (cv2's
 * knnMatch returns one neighbour there).
 * Nothing proportional to n0 * n1 is allocated. */
typedef struct b2_mnn_pair {
  const void* desc0; /* DEVICE [n0][dim] */
  int n0;
  const void* desc1; /* DEVICE [n1][dim] */
  int n1;
  int64_t* out_matches; /* DEVICE [min(n0, n1)][2] rows (i0, i1) */
  float* out_dist;      /* DEVICE [min(n0, n1)] cv2 DMatch.distance of the 0 -> 1 match, or NULL */
  int out_k;            /* written on the HOST struct: number of matches */
} b2_mnn_pair;
/* All pairs of a batch share dim and dtype; one synchronisation of `stream` at the end. */
int b2_mnn_match_batched_dev(b2_context* ctx, b2_mnn_pair* pairs, int n_pairs, int dim, int dtype, double ratio, void* stream);
/* HOST pointers (float32 integer-valued input is sent as uint8); out_matches [min(n0,n1)][2], out_dist may be NULL. */
int b2_mnn_match_host(b2_context* ctx, const void* desc0, int n0, const void* desc1, int n1, int dim, int dtype, double ratio,
                      int64_t* out_matches, float* out_dist, int* out_k);

/* ---- SIFT detector-descriptor (gtsfm/frontend/detector_descriptor/sift.py) --------------------------------------------------- */
/* cv2.SIFT_create() with its defaults restated: 3 layers per octave, contrast threshold 0.04, edge threshold 10, sigma 1.6, the
 * image doubled first (octave -1).  Images are uint8 H x W x {1, 3, 4} interleaved (RGB / RGBA go through cv2's fixed-point
 * COLOR_RGB2GRAY); H x W <= 2^24 and each side <= 16384, larger input fails with -2.  Keypoints come in cv2's order (x, y
 * ascending, size descending, angle, response descending, octave descending), consecutive duplicates in (x, y, size, angle)
 * dropped, then the mask applied as cv2 does (kept where mask[(int)(y + 0.5)][(int)(x + 0.5)] != 0).  Descriptors are 128
 * uint8 values per keypoint (cv2's float descriptors hold the same integers).  Results do not depend on the batch or the run.
 * Workspace: about 151 H W bytes per image of a batch (the Gaussian pyramid is 128 H W). */
typedef struct b2_sift_keypoint { /* the fields of cv2.KeyPoint */
  float x, y, size, angle, response;
  int32_t octave;
} b2_sift_keypoint;
typedef struct b2_sift_image {
  const uint8_t* image;             /* DEVICE image, row pitch as passed to the call */
  const uint8_t* mask;              /* DEVICE H x W uint8, dense, or NULL */
  int max_keypoints;                /* >= 1: the max_keypoints largest responses (ties to the lower index), cv2's order kept */
  b2_sift_keypoint* out_keypoints;  /* DEVICE [max_keypoints] */
  uint8_t* out_desc;                /* DEVICE [max_keypoints][128] */
  int out_n;                        /* written on the HOST struct: keypoints written */
  int out_total;                    /* written on the HOST struct: keypoints after the mask, before the top-k */
} b2_sift_image;
/* Up to 64 same-shape images: every pyramid and extrema stage is one launch over the batch, counts stay on the device, and
 * `stream` is synchronised once at the end. */
int b2_sift_detect_batched_dev(b2_context* ctx, b2_sift_image* images, int n_images, int height, int width, int channels,
                               size_t pitch, void* stream);
/* HOST pointers, dense image, optional mask: every keypoint (no top-k).  When there are more than `capacity` keypoints nothing
 * is written and the call returns -5 with *out_n = the number needed; otherwise *out_n = the number written. */
int b2_sift_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels, const uint8_t* mask,
                        b2_sift_keypoint* out_keypoints, uint8_t* out_desc, int capacity, int* out_n);

/* ---- D2-Net detector-descriptor (gtsfm/frontend/detector_descriptor/d2net.py, thirdparty/d2net/lib/{model_test,pyramid,utils}.py)
 * Single scale, use_relu, 'torch' preprocessing: VGG16 conv1_1 .. conv3_3, AvgPool2d(2, stride=1), conv4_1 .. conv4_3 with
 * dilation 2 -> dense map (H/4 - 1) x (W/4 - 1) x 512; HardDetectionModule (edge threshold 5), HandcraftedLocalizationModule,
 * bilinear descriptors, F.normalize.  Keypoints come ordered by score descending, ties in the reference's torch.nonzero order
 * (channel, row, column); the first max_keypoints are kept.  Images are uint8 H x W x {1, 3} interleaved (gray is used for all three
 * channels, as the reference repeats it); 8 <= H, W, max(H, W) <= 1600 and H + W <= 2800 (the reference resizes larger
 * images, which its scipy no longer can), otherwise -2.  With the "force_simt" option set every b2_d2net_* call that uses the
 * GPU returns -3. */
/* Floats of the weight blob: the 20 tensors dense_feature_extraction.model.{0,2,5,7,10,12,14,17,19,21}.{weight,bias} of the
 * d2_tf.pth checkpoint, in that order, each in its checkpoint layout (gtsfm_b200.weights.D2NET_ORDER). */
size_t b2_d2net_blob_floats(void);
/* HOST [3][256]: the float32 value the reference's preprocess_image('torch') gives byte u of channel c, at [c][u]. */
int b2_d2net_norm_table(float* out);
int b2_d2net_set_weights(b2_context* ctx, const float* blob, size_t n_floats);
typedef struct b2_d2net_image {
  const uint8_t* image; /* DEVICE image, row pitch as passed to the call */
  int max_keypoints;    /* >= 0: keypoints kept (capacity of the outputs) */
  float* out_xy;        /* DEVICE [max_keypoints][2] (x, y) in input pixels */
  float* out_scores;    /* DEVICE [max_keypoints] */
  float* out_desc;      /* DEVICE [max_keypoints][512], unit length */
  int out_n;            /* written on the HOST struct: keypoints written */
  int out_total;        /* written on the HOST struct: keypoints before the top-k */
} b2_d2net_image;
/* Up to 64 same-shape images, one after another through the network; counts stay on the device and `stream` is synchronised once. */
int b2_d2net_detect_batched_dev(b2_context* ctx, b2_d2net_image* images, int n_images, int height, int width, int channels,
                                size_t pitch, void* stream);
/* HOST pointers, dense image: the max_keypoints best keypoints, ordered; out_total (may be NULL) = the count before the top-k. */
int b2_d2net_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels, int max_keypoints,
                         float* out_xy, float* out_scores, float* out_desc, int* out_n, int* out_total);
/* Test-only entry points (tests/test_d2net_kernels_gpu.py), HOST pointers:
 *  b2_debug_conv_ps_host: one k_conv_ps<dilation> layer (dilation 1 or 2, padding = dilation, Cin and Cout multiples of 64) on fp32 NHWC
 *    [H][W][Cin] with OIHW weights [Cout][Cin][3][3] and bias, optional ReLU -> fp32 NHWC [H][W][Cout];
 *  b2_debug_d2net_avgpool_host: the AvgPool2d(2, stride=1) kernel on fp32 NHWC [H][W][256] -> [H - 1][W - 1][256] (hi + lo planes);
 *  b2_debug_d2net_rank_host: the keypoint ordering on n candidates (score, c, i, j) -> order[r] = candidate of rank r < min(n, max_k). */
int b2_debug_conv_ps_host(b2_context* ctx, int dilation, const float* in, int height, int width, int cin, int cout, const float* weight,
                          const float* bias, int relu, float* out);
int b2_debug_d2net_avgpool_host(b2_context* ctx, const float* in, int height, int width, float* out);
int b2_debug_d2net_rank_host(b2_context* ctx, const float* scores, const int* cij, int n, int max_k, int* order);

#ifdef __cplusplus
}
#endif
#endif /* GTSFM_B200_H */
