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
 * "lightglue_trace" = 0 | 1: (1) record LightGlue's per-layer state in host memory (b2_lightglue_trace_get; tests only).
 * "superglue_trace" = 0 | 1: (1) record SuperGlue's per-layer state in host memory (b2_superglue_trace_get; tests only).
 * "ransac_workspace_mb" = 1..: device workspace one sub-batch of b2_ransac_verify_batched_dev may use (default 1024); a call with
 * more problems than fit is cut into consecutive sub-batches, which changes no result.
 * "viewgraph_workspace_mb" = 1..: the segment window of one chunk of b2_viewgraph_cycle_filter_host's MEDIAN (default 1024);
 * a graph with more segment entries than fit is processed in several chunks, which changes no result.
 * "data_assoc_workspace_mb" = 1..: device workspace one chunk of b2_triangulate_tracks_host may use (default 256); a call
 * with more tracks than fit is cut into consecutive chunks of whole tracks, which changes no result.
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

/* Test-only: one call of the library's shared linear (the GEMM every network runs on) over np <= 16 problems on HOST fp32
 * buffers, C_z = ((([A1_z | A2_z] B_z^T) + bias) * scale, then ReLU or exact GELU) + resid_z.  path 1 runs the wgmma split-fp16
 * kernel (K1, K2 multiples of 64), path 0 the exact-fp32 SIMT kernel (K1, K2 multiples of 16, lda1, lda2, ldb multiples of
 * 4; fp32 output only, no GELU); other inputs return -2.  A, B are split into fp16 hi / lo * 2^11 planes on the device.  Device
 * copies have the host pitches.  Each output buffer (c: m ldc floats, or ceil(n / 64) m 64 when head_major; planes: m ldch
 * halves, or ceil(n / 64) m 64) is copied to the device before the launch and back whole after it, so values outside the
 * written region return unchanged unless the kernel overwrote them; on the device each output is followed by 128 rows of
 * 0xFF bytes, and the call returns -3 when the kernel wrote any of them (or its pipeline timed out).  Problems with m = 0 or
 * n = 0 are skipped.  ldr and ldch are one per launch: problems that have them must agree. */
typedef struct b2_linear_problem {
  const float* a1; int lda1;                 /* [m][lda1], the first k1 columns used */
  const float* a2; int lda2;                 /* [m][lda2], the first k2 columns used (k2 > 0) */
  const float* b;  int ldb;                  /* [n][ldb]; problem 0's is shared unless per_problem_b */
  const float* resid; int ldr;               /* [m][ldr] or NULL */
  float* c; int ldc;                         /* fp32 output or NULL (wgmma path) */
  uint16_t* c_hi; uint16_t* c_lo; int ldch;  /* fp16 plane outputs (bits) or NULL (wgmma path) */
  int m, n;
} b2_linear_problem;
typedef struct b2_linear_launch {
  int path;             /* 0 = SIMT k_gemm_nt, 1 = wgmma k_gemm_ws */
  int k1, k2, per_problem_b;
  const float* bias;    /* [max n] or NULL */
  float scale;          /* 1 for none */
  int relu, gelu, head_major, lo_unscaled;
  int resid_in_place;   /* the device C is the residual (c's rows hold it on entry); resid must be NULL */
} b2_linear_launch;
int b2_debug_linear_host(b2_context* ctx, const b2_linear_launch* launch, const b2_linear_problem* problems, int np);
/* Test-only: one 3x3 convolution layer (padding = dilation) on HOST buffers, out = act(maxpool(conv(in, weight) + bias)) with the
 * 2x2/2 max-pool (floor) optional and act = ReLU or identity.  NHWC input [height][width][cin], OIHW weight [cout][cin][3][3],
 * bias [cout]; outputs [oh][ow][cout], (oh, ow) = (height / 2, width / 2) with pool, else (height, width).
 *   path 1: k_conv_ps<dilation> through the launch helper SuperPoint's, NetVLAD's and D2-Net's layers share, on input and
 *     weights split into fp16 hi / lo * 2^11 planes on the device; fp32 and / or plane outputs.  Cin or cout not a multiple of
 *     64, or a dilation other than 1 or 2, returns -2 from that helper.  ctas = 0 launches the grid the networks launch,
 *     otherwise exactly ctas CTAs, a multiple of cout / 64 (else -2).
 *   path 0: the exact-fp32 SIMT k_conv3x3<pool> (SuperPoint under force_simt): relu = 1, dilation 1, cin a multiple of 8, cout
 *     of 64, an fp32 output only and ctas = 0, otherwise -2.
 * No output, a pool with height or width below 2, or a size below 1 return -2.  Each output is copied to the device and back
 * whole, so a value the kernel does not write returns as it went in; on the device it is followed by 0xFF guard bytes (the
 * planes: one buffer, lo after hi, then the guard), and the call returns -3 when the kernel wrote any of them (or its pipeline
 * timed out). */
typedef struct b2_conv_layer {
  int path;                             /* 1 = wgmma k_conv_ps, 0 = SIMT k_conv3x3 */
  int dilation, pool, relu, ctas;
  int height, width, cin, cout;
  const float* in;                      /* [height][width][cin] */
  const float* weight;                  /* [cout][cin][3][3] */
  const float* bias;                    /* [cout] */
  float* out;                           /* [oh][ow][cout] or NULL */
  uint16_t* out_hi; uint16_t* out_lo;   /* fp16 bits [oh][ow][cout] each, or NULL (path 1) */
} b2_conv_layer;
int b2_debug_conv_host(b2_context* ctx, const b2_conv_layer* layer);
/* Test-only: the wgmma GEMM's column-segment epilogue on HOST fp32 buffers.  A [M][K], B [256 nseg][K], bias [256 nseg]
 * (1 <= nseg <= 3, K a multiple of 64); output columns 256 s .. 256 s + 255 go to segment s of out_hi / out_lo, each
 * [nseg][4][M][64] fp16 bits (head-major, unscaled lo).  Segments with a rot_mask bit get rotary from cs / sn [M][32].
 * separate = 1 runs each segment as a launch of its own instead (rot_mask must then be 0). */
int b2_debug_gemm_segments_host(b2_context* ctx, const float* A, const float* B, const float* bias, int M, int K, int nseg,
                                int rot_mask, const float* cs, const float* sn, int separate, uint16_t* out_hi,
                                uint16_t* out_lo);
/* Test-only: one batched launch of the wgmma flash attention on HOST fp32 buffers.  Problem z (0 <= z < np <= 16) has
 * nq[z] queries, nk[z] keys and `heads` heads of 64: q as [heads][nq[z]][64], k and v as [heads][nk[z]][64] (head-major),
 * each concatenated over z; o receives softmax(scale * q k^T) v as [nq[z]][64 * heads] per problem, concatenated over z.
 * The operands are split into fp16 hi / lo planes on the device; single = 1 runs the fp16 variant (hi planes only). */
int b2_debug_attention_host(b2_context* ctx, int np, const int* nq, const int* nk, int heads, float scale, int single,
                            const float* q, const float* k, const float* v, float* o);
/* Test-only: the matchers' assignment step on HOST buffers, through the same dispatch the matchers use.  path 0 = what the
 * matcher picks, 1 = the persistent cooperative kernel (an error when N is above its limit), 2 = the multi-launch kernels;
 * ctas = the persistent kernel's CTA count (1 .. SM count; 0 = the matcher's).  *out_path receives the path that ran (1 or
 * 2), out_matches / out_scores the filtered match list (M rows of room), *out_k its length.
 *  SuperGlue: Z [M][N] scores, bin score alpha, `iters` Sinkhorn iterations -> duals u [M + 1], v [N + 1]; uint32 rows (i, j).
 *  LightGlue: sim [M][N], matchability logits z0 [M], z1 [N], ind0 [M] / ind1 [N] (NULL = identity) -> row_stats [3][M] =
 *  (max, log sum exp(x - max), logsigmoid(z0)) and col_stats [3][N] alike; int64 rows (ind0[i], ind1[j]).
 * Both: best0 [M] row maxima of the final scores, arg0 [M] / arg1 [N] row / column arg-max (first maximum). */
int b2_debug_superglue_assign_host(b2_context* ctx, int path, int ctas, const float* Z, int M, int N, float alpha, int iters,
                                   float threshold, float* u, float* v, float* best0, int* arg0, int* arg1, uint32_t* out_matches,
                                   float* out_scores, int* out_k, int* out_path);
int b2_debug_lightglue_assign_host(b2_context* ctx, int path, int ctas, const float* sim, int M, int N, const float* z0,
                                   const float* z1, const int* ind0, const int* ind1, float threshold, float* row_stats,
                                   float* col_stats, float* best0, int* arg0, int* arg1, int64_t* out_matches, float* out_scores,
                                   int* out_k, int* out_path);
/* Test-only: the LightGlue assignment's statistics and mutual arg-max alone (b2_debug_lightglue_assign_host without the
 * filter): best0 [M], arg0 [M], arg1 [N].  A row or column none of whose scores beats -inf (NaN scores) gets index 0 and,
 * for rows, best0 = -inf. */
int b2_debug_lightglue_argmax_host(b2_context* ctx, int path, const float* sim, int M, int N, const float* z0, const float* z1,
                                   float* best0, int* arg0, int* arg1, int* out_path);
/* Test-only: one LightGlue kernel on HOST arrays, as one batched launch of the matcher.  Entry i (0 <= i < np <= 16) has n[i]
 * rows (0 allowed); per-row arrays are concatenated over the entries.  Every output is copied in first (what the kernel does
 * not write comes back unchanged) and followed on the device by a guard that the kernel must not touch (B2_ERR_STATE).
 *  posenc:   kp [n][2], wr [32][2] -> cs, sn [n][32] (rotary table of the bounding-box-normalised keypoints), ind [n] = 0..n-1.
 *  ln_gelu:  LayerNorm(512, eps 1e-5; g, b) + exact GELU of h [n][512]: in place, or (hi, lo given) as split planes
 *            [n][512] (hi + lo * 2^-11) with h left alone.
 *  rowheads: x [n][256] -> o1 = sigmoid(w1.x + b1) (w1 NULL: head off) and head 2 = w2.x + b2 where mode[i] & 1, written as
 *            its sigmoid to o2 where mode[i] & 2 and raw to zraw where mode[i] & 4.
 *  prune:    entries 2p, 2p + 1 are the sides of pair p: counters [p][4] = (#conf < thr side 0, side 1, #kept side 0,
 *            side 1), kept = mat > keep_thr or conf <= thr; src [n] receives the kept rows in order.
 *  gather:   rows src[0 .. cnt[i]) of x [n][256], cs / sn [n][32], ind [n] (and planes [2][n][256], hi then lo) -> x2, cs2,
 *            sn2, ind2 (planes2) rows 0 .. cnt[i).  cnt[i] <= n[i] and src entries < n[i] are checked.
 *  filter:   (m rows, n columns) mutual check a1[a0[i]] == i, score exp(best0[i]) > th -> int64 rows (ind0[i], ind1[a0[i]]) in
 *            ascending i, their scores, *out_k.  a0 entries must lie in [0, n). */
int b2_debug_lightglue_posenc_host(b2_context* ctx, int np, const int* n, const float* kp, const float* wr, float* cs, float* sn,
                                   int* ind);
int b2_debug_lightglue_ln_gelu_host(b2_context* ctx, int np, const int* n, const float* g, const float* b, float* h, uint16_t* hi,
                                    uint16_t* lo);
int b2_debug_lightglue_rowheads_host(b2_context* ctx, int np, const int* n, const int* mode, const float* x, const float* w1,
                                     const float* b1, const float* w2, const float* b2, float* o1, float* o2, float* zraw);
int b2_debug_lightglue_prune_host(b2_context* ctx, int np, const int* n, const float* conf, const float* mat, float thr,
                                  float keep_thr, int* src, int* counters);
int b2_debug_lightglue_gather_host(b2_context* ctx, int np, const int* n, const int* cnt, const int* src, const float* x,
                                   const float* cs, const float* sn, const int* ind, const uint16_t* planes, float* x2, float* cs2,
                                   float* sn2, int* ind2, uint16_t* planes2);
int b2_debug_lightglue_filter_host(b2_context* ctx, int m, int n, const float* best0, const int* a0, const int* a1, float th,
                                   const int* ind0, const int* ind1, int64_t* out_matches, float* out_scores, int* out_k);

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
 * confidence_thresholds buffer is recomputed).  As weights.pack_lightglue writes it, each block's out_proj / to_out is
 * folded into its ffn.0 and its own slot holds the identity with a zero bias; any other projection there is refused. */
int b2_lightglue_set_weights(b2_context* ctx, const float* host_blob, size_t n_floats);
/* Host-only, needs no device: out[r] (768 ints) = the checkpoint row of each self block's QKV projection that the device
 * copy holds at row r.  The device copy is [q | k | v], 256 rows each in head-major order h * 64 + j; the checkpoint
 * interleaves them as (h * 64 + j) * 3 + {q, k, v}. */
int b2_lightglue_qkv_rows(int* out);

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
 * that stop early drop out of the later launches.  Each image goes through the same kernels as in n_pairs calls of
 * b2_lightglue_match_dev, but the wgmma attention splits its key range by the launch's total work, so internal state and
 * match scores may differ from the per-pair calls in the last bits, and a match or early-exit decision that sits on its
 * threshold to that precision could differ.  The SIMT kernels (force_simt) do not split: there results are bit-identical.
 * All pointers inside `pairs` are DEVICE pointers; out_k / out_stop_layer are written on the HOST struct.
 * enc0 / enc1: NULL, or a blob b2_lightglue_encode_batched_dev made from (kp0, desc0) / (kp1, desc1) on a context with the
 * same weights and kernel path (force_simt) under the same fp16_attention; that side then skips its layer-0 self block. */
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
  const void* enc0;     /* [b2_lightglue_encoded_bytes(n0)] or NULL */
  const void* enc1;     /* [b2_lightglue_encoded_bytes(n1)] or NULL */
} b2_lightglue_pair;
int b2_lightglue_match_batched_dev(b2_context* ctx, b2_lightglue_pair* pairs, int n_pairs, const b2_lightglue_params* params,
                                   void* stream);

/* Pair-independent encoding of one image: LightGlue's state after the layer-0 self block (input_proj is the identity
 * for SuperPoint, the positional encoding normalises by the image's own bounding box, and pruning / early exit are
 * decided after layer 0's cross block, so none of it depends on the partner).  An image matched against many partners
 * is encoded once and handed to b2_lightglue_match_batched_dev as enc0 / enc1.  `out` is a caller-allocated DEVICE
 * blob of b2_lightglue_encoded_bytes(n) bytes (n = 0 allowed) whose layout is private to the library; kp / desc are
 * DEVICE pointers.  Of `params` only fp16_attention is used.  Enqueued on `stream`, does not synchronise it. */
typedef struct b2_lightglue_image {
  const float* kp;   /* [n][2] (x, y) pixels */
  const float* desc; /* [n][256] */
  int n;
  void* out;
} b2_lightglue_image;
/* The per-layer trace, recorded by every b2_lightglue_match_* call (and cleared at its start) while
 * b2_set_option("lightglue_trace", 1) is set; off by default (it synchronises after every layer).  One record per active
 * side and layer: meta [8] = (pair index in the call, side, layer, n rows, heads, #unconfident, #kept, early exit fired
 * after this layer); x [n][256] after the layer, ind [n] original row indices; with heads = 1 also conf [n], mat [n] (the
 * confidence and matchability the pruning decision read) and keep [#kept] (the rows kept, ascending).  NULL arrays are
 * skipped: call once with meta only to size them. */
int b2_lightglue_trace_count(b2_context* ctx);
int b2_lightglue_trace_get(b2_context* ctx, int i, int* meta, float* x, int* ind, float* conf, float* mat, int* keep);
size_t b2_lightglue_encoded_bytes(int n);
int b2_lightglue_encode_batched_dev(b2_context* ctx, const b2_lightglue_image* imgs, int n_imgs, const b2_lightglue_params* params,
                                    void* stream);

/* ---- SuperGlue --------------------------------------------------------------------------------------------------- */
/* `blob`: packed fp32 tensors in gtsfm_b200/weights.py::SUPERGLUE_ORDER with eval-mode BatchNorm already folded
 * into the preceding Conv1d by the host loader, and each GNN layer's attn.merge folded into its mlp.0 (the merge slot
 * holds the identity with a zero bias; any other merge is refused), as weights.pack_superglue writes it. */
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
/* The per-layer trace, recorded by every b2_superglue_match_* call (and cleared at its start) while
 * b2_set_option("superglue_trace", 1) is set; off by default (it synchronises after every layer).  meta [5] = (layer, side,
 * n rows, kind, columns); out receives n x columns floats, row-major.  Records, in order: kind 0, x [n][256] of side 0 and 1
 * after the keypoint encoder (layer -1) and after each GNN layer 0..17; kind 1, final_proj's md [n][256] of side 0 and 1
 * (layer 18); kind 2, the score matrix Z = md0 md1^T / 16 [M][N] (layer 18, side -1).  A NULL `out` is skipped: call once
 * with meta only to size it. */
int b2_superglue_trace_count(b2_context* ctx);
int b2_superglue_trace_get(b2_context* ctx, int i, int* meta, float* out);

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
/* Batched verification: n independent problems, every stage launched once for all of them, results equal bit for bit to
 * what the per-pair entry points return for each problem alone (same seed, same kernels, fixed-order reductions).
 * Points: either x1 / x2, DEVICE [k][2] double ready to use (calibrated for mode 0, pixels for mode 1), or, when both are
 * NULL, kp1 / kp2 DEVICE [n][2] float pixel coordinates + matches DEVICE [k][2] int64 rows, which the library gathers and,
 * for mode 0, calibrates with cal1 / cal2 = {f, u0, v0} as b2_ransac_essential_dev does.  Mode 1 estimates F on pixels and
 * then recovers the pose on the device as well: E = K2^T F K1 and the inliers calibrated with each side's cal
 * (gtsfm/utils/verification.py:54-112), so cal is required for mode 1 and for gathered mode 0 problems (f > 0).
 * threshold / max_iters: as in b2_ransac_params, per problem (thr_px / max(f) differs per pair; E callers pass 1000, F callers
 * 10^6).  mask: DEVICE [k] uint8, written; may be NULL. */
typedef struct b2_ransac_problem {
  const float* kp1;
  const float* kp2;
  const int64_t* matches;
  const double* x1;
  const double* x2;
  int k;
  int mode;          /* 0 = essential (5-point), 1 = fundamental (8-point) */
  int max_iters;
  double cal1[3];
  double cal2[3];
  double threshold;
  uint8_t* mask;
} b2_ransac_problem;
typedef struct b2_ransac_result {
  int status;        /* 0 ok, 1 no model (k below the minimal sample or nothing valid; mask all zero), as the per-pair return value */
  int num_inliers;
  double model[9];   /* E (mode 0) or F (mode 1), row-major */
  double R[9];       /* i2Ri1 row-major, t unit i2ti1 (cv2.recoverPose semantics) */
  double t[3];
} b2_ransac_result;
/* `params` gives the confidence and the seed of the whole call (its threshold and max_iters are not read); `results` is a
 * HOST array of n.  n = 0 and k = 0 problems are legal.  Bad arguments return B2_ERR_ARG before anything is launched.  The
 * results of a sub-batch arrive in one copy and the call synchronises `stream` once per sub-batch, plus once per further
 * sampling round where a problem's budget exceeds one round of 16 384 hypotheses (mode 1 at 10^6: the flags of all problems
 * are read together and the problems whose confidence bound is met leave the later rounds). */
int b2_ransac_verify_batched_dev(b2_context* ctx, const b2_ransac_problem* problems, int n, const b2_ransac_params* params,
                                 b2_ransac_result* results, void* stream);
/* Device workspace one problem takes in a batched call, and the cut of n problems into consecutive sub-batches under
 * `budget_bytes` that b2_ransac_verify_batched_dev makes: out_first[i] is the first problem of sub-batch i, out_first[count] =
 * n (room for n + 1), returns count.  A problem that alone exceeds the budget forms a sub-batch of its own.  Pure host
 * functions (pointer fields are only tested for NULL). */
size_t b2_ransac_workspace_bytes(const b2_ransac_problem* problem);
int b2_ransac_plan(const b2_ransac_problem* problems, int n, size_t budget_bytes, int* out_first);
/* Stream synchronisations the RANSAC entry points have performed through `ctx` since creation. */
uint64_t b2_ransac_sync_count(const b2_context* ctx);
/* cv2.recoverPose restated: decompose E, pick (R, t) with most points in front of both cameras. */
int b2_recover_pose_host(b2_context* ctx, const double* E, const double* x1, const double* x2, int k, double* out_R,
                         double* out_t, int* out_num_good);

/* Test-only: the verifier's intermediate state.  One RANSAC candidate (the layout the kernels keep on the device). */
typedef struct b2_ransac_candidate {
  double model[9];
  double cost;  /* MSAC cost; 1e300 when not valid */
  int ninl;
  int valid;
} b2_ransac_candidate;
/* A record is one k_rs_select launch: a sampling batch, or the E extension stage (always the record after the last
 * batch when it is enqueued).  Array pointers may be NULL (not recorded); the arrays have room for `max_records`. */
typedef struct b2_ransac_trace {
  int batch;                       /* in: hypotheses per launch, 1 .. 16384 (production: 16384) */
  int max_records;                 /* in: records the arrays below hold */
  int* nsol;                       /* [max_records][batch] solutions per sample */
  double* models;                  /* [max_records][batch][10][9] */
  double* cost;                    /* [max_records][batch * 10] MSAC cost per slot (1e300 for an empty slot) */
  int* ninl;                       /* [max_records][batch * 10] */
  b2_ransac_candidate* selected;   /* [max_records][8] the candidate list after the record's k_rs_select */
  int* more;                       /* [max_records] the confidence flag that select wrote (-1: the extension writes none) */
  int batches;                     /* out: sampling batches run (the extension not counted) */
  int ext_go;                      /* out: -1 extension not enqueued, else the flag it ran under (0: its kernels returned) */
  int records;                     /* out: records written (<= max_records) */
  b2_ransac_candidate prerefine[8];/* out: the list handed to k_rs_refine */
  b2_ransac_candidate refined[8];  /* out: the list after k_rs_refine */
  b2_ransac_candidate pick;        /* out: k_rs_pick's result */
  int mask_count;                  /* out: k_rs_mask's inlier count */
  int votes[4];                    /* out (E): cheirality votes of (R1,t), (R2,t), (R1,-t), (R2,-t) */
  int winner;                      /* out (E): index of the winning decomposition */
  double pose_cands[21];           /* out (E): the device's R1 [9], R2 [9], t [3] */
} b2_ransac_trace;
/* Test-only: rs_run with a trace.  mode 0 = essential (5-point, Sampson), 1 = fundamental (8-point, epiline).  Same
 * arguments and return value as b2_ransac_essential_host / _fundamental_host; out_R / out_t are used for mode 0. */
int b2_debug_ransac_trace_host(b2_context* ctx, int mode, const double* x1, const double* x2, int k,
                               const b2_ransac_params* params, b2_ransac_trace* trace, double* out_model, uint8_t* out_mask,
                               int* out_num_inliers, double* out_R, double* out_t);
/* Test-only: b2_recover_pose_host that also returns the device's four decompositions (R1 [9], R2 [9], t [3]), the four
 * vote totals and the winner's index. */
int b2_debug_recover_pose_host(b2_context* ctx, const double* E, const double* x1, const double* x2, int k, double* out_cands,
                               int* out_votes, int* out_winner, double* out_R, double* out_t, int* out_num_good);

/* ---- Two-view refinement (gtsfm/two_view_estimator.py:350-481 with bundle_adjust_2view) -------------------------------
 * For each verified pair: triangulate every verified row in the cameras Pose3() / Pose3(R, t)^-1 (DLT + gtsam's point
 * refinement, cheirality, reprojection and angle checks), bundle-adjust the two cameras (pose + Cal3Bundler f, k1, k2)
 * and the points with gtsam's robust (Huber 1.345) two-view graph and Levenberg-Marquardt schedule, reject the pair when
 * the Hessian at the optimum is indeterminate, keep the tracks whose reprojection errors are below the threshold in both
 * images, and apply the inlier-support thresholds.  fp64 throughout; oracle/twoview_ba_ref.py is the NumPy statement.
 * Cameras are distortion-free on input (k1 = k2 = 0): cal = {f, u0, v0}.  Pairs with fewer than min_num_inliers verified
 * rows are not adjusted; their verified rows go through the inlier-support decision as they are. */
typedef struct b2_twoview_problem {
  const float* kp1;        /* DEVICE [n1][2] pixel coordinates of image 1 */
  const float* kp2;        /* DEVICE [n2][2] */
  const int64_t* matches;  /* DEVICE [k][2] putative match rows */
  const uint8_t* mask;     /* DEVICE [k] verification's inlier mask: the verified rows */
  int k;
  double cal1[3];          /* f, u0, v0 */
  double cal2[3];
  double R[9];             /* verification's i2Ri1 (row-major) and unit i2ti1 */
  double t[3];
  uint8_t* out_mask;       /* DEVICE [k] or NULL: 1 for the rows of the refined v_corr_idxs */
  int64_t* out_rows;       /* DEVICE [k][2] or NULL: those rows of `matches`, compacted in row order */
} b2_twoview_problem;
typedef struct b2_twoview_params {
  int max_iters;                        /* LM iterations (the reference: 100) */
  int min_num_inliers;                  /* 15 (InlierSupportProcessor, and the condition of two_view_estimator.py:412) */
  double min_inlier_ratio;              /* 0.1; the ratio is the verified rows over k (the pre-BA ratio, :426) */
  double ba_reproj_error_threshold;     /* 0.5 px */
  double tri_reproj_error_threshold;    /* triangulation's reproj_error_threshold: inf by default, 100 in sift_front_end */
  double min_triangulation_angle;       /* degrees, 0 by default */
} b2_twoview_params;
typedef struct b2_twoview_result {
  int status;          /* 0: R, t valid and num_rows rows kept; 1: the pair fails (None, None, empty) */
  int num_rows;        /* rows set in out_mask / written to out_rows (0 on failure) */
  int num_verified;    /* verified rows (mask) */
  int num_tracks;      /* verified rows that triangulated */
  int iterations;      /* successful LM iterations */
  int bundle_adjusted; /* num_verified >= min_num_inliers: the refinement ran */
  int indeterminate;   /* the Hessian at the optimum had a pivot at or below 1e-10 of its diagonal entry */
  int trace_len;       /* costs recorded by the LM (initial + one per outer iteration) */
  double R[9];         /* refined i2Ri1 (the input pose when no track survived) */
  double t[3];         /* refined unit i2ti1 */
  double final_error;  /* graph error at the optimum */
} b2_twoview_result;
/* n pairs, each stage launched once per sub-batch (3 kernels), one synchronisation per sub-batch; results HOST [n].  A
 * pair's result does not depend on what it is batched with.  Bad arguments return B2_ERR_ARG before any launch. */
int b2_twoview_ba_batched_dev(b2_context* ctx, const b2_twoview_problem* problems, int n, const b2_twoview_params* params,
                              b2_twoview_result* results, void* stream);
/* Device workspace of one problem and the cut into sub-batches under `budget_bytes` (b2_set_option "ransac_workspace_mb"
 * is the budget of a call), as b2_ransac_workspace_bytes / b2_ransac_plan.  Pure host functions. */
size_t b2_twoview_ba_workspace_bytes(const b2_twoview_problem* problem, const b2_twoview_params* params);
int b2_twoview_ba_plan(const b2_twoview_problem* problems, int n, const b2_twoview_params* params, size_t budget_bytes,
                       int* out_first);
/* Test-only: b2_twoview_ba_batched_dev that also returns each pair's LM cost trace: out_trace HOST [n][max_iters + 2],
 * entries [0, trace_len) valid (the cost before the first iteration, then after each). */
int b2_debug_twoview_ba_trace_host(b2_context* ctx, const b2_twoview_problem* problems, int n, const b2_twoview_params* params,
                                   b2_twoview_result* results, double* out_trace, void* stream);

/* ---- Two-view reports: ground-truth metrics (gtsfm/two_view_estimator.py:290-344, 663-731; utils/metrics.py:38-129) ----
 * One unit per (pair, stage): the stage's rows are the rows of `matches` where `mask` is set (NULL: every row), in row
 * order.  With ground truth for both images (has_gt), each row gets its squared Sampson distance under the ground-truth
 * F = K2^-T [t]x R K1^-1 of i2Ti1 = wTi2.between(wTi1) and the inlier byte d2 < eval_threshold_px^2; the inlier count,
 * the np.nanmean of the inliers' and of the outliers' distances, and the rotation / unit-translation angles between the
 * stage's estimate (has_pose) and the ground truth.  fp64; oracle/twoview_report_ref.py is the NumPy statement.
 * Ground-truth cameras are distortion-free: cal = {f, u0, v0}; wRi row-major, wti the camera centre. */
typedef struct b2_twoview_eval_problem {
  const float* kp1;        /* DEVICE [n1][2] pixel coordinates of image 1 */
  const float* kp2;        /* DEVICE [n2][2] */
  const int64_t* matches;  /* DEVICE [k][2] match rows */
  const uint8_t* mask;     /* DEVICE [k] or NULL: the rows of the stage (NULL: all k) */
  int k;
  int has_pose;            /* the stage has an estimate R, t */
  int has_gt;              /* ground-truth cameras for both images */
  int pad_;
  double R[9];             /* the stage's i2Ri1 (row-major) and i2ti1 (normalised here) */
  double t[3];
  double wRi1[9];          /* ground truth wTi1, wTi2 */
  double wti1[3];
  double wRi2[9];
  double wti2[3];
  double cal1[3];          /* ground-truth f, u0, v0 */
  double cal2[3];
  double* out_d2;          /* device-accessible [k] or NULL (device or page-locked host memory): squared Sampson
                              distance of the stage's j-th row */
  uint8_t* out_inlier;     /* device-accessible [k] or NULL: its inlier byte */
} b2_twoview_eval_problem;
typedef struct b2_twoview_eval_params {
  double eval_threshold_px; /* 4 in the reference's configs */
} b2_twoview_eval_params;
typedef struct b2_twoview_eval_result {
  int num_rows;        /* the stage's rows */
  int num_inliers_gt;  /* rows with d2 < thr^2 (0 without ground truth or rows) */
  int no_gt;           /* no ground truth: the reference's mask and distances are None */
  int no_rows;         /* no rows: likewise None */
  double inlier_avg_reproj_error_gt;   /* NaN for an empty selection, as _masked_nanmean */
  double outlier_avg_reproj_error_gt;
  double R_error_deg;  /* NaN where the reference has None (no estimate or no ground truth) */
  double U_error_deg;
} b2_twoview_eval_result;
/* n units, one launch and one synchronisation; results HOST [n].  A unit's result does not depend on what it is batched
 * with.  Bad arguments return B2_ERR_ARG before any launch. */
int b2_twoview_eval_batched_dev(b2_context* ctx, const b2_twoview_eval_problem* problems, int n, const b2_twoview_eval_params* params,
                                b2_twoview_eval_result* results, void* stream);

/* ---- View-graph filter: cycle-consistent rotations (gtsfm/view_graph_estimator/cycle_consistent_rotation_estimator.py) --
 * Edge e = (edges[e][0], edges[e][1]) with 0 <= i1 < i2, each at most once, and R[e] its i2Ri1 (row-major).  Every node
 * set i0 < i1 < i2 whose three edges are inputs is a triplet with cycle error |rotvec((R(i0,i2)^T R(i1,i2)) R(i0,i1))| in
 * degrees; an edge's aggregate is the median (the mean of the two middle values for an even count) or the minimum of the
 * errors of its triplets, NaN when one of them is NaN.  An edge is kept when its aggregate < error_threshold_deg, or when it
 * is in no triplet (aggregate NaN, num_cycles 0).  fp64; oracle/view_graph_ref.py is the NumPy statement.  Image indices may
 * be sparse and large: memory is O(edges) plus the segment window of "viewgraph_workspace_mb" (b2_set_option) and 8 bytes
 * per edge (MEDIAN only); a run cut into several windows returns what one window returns, bit for bit. */
#define B2_VG_MEDIAN 0 /* EdgeErrorAggregationCriterion.MEDIAN_EDGE_ERROR */
#define B2_VG_MIN 1    /* EdgeErrorAggregationCriterion.MIN_EDGE_ERROR */
typedef struct b2_viewgraph_params {
  int criterion;               /* B2_VG_MEDIAN or B2_VG_MIN */
  int pad_;
  double error_threshold_deg;  /* 7 in the reference */
} b2_viewgraph_params;
/* HOST inputs and outputs, all in input order: keep [n], aggregate [n], num_cycles [n] (the triplets of each edge).  Bad
 * arguments (n < 0, a negative index, i1 >= i2) return B2_ERR_ARG before any launch; a repeated edge returns B2_ERR_ARG
 * after the run, with the outputs untouched.  One synchronisation; the result does not depend on the input order. */
int b2_viewgraph_cycle_filter_host(b2_context* ctx, const int32_t* edges, const double* R, int n, const b2_viewgraph_params* params,
                                   uint8_t* keep, double* aggregate, int32_t* num_cycles, void* stream);
/* Test-only: every triplet once, HOST out_nodes [capacity][3] (sorted node ids) and out_error [capacity] (degrees), in no
 * particular order; *out_count = the number of triplets (entries past `capacity` are not written). */
int b2_debug_viewgraph_triplets_host(b2_context* ctx, const int32_t* edges, const double* R, int n, int64_t capacity,
                                     int32_t* out_nodes, double* out_error, int64_t* out_count, void* stream);

/* ---- Data association: triangulation of 2-D tracks (gtsfm/data_association/data_assoc.py:205-273,
 * point3d_initializer.py:139-295) -----------------------------------------------------------------------------------------
 * Track t is measurements [track_off[t], track_off[t+1]) of meas_cam (image index, 0 <= i < num_images) and meas_uv
 * (pixels).  Camera i is cams[i] = R_wTi (9, row-major), t_wTi (3), f, u0, v0 (Cal3Bundler without distortion), used only
 * where cam_valid[i] != 0.  RANSAC_SAMPLE_UNIFORM: min(num_hypotheses, C(n, 2)) two-view hypotheses per track of n
 * measurements (every pair when C(n, 2) <= num_hypotheses, else a keyed permutation of the pairs, seed and track position:
 * csrc/data_assoc_math.cuh), each triangulated with triangulatePoint3(rank_tol 1e-9, optimize) and scored by its inliers
 * (projectSafe error < reproj_error_threshold); most inliers wins, then the lower average inlier error, then the earlier
 * hypothesis.  NO_RANSAC: every measurement is an inlier.  Then, in this order: < 2 inliers -> INLIERS_UNDERCONSTRAINED,
 * < 2 inliers with a camera -> POSES_UNDERCONSTRAINED, n-view triangulatePoint3 of those failing -> CHEIRALITY_FAILURE, an
 * inlier's error (NaN without a camera) not below the threshold -> EXCEEDS_REPROJ_THRESH, every pairwise triangulation
 * angle below min_triangulation_angle -> LOW_TRIANGULATION_ANGLE, else SUCCESS.  fp64; oracle/data_assoc_ref.py is the
 * NumPy statement.  Tracks are processed in chunks under "data_assoc_workspace_mb" (b2_set_option); a chunked run returns
 * what one chunk returns, bit for bit. */
#define B2_TRI_NO_RANSAC 0      /* TriangulationSamplingMode.NO_RANSAC */
#define B2_TRI_SAMPLE_UNIFORM 1 /* TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM */
typedef struct b2_triangulation_params {
  int mode;                       /* B2_TRI_NO_RANSAC or B2_TRI_SAMPLE_UNIFORM */
  int num_hypotheses;             /* TriangulationOptions.num_ransac_hypotheses() (>= 1; unused by NO_RANSAC) */
  double reproj_error_threshold;  /* px, > 0, may be inf */
  double min_triangulation_angle; /* degrees */
  uint64_t seed;                  /* keys the permutation of tracks with more pairs than hypotheses */
} b2_triangulation_params;
/* HOST inputs and outputs.  Per track: exit_code [T] (TriangulationExitCode), point [T][3] (NaN unless the n-view
 * triangulation ran: exit codes 0, 4, 5), avg_err [T] (nanmean of the inliers' errors; NaN for exit codes 1-3, the
 * reference's None); per measurement: inlier [M] (the RANSAC inlier set, or all for NO_RANSAC).  Bad arguments return
 * B2_ERR_ARG before any launch.  One synchronisation per chunk. */
int b2_triangulate_tracks_host(b2_context* ctx, const int64_t* track_off, int64_t T, const int32_t* meas_cam, const double* meas_uv,
                               const double* cams, const uint8_t* cam_valid, int num_images, const b2_triangulation_params* params,
                               int8_t* exit_code, double* point, double* avg_err, uint8_t* inlier, void* stream);

/* ---- LMedS verifier (gtsfm/frontend/verifier/lmeds.py: cv2.findEssentialMat / findFundamentalMat with LMEDS) ----------
 * A batched device restatement of cv2's LMeDS estimator: cv::RNG subsets (seed 2^64 - 1, F subsets with collinear points
 * redrawn), max(3, RANSACUpdateNumIters(confidence, 0.45, m, max_iters)) subsets, every real root of the 5-point problem (E)
 * or of the 7-point cubic (F, points rounded to float32 and F33 = 1), the median of the float errors, the lowest median in
 * visiting order, and the inliers err <= (float)sigma^2 with sigma = max(0.001, 2.5 * 1.4826 * (1 + 5 / (k - m)) * sqrt(median)).
 * Problems and results are b2_ransac_problem / b2_ransac_result: mode 0 = E (5-point, calibrated points), 1 = F (7-point,
 * pixels); `threshold` is not read; `max_iters` is cv2's maxIters (<= 0: 1000, at most 65 536).  An E problem needs k >= 6,
 * an F problem k >= 8 (the reference's guards; status 1 below that); status is 0 when a model was found (F: and at least 7
 * inliers), and the pose is recovered as b2_ransac_verify_batched_dev does.  One synchronisation per sub-batch. */
typedef struct b2_lmeds_params {
  double confidence[2];  /* per mode: E 0.999 (cv2.findEssentialMat prob), F 0.99 (cv2.findFundamentalMat confidence) */
} b2_lmeds_params;
int b2_lmeds_verify_batched_dev(b2_context* ctx, const b2_ransac_problem* problems, int n, const b2_lmeds_params* params,
                                b2_ransac_result* results, void* stream);
/* Device workspace of one problem, and the cut into sub-batches under `budget_bytes` (b2_set_option "ransac_workspace_mb"
 * is the budget of a call), as b2_ransac_workspace_bytes / b2_ransac_plan.  Pure host functions. */
size_t b2_lmeds_workspace_bytes(const b2_ransac_problem* problem, const b2_lmeds_params* params);
int b2_lmeds_plan(const b2_ransac_problem* problems, int n, const b2_lmeds_params* params, size_t budget_bytes, int* out_first);
/* Test-only: one problem on host points (x1 / x2 [k][2] double), with the intermediate state. */
typedef struct b2_lmeds_trace {
  int cap;            /* in: subsets the arrays below hold (>= the problem's iteration count) */
  int* idx;           /* [cap][m] subset table */
  int* nsol;          /* [cap] solutions per subset */
  double* models;     /* [cap][10][9] */
  float* medians;     /* [cap * 10] median per slot (NaN: empty slot) */
  int niters;         /* out: iteration count */
  int drawn;          /* out: subsets drawn */
  int slot;           /* out: chosen slot (subset * 10 + solution), -1 none */
  float min_median;   /* out */
  double sigma;       /* out */
  float thr;          /* out: (float)sigma^2 */
  int count;          /* out: inliers */
} b2_lmeds_trace;
int b2_debug_lmeds_trace_host(b2_context* ctx, int mode, const double* x1, const double* x2, int k, const b2_lmeds_params* params,
                              int max_iters, b2_lmeds_trace* trace, b2_ransac_result* result, uint8_t* out_mask);

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

/* ---- ORB detector-descriptor (gtsfm/frontend/detector_descriptor/orb.py) ------------------------------------------------------ */
/* cv2.ORB_create() with its defaults restated bit for bit: 500 features, scale factor 1.2f, 8 levels, edge threshold 31, FAST
 * threshold 20, Harris score, patch 31, WTA_K 2.  Images are uint8 H x W x {1, 3, 4} interleaved (RGB / RGBA go through cv2's
 * fixed-point COLOR_RGB2GRAY); H x W <= 2^24 and each side <= 16384, larger input fails with -2.  A mask keeps a keypoint where
 * it is non-zero, on every level as cv2 carries it down the pyramid.  Keypoints (b2_sift_keypoint: x, y, size = 31 s_l, angle,
 * Harris response, octave = level) come level by level, each level by response descending, then y, then x (cv2's order within
 * a level is std::nth_element's and is not reproduced); the set and every field equal cv2's.  Descriptors are 32 uint8 bytes per
 * keypoint.  Results do not depend on the batch or the run.  Workspace: about 40 H W bytes per image of a batch. */
typedef struct b2_orb_image {
  const uint8_t* image;             /* DEVICE image, row pitch as passed to the call */
  const uint8_t* mask;              /* DEVICE H x W uint8, dense, or NULL */
  int max_keypoints;                /* >= 1: the max_keypoints largest responses (ties to the lower index), the order kept */
  b2_sift_keypoint* out_keypoints;  /* DEVICE [max_keypoints] */
  uint8_t* out_desc;                /* DEVICE [max_keypoints][32] */
  int out_n;                        /* written on the HOST struct: keypoints written */
  int out_total;                    /* written on the HOST struct: keypoints before the top-k */
} b2_orb_image;
/* Up to 64 same-shape images: every stage is one launch over the batch, counts stay on the device, and `stream` is synchronised
 * once at the end. */
int b2_orb_detect_batched_dev(b2_context* ctx, b2_orb_image* images, int n_images, int height, int width, int channels,
                              size_t pitch, void* stream);
/* HOST pointers, dense image, optional mask: every keypoint (no top-k).  When there are more than `capacity` keypoints nothing
 * is written and the call returns -5 with *out_n = the number needed; otherwise *out_n = the number written. */
int b2_orb_detect_host(b2_context* ctx, const uint8_t* image, int height, int width, int channels, const uint8_t* mask,
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
 *  b2_debug_d2net_avgpool_host: the AvgPool2d(2, stride=1) kernel on fp32 NHWC [H][W][256] -> [H - 1][W - 1][256] (hi + lo planes);
 *  b2_debug_d2net_rank_host: the keypoint ordering on n candidates (score, c, i, j) -> order[r] = candidate of rank r < min(n, max_k). */
int b2_debug_d2net_avgpool_host(b2_context* ctx, const float* in, int height, int width, float* out);
int b2_debug_d2net_rank_host(b2_context* ctx, const float* scores, const int* cij, int n, int max_k, int* order);

/* ---- baseline JPEG decode (gtsfm/utils/io.py:39-72 load_image: np.asarray(PIL.Image.open(f).convert("RGB"))) --------------------
 * Output equals PIL's (libjpeg-turbo defaults: islow IDCT, fancy upsampling, jdcolor.c's fixed-point YCbCr -> RGB) bit for bit.
 * Scope: SOF0 / SOF1, 8-bit, Huffman coded, one scan holding every component: 3-component YCbCr with luma sampling h1v1, h2v1,
 * h1v2 or h2v2 and chroma 1x1, or 1-component gray (replicated to three channels); optional restart intervals; any size.
 * EXIF orientation is not applied.  Everything else is refused with a status naming it:
 *   -2 beyond the limits (a side over 16384, over 2^26 pixels, a file over 256 MiB, or an output pitch under 3 W)
 *   -10 not a JPEG / corrupt header, -11 progressive, -12 arithmetic coding, -13 lossless or hierarchical, -14 not 8-bit,
 *   -15 not 1 or 3 components (CMYK / YCCK), -16 RGB colour space (Adobe transform 0, or component ids R G B without JFIF),
 *   -17 other sampling factors, -18 multi-scan, -19 DNL, -20 truncated (no EOI after the scan), -21 corrupt entropy-coded data
 *   (invalid code, coefficient index past 63, wrong MCU count, restart marker out of sequence), -22 a Huffman table with an
 *   all-ones code (which encoders never write).
 * b2_jpeg_status_string(code) gives the text of a status. */
const char* b2_jpeg_status_string(int code);
/* Header only (markers up to SOS, plus the presence of an EOI after the scan): no context, no GPU.  0 or a status above. */
int b2_jpeg_info_host(const uint8_t* data, size_t size, int* height, int* width, int* components);
typedef struct b2_jpeg_image {
  const uint8_t* data; /* HOST file bytes */
  size_t size;
  uint8_t* out;        /* DEVICE H x W x 3 uint8, row pitch out_pitch bytes (>= 3 W) */
  size_t out_pitch;
  int out_status;      /* written on the HOST struct: 0, or a status above (nothing is written to `out`) */
  int out_rounds;      /* written on the HOST struct: synchronisation rounds the entropy decode took (9 = serial fallback) */
} b2_jpeg_image;
/* Up to 256 images of any sizes and sampling factors.  The compressed bytes go up in one copy through pinned staging, every
 * stage is one launch over the batch, and `stream` is synchronised once.  Returns 0 when the batch ran (per-image results in
 * out_status), -2 for more than 256 images.  Workspace: 2 bytes per coefficient (64 per block) plus the MCU-padded component planes, about 4.5 bytes per pixel at 4:2:0
 * and 9 at 4:4:4, plus about 3 x the compressed size. */
int b2_jpeg_decode_batched_dev(b2_context* ctx, b2_jpeg_image* images, int n_images, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GTSFM_B200_H */
