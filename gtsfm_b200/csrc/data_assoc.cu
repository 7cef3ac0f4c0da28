// Data association's triangulation for sm_90a: DataAssociation.run_triangulation over a batch of 2-D tracks
// (gtsfm/data_association/data_assoc.py:205-273, point3d_initializer.py:139-295), fp64 throughout.  The per-track maths is
// data_assoc_math.cuh on twoview_math.cuh's DLT and point LM; oracle/data_assoc_ref.py states the same in NumPy.
//
// Most tracks have 2-4 measurements while a few span hundreds of images, so the RANSAC work is spread over hypotheses,
// not tracks:
//   k_da_hyp    one thread per hypothesis of the chunk's flat hypothesis grid (offsets: a host scan of the per-track
//               counts): its pair, the two-view triangulation, the errors of the whole track -> votes and average error
//   k_da_track  one thread per track: the best hypothesis (most votes, then the lower average, then the earlier one), its
//               inlier set again from the same compiled scoring function (da_score), then the n-view triangulation of the inliers with a camera and
//               the exit-code checks.  NO_RANSAC runs this kernel alone.
// Chunks hold whole tracks under "data_assoc_workspace_mb"; nothing in a track's arithmetic depends on the chunk, so a
// chunked run returns the bits of an unchunked one.
#include <math.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "data_assoc_math.cuh"
#include "../../include/gtsfm_b200.h"

namespace {
constexpr int DA_THREADS = 128;

struct DaChunk {
  const tvmath::Cam* cams;
  const uint8_t* cam_valid;
  const int64_t* track_off;  // [T + 1], chunk-local
  const int64_t* hyp_off;    // [T + 1], chunk-local
  const int32_t* meas_cam;
  const double* meas_uv;
  int32_t* sel;              // [M] scratch: the measurements the final triangulation uses, per track at its offset
  int* votes;                // [H]
  double* herr;              // [H]
  int8_t* exit_code;
  double* point;
  double* avg_err;
  uint8_t* inlier;
  int* flags;                // bit 0: a rebuilt inlier set disagreed with its votes
  int64_t T, H;
  int64_t track0;            // position of the chunk's first track in the input (keys the sampler)
  int mode, num_hyp;
  double thr, min_angle;
  uint64_t seed;
};

__device__ __forceinline__ const tvmath::Cam* cam_or_null(const DaChunk& c, int64_t m) {
  const int i = c.meas_cam[m];
  return c.cam_valid[i] ? c.cams + i : nullptr;
}

// Hypothesis h of track t (n measurements from `m0`): -1 when skipped (a camera without a pose, or a failed
// triangulation), else its votes, with the sum of the inlier errors in *sum and, when `inlier` is not NULL, the inlier
// mask of the track's measurements.  Not inlined: k_da_hyp's scoring and k_da_track's rebuild of the winner's inlier set
// run this one compiled body, so the rebuilt set is the one that was voted for, bit for bit.
__device__ __noinline__ int da_score(const DaChunk& c, int64_t t, int64_t h, int64_t m0, int n, double* sum, double* X,
                                     uint8_t* inlier) {
  const int64_t pairs = (int64_t)n * (n - 1) / 2;
  const int64_t hyps = c.hyp_off[t + 1] - c.hyp_off[t];
  const int64_t p = damath::sample_pair(damath::sampler_key(c.seed, (uint64_t)(c.track0 + t)), h, pairs, hyps);
  int k1, k2;
  damath::pair_of(p, n, &k1, &k2);
  const tvmath::Cam* c1 = cam_or_null(c, m0 + k1);
  const tvmath::Cam* c2 = cam_or_null(c, m0 + k2);
  *sum = 0.0;
  if (!c1 || !c2) return -1;
  const damath::PairViews v{{c1, c2}, {c.meas_uv + 2 * (m0 + k1), c.meas_uv + 2 * (m0 + k2)}};
  if (!damath::triangulate_views(v, X)) return -1;
  int votes = 0;
  double s = 0.0;
  for (int k = 0; k < n; ++k) {
    const double e = damath::reproj_error(cam_or_null(c, m0 + k), c.meas_uv + 2 * (m0 + k), X);
    const bool in = e < c.thr;
    if (in) s += e, ++votes;
    if (inlier) inlier[k] = in;
  }
  *sum = s;
  return votes;
}

__global__ void __launch_bounds__(DA_THREADS) k_da_hyp(DaChunk c) {
  const int64_t g = (int64_t)blockIdx.x * DA_THREADS + threadIdx.x;
  if (g >= c.H) return;
  int64_t lo = 0, hi = c.T;  // the track t with hyp_off[t] <= g < hyp_off[t + 1]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) / 2;
    if (c.hyp_off[mid] <= g) lo = mid;
    else hi = mid;
  }
  const int64_t t = lo, m0 = c.track_off[t];
  double X[3], sum;
  const int votes = da_score(c, t, g - c.hyp_off[t], m0, (int)(c.track_off[t + 1] - m0), &sum, X, nullptr);
  c.votes[g] = votes;
  c.herr[g] = votes > 0 ? sum / votes : 0.0;
}

__global__ void __launch_bounds__(DA_THREADS) k_da_track(DaChunk c) {
  const int64_t t = (int64_t)blockIdx.x * DA_THREADS + threadIdx.x;
  if (t >= c.T) return;
  const int64_t m0 = c.track_off[t];
  const int n = (int)(c.track_off[t + 1] - m0);
  double* P = c.point + 3 * t;
  P[0] = P[1] = P[2] = NAN;
  c.avg_err[t] = NAN;
  int num_in = 0;
  if (c.mode == B2_TRI_NO_RANSAC) {
    for (int k = 0; k < n; ++k) c.inlier[m0 + k] = 1;
    num_in = n;
  } else {
    int64_t best = -1;
    int best_votes = 0;
    double best_err = 3.4028234663852886e38;  // point3d_initializer.MAX_TRACK_REPROJ_ERROR
    for (int64_t g = c.hyp_off[t]; g < c.hyp_off[t + 1]; ++g) {
      const int v = c.votes[g];
      if (v > 0 && (v > best_votes || (v == best_votes && c.herr[g] < best_err))) best = g, best_votes = v, best_err = c.herr[g];
    }
    double X[3], sum;
    if (best >= 0) {
      num_in = da_score(c, t, best - c.hyp_off[t], m0, n, &sum, X, c.inlier + m0);
      if (num_in != best_votes) atomicOr(c.flags, 1);  // cannot happen: the same code scored it
    } else {
      for (int k = 0; k < n; ++k) c.inlier[m0 + k] = 0;
    }
  }
  if (num_in < 2) {
    c.exit_code[t] = damath::INLIERS_UNDERCONSTRAINED;
    return;
  }
  int nv = 0;
  for (int k = 0; k < n; ++k)
    if (c.inlier[m0 + k] && cam_or_null(c, m0 + k)) c.sel[m0 + nv++] = (int32_t)(m0 + k);
  if (nv < 2) {
    c.exit_code[t] = damath::POSES_UNDERCONSTRAINED;
    return;
  }
  const damath::ListViews v{c.cams, c.meas_cam, c.meas_uv, c.sel + m0, nv};
  double X[3];
  if (!damath::triangulate_views(v, X)) {
    c.exit_code[t] = damath::CHEIRALITY_FAILURE;
    return;
  }
  P[0] = X[0], P[1] = X[1], P[2] = X[2];
  bool within = true;
  double sum = 0.0;
  int cnt = 0;
  for (int k = 0; k < n; ++k) {
    if (!c.inlier[m0 + k]) continue;
    const double e = damath::reproj_error(cam_or_null(c, m0 + k), c.meas_uv + 2 * (m0 + k), X);
    within = within && e < c.thr;
    if (!isnan(e)) sum += e, ++cnt;
  }
  c.avg_err[t] = cnt ? sum / cnt : NAN;
  if (!within) c.exit_code[t] = damath::EXCEEDS_REPROJ_THRESH;
  else if (!damath::angle_at_least(v, X, c.min_angle)) c.exit_code[t] = damath::LOW_TRIANGULATION_ANGLE;
  else c.exit_code[t] = damath::SUCCESS;
}
}  // namespace

struct DataAssocState {
  DevBuf flags, cams, valid, track_off, hyp_off, meas_cam, meas_uv, sel, votes, herr, exit_code, point, avg_err, inlier;
};

void da_destroy(b2_context* ctx) {
  delete ctx->da;
  ctx->da = nullptr;
}

extern "C" int b2_triangulate_tracks_host(b2_context* ctx, const int64_t* track_off, int64_t T, const int32_t* meas_cam,
                                          const double* meas_uv, const double* cams, const uint8_t* cam_valid, int num_images,
                                          const b2_triangulation_params* params, int8_t* exit_code, double* point, double* avg_err,
                                          uint8_t* inlier, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (!params) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: params is NULL");
  const b2_triangulation_params prm = *params;
  if (prm.mode != B2_TRI_NO_RANSAC && prm.mode != B2_TRI_SAMPLE_UNIFORM)
    return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: mode must be B2_TRI_NO_RANSAC or B2_TRI_SAMPLE_UNIFORM");
  if (prm.mode == B2_TRI_SAMPLE_UNIFORM && prm.num_hypotheses < 1)
    return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: num_hypotheses must be >= 1");
  if (!(prm.reproj_error_threshold > 0.0)) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: reproj_error_threshold must be > 0");
  if (isnan(prm.min_triangulation_angle)) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: min_triangulation_angle is NaN");
  if (T < 0 || num_images < 0) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: T < 0 or num_images < 0");
  if (T == 0) return B2_OK;
  if (!track_off || !exit_code || !point || !avg_err) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: a track array is NULL");
  if (track_off[0] != 0) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: track_off[0] must be 0");
  for (int64_t t = 0; t < T; ++t)
    if (track_off[t + 1] < track_off[t] || track_off[t + 1] - track_off[t] > (1 << 20))
      return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: track_off must be non-decreasing, with at most 2^20 measurements per track");
  const int64_t M = track_off[T];
  if (M > 0 && (!meas_cam || !meas_uv || !inlier)) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: a measurement array is NULL");
  if (M >= (1ll << 31)) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: more than 2^31 - 1 measurements");
  for (int64_t m = 0; m < M; ++m)
    if (meas_cam[m] < 0 || meas_cam[m] >= num_images) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: meas_cam out of [0, num_images)");
  if (num_images > 0 && (!cams || !cam_valid)) return b2_fail(ctx, B2_ERR_ARG, "triangulate tracks: cams or cam_valid is NULL");

  // per-track hypothesis counts and the chunk plan (whole tracks under the budget; a track larger than it runs alone)
  std::vector<int64_t> hyp(T + 1, 0);
  for (int64_t t = 0; t < T; ++t) {
    const int64_t n = track_off[t + 1] - track_off[t], pairs = n * (n - 1) / 2;
    hyp[t + 1] = hyp[t] + (prm.mode == B2_TRI_NO_RANSAC ? 0 : std::min<int64_t>(pairs, prm.num_hypotheses));
  }
  const int64_t budget = (int64_t)ctx->da_workspace_mb << 20;
  const int64_t per_track = 2 * 8 + 1 + 3 * 8 + 8, per_meas = 4 + 16 + 4 + 1, per_hyp = 4 + 8;
  std::vector<int64_t> cut{0};
  int64_t maxT = 0, maxM = 0, maxH = 0;
  for (int64_t t = 0; t < T;) {
    const int64_t t0 = t;
    int64_t bytes = 0;
    do {
      bytes += per_track + per_meas * (track_off[t + 1] - track_off[t]) + per_hyp * (hyp[t + 1] - hyp[t]);
      ++t;
    } while (t < T && bytes + per_track + per_meas * (track_off[t + 1] - track_off[t]) + per_hyp * (hyp[t + 1] - hyp[t]) <= budget);
    cut.push_back(t);
    maxT = std::max(maxT, t - t0);
    maxM = std::max(maxM, track_off[t] - track_off[t0]);
    maxH = std::max(maxH, hyp[t] - hyp[t0]);
  }

  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  if (!ctx->da) ctx->da = new DataAssocState();
  DataAssocState* s = ctx->da;
  std::vector<tvmath::Cam> hc((size_t)num_images);
  for (int i = 0; i < num_images; ++i) {
    const double* c = cams + 15 * (size_t)i;
    tvmath::Cam& d = hc[i];
    memcpy(d.R, c, 9 * sizeof(double));
    memcpy(d.t, c + 9, 3 * sizeof(double));
    d.cal[0] = c[12], d.cal[1] = 0.0, d.cal[2] = 0.0, d.cal[3] = c[13], d.cal[4] = c[14];
  }
  B2_CUDA(ctx, s->cams.ensure(std::max<size_t>(1, hc.size()) * sizeof(tvmath::Cam)));
  B2_CUDA(ctx, s->valid.ensure(std::max(1, num_images)));
  B2_CUDA(ctx, s->track_off.ensure((size_t)(maxT + 1) * 8));
  B2_CUDA(ctx, s->hyp_off.ensure((size_t)(maxT + 1) * 8));
  B2_CUDA(ctx, s->meas_cam.ensure(std::max<size_t>(1, maxM) * 4));
  B2_CUDA(ctx, s->meas_uv.ensure(std::max<size_t>(1, maxM) * 16));
  B2_CUDA(ctx, s->sel.ensure(std::max<size_t>(1, maxM) * 4));
  B2_CUDA(ctx, s->inlier.ensure(std::max<size_t>(1, maxM)));
  B2_CUDA(ctx, s->votes.ensure(std::max<size_t>(1, maxH) * 4));
  B2_CUDA(ctx, s->herr.ensure(std::max<size_t>(1, maxH) * 8));
  B2_CUDA(ctx, s->exit_code.ensure((size_t)maxT));
  B2_CUDA(ctx, s->point.ensure((size_t)maxT * 24));
  B2_CUDA(ctx, s->avg_err.ensure((size_t)maxT * 8));
  B2_CUDA(ctx, s->flags.ensure(sizeof(int)));
  B2_CUDA(ctx, cudaMemsetAsync(s->flags.p, 0, sizeof(int), st));
  if (num_images > 0) {
    B2_CUDA(ctx, cudaMemcpyAsync(s->cams.p, hc.data(), hc.size() * sizeof(tvmath::Cam), cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->valid.p, cam_valid, (size_t)num_images, cudaMemcpyHostToDevice, st));
  }
  std::vector<int64_t> loc_off((size_t)maxT + 1), loc_hyp((size_t)maxT + 1);
  for (size_t j = 0; j + 1 < cut.size(); ++j) {
    const int64_t t0 = cut[j], t1 = cut[j + 1], nt = t1 - t0, mb = track_off[t0], nm = track_off[t1] - mb, nh = hyp[t1] - hyp[t0];
    for (int64_t t = 0; t <= nt; ++t) loc_off[t] = track_off[t0 + t] - mb, loc_hyp[t] = hyp[t0 + t] - hyp[t0];
    B2_CUDA(ctx, cudaMemcpyAsync(s->track_off.p, loc_off.data(), (size_t)(nt + 1) * 8, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(s->hyp_off.p, loc_hyp.data(), (size_t)(nt + 1) * 8, cudaMemcpyHostToDevice, st));
    if (nm > 0) {
      B2_CUDA(ctx, cudaMemcpyAsync(s->meas_cam.p, meas_cam + mb, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
      B2_CUDA(ctx, cudaMemcpyAsync(s->meas_uv.p, meas_uv + 2 * mb, (size_t)nm * 16, cudaMemcpyHostToDevice, st));
    }
    DaChunk c{s->cams.as<tvmath::Cam>(), s->valid.as<uint8_t>(), s->track_off.as<int64_t>(), s->hyp_off.as<int64_t>(),
              s->meas_cam.as<int32_t>(), s->meas_uv.as<double>(), s->sel.as<int32_t>(), s->votes.as<int>(), s->herr.as<double>(),
              s->exit_code.as<int8_t>(), s->point.as<double>(), s->avg_err.as<double>(), s->inlier.as<uint8_t>(), s->flags.as<int>(),
              nt, nh, t0, prm.mode, prm.num_hypotheses, prm.reproj_error_threshold, prm.min_triangulation_angle, prm.seed};
    if (nh > 0) {
      B2_LAUNCH(ctx, k_da_hyp, (unsigned)((nh + DA_THREADS - 1) / DA_THREADS), DA_THREADS, 0, st, c);
      B2_CHECK_LAUNCH(ctx);
    }
    B2_LAUNCH(ctx, k_da_track, (unsigned)((nt + DA_THREADS - 1) / DA_THREADS), DA_THREADS, 0, st, c);
    B2_CHECK_LAUNCH(ctx);
    B2_CUDA(ctx, cudaMemcpyAsync(exit_code + t0, c.exit_code, (size_t)nt, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(point + 3 * t0, c.point, (size_t)nt * 24, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(avg_err + t0, c.avg_err, (size_t)nt * 8, cudaMemcpyDeviceToHost, st));
    if (nm > 0) B2_CUDA(ctx, cudaMemcpyAsync(inlier + mb, c.inlier, (size_t)nm, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
  }
  int flags = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&flags, s->flags.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (flags) return b2_fail(ctx, B2_ERR_STATE, "triangulate tracks: a rebuilt inlier set disagreed with its hypothesis's votes");
  return B2_OK;
}
