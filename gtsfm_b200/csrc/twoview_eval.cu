// Ground-truth evaluation of the two-view reports for sm_90a: the metrics GTSfM's run_2view puts into its pre-BA and
// post-BA TwoViewEstimationReport (gtsfm/two_view_estimator.py:290-344, 663-731; gtsfm/utils/metrics.py:38-129) for a
// batch of (pair, stage) units.  oracle/twoview_report_ref.py states the same maths in NumPy.
//   k_tv_eval  one CTA per unit: the ground-truth F of the pair (thread 0, twoview_eval.cuh), then every evaluated row in
//              row order: its squared Sampson distance and inlier byte written at the row's rank among the evaluated
//              rows, and per-thread sums that are reduced in a fixed tree, so a unit's result does not depend on what it
//              is batched with; the pose errors of the stage's estimate against the ground truth.
// A call is one launch, one copy of the problem table in, one copy of the results out and one synchronisation.
#include <math.h>
#include <string.h>

#include <string>

#include "common.cuh"
#include "twoview_eval.cuh"
#include "../../include/gtsfm_b200.h"

using namespace tveval;

namespace {
constexpr int TE_THREADS = 256;

struct TeOut {
  int num_rows, num_inliers, no_gt, no_rows;
  double inlier_avg, outlier_avg, R_error_deg, U_error_deg;
};
}  // namespace

__global__ void __launch_bounds__(TE_THREADS) k_tv_eval(const b2_twoview_eval_problem* __restrict__ tab, double thr2,
                                                        TeOut* __restrict__ out) {
  __shared__ double sF[9];
  __shared__ int s_warp[TE_THREADS / 32];
  __shared__ double s_sum[2][TE_THREADS / 32];
  __shared__ int s_cnt[2][TE_THREADS / 32];
  const b2_twoview_eval_problem& p = tab[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    double R[9], t[3];
    gt_relative(p.wRi1, p.wti1, p.wRi2, p.wti2, R, t);
    gt_fundamental(R, t, p.cal1, p.cal2, sF);
    TeOut& o = out[blockIdx.x];
    const bool pose = p.has_gt && p.has_pose;
    o.R_error_deg = pose ? rotation_angle_deg(p.R, R) : NAN;
    o.U_error_deg = pose ? unit_angle_deg(p.t, t) : NAN;
  }
  __syncthreads();
  // every thread owns the rows tid, tid + 256, ...: its partial sums only depend on the unit's own rows
  int base = 0, n_in = 0, n_out = 0;
  double s_in = 0.0, s_out = 0.0;
  for (int r0 = 0; r0 < p.k; r0 += TE_THREADS) {
    const int row = r0 + tid;
    const int keep = row < p.k && (p.mask == nullptr || p.mask[row] != 0);
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int off = base, tot = 0;
    for (int w = 0; w < TE_THREADS / 32; ++w) off += w < warp ? s_warp[w] : 0, tot += s_warp[w];
    off += __popc(bal & ((1u << lane) - 1u));
    if (keep && p.has_gt) {
      const long long i1 = p.matches[2 * row], i2 = p.matches[2 * row + 1];
      const double d2 = sampson_sq(sF, (double)p.kp1[2 * i1], (double)p.kp1[2 * i1 + 1], (double)p.kp2[2 * i2],
                                   (double)p.kp2[2 * i2 + 1]);
      const bool inl = d2 < thr2;  // strict, as the reference; NaN is an outlier
      if (p.out_d2) p.out_d2[off] = d2;
      if (p.out_inlier) p.out_inlier[off] = (uint8_t)inl;
      if (inl) {
        ++n_in, s_in += d2;
      } else if (!isnan(d2)) {  // np.nanmean: NaN entries leave both the sum and the count
        ++n_out, s_out += d2;
      }
    }
    base += tot;
    __syncthreads();
  }
  for (int o = 16; o > 0; o >>= 1) {
    n_in += __shfl_down_sync(0xffffffffu, n_in, o);
    n_out += __shfl_down_sync(0xffffffffu, n_out, o);
    s_in += __shfl_down_sync(0xffffffffu, s_in, o);
    s_out += __shfl_down_sync(0xffffffffu, s_out, o);
  }
  if (lane == 0) s_cnt[0][warp] = n_in, s_cnt[1][warp] = n_out, s_sum[0][warp] = s_in, s_sum[1][warp] = s_out;
  __syncthreads();
  if (tid == 0) {
    int ci = 0, co = 0;
    double si = 0.0, so = 0.0;
    for (int w = 0; w < TE_THREADS / 32; ++w) ci += s_cnt[0][w], co += s_cnt[1][w], si += s_sum[0][w], so += s_sum[1][w];
    TeOut& o = out[blockIdx.x];
    o.num_rows = base;
    o.no_gt = !p.has_gt;
    o.no_rows = base == 0;
    const bool metrics = p.has_gt && base > 0;
    o.num_inliers = metrics ? ci : 0;
    o.inlier_avg = metrics && ci > 0 ? si / ci : NAN;
    o.outlier_avg = metrics && co > 0 ? so / co : NAN;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct TwoViewEvalState {
  DevBuf tab, out;
  HostBuf htab, hout;
};

static int te_check(b2_context* ctx, const b2_twoview_eval_problem* problems, int n, const b2_twoview_eval_params* prm) {
  if (!prm) return b2_fail(ctx, B2_ERR_ARG, "twoview eval: params is NULL");
  if (!(prm->eval_threshold_px > 0.0) || !isfinite(prm->eval_threshold_px))
    return b2_fail(ctx, B2_ERR_ARG, "twoview eval: eval_threshold_px must be finite and > 0");
  for (int i = 0; i < n; ++i) {
    const b2_twoview_eval_problem& p = problems[i];
    const std::string at = "twoview eval problem " + std::to_string(i) + ": ";
    if (p.k < 0) return b2_fail(ctx, B2_ERR_ARG, at + "k < 0");
    if (p.k > 0 && p.has_gt && (!p.kp1 || !p.kp2 || !p.matches)) return b2_fail(ctx, B2_ERR_ARG, at + "no points / matches");
    if (p.has_gt && !(p.cal1[0] > 0.0 && p.cal2[0] > 0.0)) return b2_fail(ctx, B2_ERR_ARG, at + "focal length must be > 0");
  }
  return B2_OK;
}

void te_destroy(b2_context* ctx) {
  delete ctx->te;
  ctx->te = nullptr;
}

extern "C" int b2_twoview_eval_batched_dev(b2_context* ctx, const b2_twoview_eval_problem* problems, int n,
                                           const b2_twoview_eval_params* params, b2_twoview_eval_result* results, void* stream) {
  if (!ctx || n < 0 || (n > 0 && (!problems || !results))) return B2_ERR_ARG;
  if (int rc = te_check(ctx, problems, n, params)) return rc;
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->te) ctx->te = new TwoViewEvalState();
  TwoViewEvalState* s = ctx->te;
  const size_t tb = (size_t)n * sizeof(b2_twoview_eval_problem), ob = (size_t)n * sizeof(TeOut);
  B2_CUDA(ctx, s->tab.ensure(tb));
  B2_CUDA(ctx, s->out.ensure(ob));
  B2_CUDA(ctx, s->htab.ensure(tb));
  B2_CUDA(ctx, s->hout.ensure(ob));
  cudaStream_t st = stream ? (cudaStream_t)stream : cudaStreamLegacy;
  memcpy(s->htab.p, problems, tb);
  B2_CUDA(ctx, cudaMemcpyAsync(s->tab.p, s->htab.p, tb, cudaMemcpyHostToDevice, st));
  const double thr = params->eval_threshold_px;
  B2_LAUNCH(ctx, k_tv_eval, dim3(n), TE_THREADS, 0, st, s->tab.as<b2_twoview_eval_problem>(), thr * thr, s->out.as<TeOut>());
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaMemcpyAsync(s->hout.p, s->out.p, ob, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  const TeOut* ho = s->hout.as<TeOut>();
  for (int i = 0; i < n; ++i) {
    b2_twoview_eval_result& r = results[i];
    const TeOut& o = ho[i];
    r.num_rows = o.num_rows, r.num_inliers_gt = o.num_inliers, r.no_gt = o.no_gt, r.no_rows = o.no_rows;
    r.inlier_avg_reproj_error_gt = o.inlier_avg, r.outlier_avg_reproj_error_gt = o.outlier_avg;
    r.R_error_deg = o.R_error_deg, r.U_error_deg = o.U_error_deg;
  }
  return B2_OK;
}
