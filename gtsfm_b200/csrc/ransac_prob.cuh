// The RANSAC verifier's problem record (ransac.cu), shared with the LMedS verifier (lmeds.cu), which launches ransac.cu's
// gather and pose kernels on a table of these records.
#pragma once
#include "common.cuh"

// best-model record kept on the device between rounds (the header's b2_ransac_candidate, so traces copy it as is)
using RsBest = b2_ransac_candidate;

// One problem as the kernels see it.  The host keeps the table of a sub-batch in pinned memory and uploads it once for the
// stages that run on every problem (gather, refine, pick, mask, pose) and once per sampling round, compacted to the problems
// that run the round, with the round fields set.
struct RsProb {
  const float *kp1, *kp2;     // k_rs_gather's input (null: x1 / x2 are ready)
  const long long* matches;
  double g1[3], g2[3];        // f, u0, v0 applied by k_rs_gather
  double *x1, *x2;            // [k][2] points every later stage reads
  int k, mode;                // mode 0 = essential (5-point, Sampson), 1 = fundamental (8-point, epiline)
  double thr2;
  // ---- this sampling round
  int sample0, n;             // counter of the first sample, samples drawn
  const int* go;              // extension stage: the round's kernels return at once unless *go
  int* more;                  // where k_rs_select writes "the confidence bound needs more than done_after samples" (null: nowhere)
  double done_after;
  // ---- the problem's slices of the workspace
  double* models;
  int* nsol;
  double* cost;
  int* ninl;
  RsBest *cand, *best;        // RS_TOP candidates, the result
  int* count;                 // inliers counted by k_rs_mask
  uint8_t* mask;
  // ---- pose recovery
  const double* E;            // the essential matrix, or (pose_cal) the fundamental matrix it is formed from
  const uint8_t* pose_mask;   // null: every point votes
  int* gvotes;                // [4] votes + [1] CTA counter, zero on entry
  double* pose;               // R[9], t[3], votes of the winner
  double* pose_cands;         // R1[9], R2[9], t[3], winner (tests only, else null)
  int pose_on, pose_cal;      // pose_cal: x1 / x2 are pixels, E = K2^T F K1 and the points are calibrated with c1 / c2
  double c1[3], c2[3];
};

constexpr int RS_POSE_THREADS = 128;
// defined in ransac.cu
__global__ void k_rs_gather(const RsProb* __restrict__ tab);
__global__ void k_rs_pose(const RsProb* __restrict__ tab);
