"""LMedS verification throughput on seeded oracle.verifier_ref.synthetic_two_view scenes (50 % inliers).

Arms, per shape (E and F at k = 2000, the SuperPoint + LightGlue size, and k = 5000, the SIFT two-way size):
  * device: one b2_lmeds_verify_batched_dev call over 32 problems whose points are already on the device;
  * plugin: B200LMEDS.verify_many over the same 32 pairs from host keypoints (uploads, gather, masks back), E only;
  * cv2: cv2.findEssentialMat / findFundamentalMat with LMEDS, one single-threaded process per host core.
Each arm is warmed and then timed `--reps` times with a host clock around work that ends in a synchronise (median and spread
reported).  Also: device time per stage of one 32-problem call (CUDA events around the k_lm_* / k_rs_* launches), and for
k_lm_score the bytes its shapes require (each live slot reads the k points, 32 B each, once when they fit shared memory and
once per radix pass otherwise) against the bytes per second it achieves, with its 4 selection passes.  The card's name and
power limit are read in the same run.  Writes one JSON line to --out.

    python profiles/bench_lmeds.py --out profiles/h100_lmeds.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from multiprocessing import get_context
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

STAGES = ["k_lm_subsets", "k_lm_hyp", "k_lm_score", "k_lm_select", "k_rs_pose"]
BATCH = 32


def _scene(seed, k, mode):
    from oracle import verifier_ref as vr

    kp1, kp2, m, K, _, _, _ = vr.synthetic_two_view(seed, k, 0.5)
    if mode == 0:
        return vr.calibrate(kp1, *K), vr.calibrate(kp2, *K), kp1, kp2, m, K
    return kp1, kp2, kp1, kp2, m, K


def _cv2_one(args):
    import cv2

    cv2.setNumThreads(1)
    x1, x2, mode = args
    if mode == 0:
        cv2.findEssentialMat(x1, x2, np.eye(3), method=cv2.LMEDS)
    else:
        cv2.findFundamentalMat(x1, x2, method=cv2.FM_LMEDS)
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cv2-pairs", type=int, default=0, help="pairs per cv2 timing (default: 4 per host core)")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_lmeds.json"))
    a = ap.parse_args()

    import torch

    from gtsfm_b200 import _lib
    from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
    from gtsfm_b200.verifier import B200LMEDS, lmeds_verify_batched_dev, ransac_problem

    assert torch.cuda.is_available(), "bench_lmeds measures the device path: no GPU found"
    ctx = _lib.Context(0)
    cores = os.cpu_count() or 1
    n_cv2 = a.cv2_pairs or 4 * cores
    out = {"batch": BATCH, "reps": a.reps, "host_cores": cores, "inlier_ratio": 0.5, "shapes": {}}
    for k in (2000, 5000):
        for mode in (0, 1):
            name = f"{'E' if mode == 0 else 'F'}_k{k}"
            scenes = [_scene(1000 + 7 * i + k, k, mode) for i in range(BATCH)]
            keep, probs = [], []
            for x1, x2, _, _, _, K in scenes:
                d1 = torch.from_numpy(np.ascontiguousarray(x1)).cuda()
                d2 = torch.from_numpy(np.ascontiguousarray(x2)).cuda()
                mk = torch.zeros(k, dtype=torch.uint8, device="cuda")
                keep += [d1, d2, mk]
                probs.append(ransac_problem(k, mode, 0.0, 1000, x1=d1, x2=d2, mask=mk, cal1=K, cal2=K))
            res = {}

            def timed(fn, reps):
                fn()
                torch.cuda.synchronize()
                ts = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    ts.append(time.perf_counter() - t0)
                return ts

            ts = timed(lambda: lmeds_verify_batched_dev(ctx, probs), a.reps)
            res["device_pairs_per_s"] = {"median": BATCH / float(np.median(ts)), "min": BATCH / max(ts), "max": BATCH / min(ts)}
            if mode == 0:
                v = B200LMEDS(use_intrinsics_in_verification=True, estimation_threshold_px=4.0)
                items = []
                for _, _, kp1, kp2, m, K in scenes:
                    cal = Cal3Bundler(K[0], 0.0, 0.0, K[1], K[2])
                    items.append((Keypoints(kp1.astype(np.float32)), Keypoints(kp2.astype(np.float32)), m.astype(np.int64), cal, cal))
                ts = timed(lambda: v.verify_many(items), a.reps)
                res["plugin_pairs_per_s"] = {"median": BATCH / float(np.median(ts)), "min": BATCH / max(ts), "max": BATCH / min(ts)}
            # device time per stage of one call
            stage = {}
            for s in STAGES:
                ctx.profile_start(s)
                lmeds_verify_batched_dev(ctx, probs)
                stage[s] = round(ctx.profile_stop()[0], 4)
            res["stage_ms"] = stage
            # k_lm_score: bytes its shapes require, against what it achieves
            from oracle import lmeds_ref as lr

            niters = lr.niters(lr.E_CONFIDENCE if mode == 0 else lr.F_CONFIDENCE, 5 if mode == 0 else 7)
            lib = ctx.lib
            tr_slots = 0
            for x1, x2, _, _, _, _ in scenes[:4]:  # live slots: solutions per subset, from the trace of four problems
                tr = _lib.LmedsTrace()
                nsol = np.zeros(1024, np.int32)
                tr.cap, tr.nsol = 1024, nsol.ctypes.data
                r = _lib.RansacResult()
                a1, a2 = np.ascontiguousarray(x1), np.ascontiguousarray(x2)
                ctx.check(lib.b2_debug_lmeds_trace_host(ctx.handle, mode, _lib.ptr(a1), _lib.ptr(a2), k, _lib.C.byref(_lmeds_params()),
                                                        1000, _lib.C.byref(tr), _lib.C.byref(r), None), "lmeds_trace")
                tr_slots += int(nsol[:tr.niters].sum())
            live_slots = tr_slots / 4 * BATCH
            reads = 1 if k <= 11264 else 5
            score_bytes = live_slots * k * 32 * reads
            res["score"] = {"subsets_per_problem": niters, "live_slots": live_slots, "selection_passes": 4,
                            "point_reads_per_slot": reads, "bytes": score_bytes,
                            "achieved_GBps": score_bytes / (stage["k_lm_score"] * 1e-3) / 1e9 if stage["k_lm_score"] > 0 else None}
            # cv2, one single-threaded process per host core
            work = [(s[0], s[1], mode) for s in (scenes * (n_cv2 // BATCH + 1))[:n_cv2]]
            with get_context("spawn").Pool(cores) as pool:
                pool.map(_cv2_one, work[:cores])
                t0 = time.perf_counter()
                pool.map(_cv2_one, work, chunksize=1)
                dt = time.perf_counter() - t0
            res["cv2_pairs_per_s"] = {"value": n_cv2 / dt, "processes": cores, "pairs": n_cv2}
            res["bound_stage"] = max(stage, key=stage.get)
            out["shapes"][name] = res
            print(name, json.dumps(res), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    out.update(gpu=name, power_limit=power)
    Path(a.out).write_text(json.dumps(out) + "\n")
    print(json.dumps(out))


def _lmeds_params():
    from gtsfm_b200.verifier import lmeds_params

    return lmeds_params()


if __name__ == "__main__":
    main()
