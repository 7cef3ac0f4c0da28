"""ORB detector-descriptor throughput on bench_sift.py's two workloads: the 12 lund-door frames at loader resolution
(1135 x 760 gray) and 21 seeded 2880 x 3840 RGB synthetic_sequence frames.

Arms, per workload:
- images/s of the batched device path (OrbEngine.extract_many, top 5000, images already on the GPU), of the plugin on host
  arrays (B200ORBDetectorDescriptor.detect_and_describe) and of the reference's cv2 ORB (oracle/orb_ref.py) with one
  single-threaded process per host core;
- pairs/s of the whole ORB front end on sequential pairs: device detect -> TwoWayEngine.match_batched_dev at ratio 0.8, against
  cv2 ORB on every frame plus cv2 two-way matching of every pair, on every core;
- device time per stage (CUDA events around the k_orb_* launches), and for the stages that stream whole byte planes the bytes
  they must move, computed from the shapes, over their time as a share of the H100 SXM's 3.35 TB/s.
The card name and power limit are read in the same run.  Writes one JSON line to --out.

    python profiles/bench_orb.py --out profiles/h100_orb.json
"""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HBM_TBS = 3.35  # H100 SXM data sheet
STAGES = ("k_orb_gray", "k_orb_resize", "k_orb_fast", "k_orb_nms", "k_orb_blur", "k_orb_select", "k_orb_finish", "k_orb_describe")


def stage_bytes(h: int, w: int, channels: int) -> dict:
    """Bytes the plane-streaming stages must read and write for one image (every plane pixel once per read or write)."""
    from oracle.orb_ref import level_sizes

    p = [lh * lw for lh, lw in level_sizes(h, w)]
    return {"k_orb_gray": h * w * channels + h * w, "k_orb_resize": sum(p[l - 1] + p[l] for l in range(1, len(p))),
            "k_orb_fast": 2 * sum(p), "k_orb_blur": 2 * sum(p)}


def _cv2_detect(arr):
    import cv2

    cv2.setNumThreads(1)
    from oracle import orb_ref

    return orb_ref.detect_and_describe(arr)[3]


def _cv2_match(args):
    import cv2

    cv2.setNumThreads(1)
    from oracle import twoway_ref

    return len(twoway_ref.twoway_match(args[0], args[1], 0.8)[0])


def workload(name, frames, reps, pool, cores, ctx):
    import torch

    from gtsfm_b200.detector_descriptor import B200ORBDetectorDescriptor, OrbEngine
    from gtsfm_b200.gtsfm_api import Image
    from gtsfm_b200.matcher import TwoWayEngine

    eng, mt = OrbEngine(ctx=ctx), TwoWayEngine(ctx=ctx)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    n, npairs = len(frames), len(frames) - 1

    def front_end():
        out = eng.extract_many(dev, max_keypoints=5000)
        return out, mt.match_batched_dev([(out[i][1], out[i + 1][1]) for i in range(npairs)], 0.8)

    for _ in range(2):
        front_end()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        eng.extract_many(dev, max_keypoints=5000)
    torch.cuda.synchronize()
    dev_ips = reps * n / (time.perf_counter() - t0)
    t0 = time.perf_counter()
    for _ in range(reps):
        out, res = front_end()
    torch.cuda.synchronize()
    dev_pps = reps * npairs / (time.perf_counter() - t0)
    stage_ms = {}
    for st in STAGES:
        ctx.profile_start(st)
        for _ in range(reps):
            eng.extract_many(dev, max_keypoints=5000)
        ms, launches, _ = ctx.profile_stop()
        stage_ms[st] = round(ms / (reps * n), 4)
    h, w = frames[0].shape[:2]
    ch = 1 if frames[0].ndim == 2 else frames[0].shape[2]
    sb = stage_bytes(h, w, ch)
    tbs = {k: round(v / (stage_ms[k] * 1e-3) / 1e12, 3) for k, v in sb.items() if stage_ms[k] > 0}

    det = B200ORBDetectorDescriptor(max_keypoints=5000)
    det._engine = eng
    det.detect_and_describe(Image(frames[0]))
    plug_reps = max(1, reps // 4)
    t0 = time.perf_counter()
    for _ in range(plug_reps):
        for f in frames:
            det.detect_and_describe(Image(f))
    plugin_ips = plug_reps * n / (time.perf_counter() - t0)

    pool.map(_cv2_detect, frames[: min(n, cores)])
    work = frames * max(1, (2 * cores + n - 1) // n)
    t0 = time.perf_counter()
    pool.map(_cv2_detect, work, chunksize=1)
    cv2_ips = len(work) / (time.perf_counter() - t0)
    t0 = time.perf_counter()
    desc = pool.map(_cv2_detect, frames, chunksize=1)
    counts = pool.map(_cv2_match, [(desc[i], desc[i + 1]) for i in range(npairs)], chunksize=1)
    cv2_pps = npairs / (time.perf_counter() - t0)
    return {"workload": name, "frames": n, "frame": list(frames[0].shape), "mean_kp": float(np.mean([len(o[0]) for o in out])),
            "mean_total_kp": float(np.mean([o[2] for o in out])), "mean_matches": float(np.mean([len(m) for m in res])),
            "cv2_mean_matches": float(np.mean(counts)), "batched_dev_images_per_s": round(dev_ips, 1),
            "plugin_host_images_per_s": round(plugin_ips, 1), "cv2_images_per_s": round(cv2_ips, 2),
            "batched_vs_cv2": round(dev_ips / cv2_ips, 1), "front_end_dev_pairs_per_s": round(dev_pps, 1),
            "cv2_front_end_pairs_per_s": round(cv2_pps, 2), "front_end_vs_cv2": round(dev_pps / cv2_pps, 1),
            "stage_ms_per_image": stage_ms, "stage_bytes_per_image": sb, "stage_tb_per_s": tbs,
            "stage_share_hbm_peak": {k: round(v / HBM_TBS, 3) for k, v in tbs.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--synthetic-frames", type=int, default=21)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_orb.json"))
    a = ap.parse_args()

    from gtsfm_b200 import _lib
    from gtsfm_b200 import synthetic as syn

    lund = np.load(ROOT / "tests" / "golden" / "lund_door_images.npz")
    lund_frames = [lund[f"gray_{i}"] for i in range(1, 13)]
    synth_frames = syn.synthetic_sequence(a.synthetic_frames, 2880, 3840)[0]
    ctx = _lib.Context(0)
    cores = os.cpu_count() or 1
    with mp.get_context("spawn").Pool(cores) as pool:  # fresh processes: cv2's thread pool does not survive a fork
        rows = [workload("lund_door_loader", lund_frames, a.reps, pool, cores, ctx), workload("synthetic_12mp", synth_frames, a.reps, pool, cores, ctx)]
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    line = {"workload": "orb", "cv2_cores": cores, "max_keypoints": 5000, "ratio": 0.8, "results": rows, "hbm_peak_tbs": HBM_TBS,
            "gpu": name, "power_limit": power}
    s = json.dumps(line)
    print(s)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(s + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
