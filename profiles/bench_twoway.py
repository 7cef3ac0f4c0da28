"""Two-way matcher throughput: cv2 SIFT (top 5000) on seeded synthetic_sequence frames, sequential pairs, ratio test 0.8.

Arms: the batched device path (TwoWayEngine.match_batched_dev, descriptors already on the GPU), the per-pair plugin
(B200TwoWayMatcher.match on host arrays) and the reference's cv2 two-way matching (oracle/twoway_ref.py, one single-threaded
cv2 process per host core).  Also k_mnn_top2's device time per pair (CUDA events) and its share of the H100 SXM dense INT8
peak (the u8 instance, which runs every pair of this workload; the fp16 instance's skip pass is reported apart), and the card name and power limit read in the same run.  Writes one JSON line to --out.

    python profiles/bench_twoway.py --frames 21 --out profiles/h100_twoway_sift.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import multiprocessing as mp
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

INT8_PEAK_TOPS = 1979.0  # H100 SXM data sheet, dense


def sift_features(n_frames, max_kp, height, width):
    import cv2

    from gtsfm_b200 import synthetic as syn

    frames, _ = syn.synthetic_sequence(n_frames, height, width)
    sift = cv2.SIFT_create(nfeatures=max_kp)
    return [sift.detectAndCompute(cv2.cvtColor(f, cv2.COLOR_RGB2GRAY), None)[1] for f in frames]


def _cv2_pair(args):
    import cv2

    cv2.setNumThreads(1)
    from oracle import twoway_ref

    return len(twoway_ref.twoway_match(args[0], args[1], 0.8)[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=21)
    ap.add_argument("--max-kp", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--height", type=int, default=2880)  # large enough for ~5000 SIFT keypoints per frame
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_twoway_sift.json"))
    a = ap.parse_args()

    import torch

    from gtsfm_b200 import _lib
    from gtsfm_b200.matcher import B200TwoWayMatcher, TwoWayEngine

    desc = sift_features(a.frames, a.max_kp, a.height, a.width)
    print("features", [len(d) for d in desc], flush=True)
    pairs = [(desc[i], desc[i + 1]) for i in range(len(desc) - 1)]
    ctx = _lib.Context(0)
    eng = TwoWayEngine(ctx=ctx)
    dev = [(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()) for x, y in pairs]

    # batched device path
    for _ in range(3):
        eng.match_batched_dev(dev, 0.8)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.reps):
        res = eng.match_batched_dev(dev, 0.8)
    torch.cuda.synchronize()
    batched = a.reps * len(pairs) / (time.perf_counter() - t0)

    # kernel time (separate passes).  Every SIFT pair takes the u8 instance; the fp16 instance is launched too, since the
    # device path learns that the descriptors are integer-valued only on the device, and it skips every pair.
    ctx.profile_start("k_mnn_top2<true>")
    for _ in range(a.reps):
        eng.match_batched_dev(dev, 0.8)
    ms, launches, work = ctx.profile_stop()
    kern_ms_pair = ms / (a.reps * len(pairs))
    share = (work / (ms * 1e-3)) / (INT8_PEAK_TOPS * 1e12) if ms > 0 else 0.0
    ctx.profile_start("k_mnn_top2<false>")
    for _ in range(a.reps):
        eng.match_batched_dev(dev, 0.8)
    ms_skip, _, work_skip = ctx.profile_stop()
    assert work_skip == 0.0, "a SIFT pair took the fp16 path"

    print("batched", batched, "kernel ms/pair", kern_ms_pair, flush=True)
    # per-pair plugin on host arrays
    plug = B200TwoWayMatcher(ratio_test_threshold=0.8)
    plug._engine = eng
    for x, y in pairs[:2]:
        plug.match(None, None, x, y, None, None)
    t0 = time.perf_counter()
    for _ in range(max(1, a.reps // 4)):
        host = [plug.match(None, None, x, y, None, None) for x, y in pairs]
    plugin = max(1, a.reps // 4) * len(pairs) / (time.perf_counter() - t0)
    assert all(np.array_equal(h.astype(np.int64), r.cpu().numpy()) for h, r in zip(host, res))

    print("plugin", plugin, flush=True)
    # the reference's cv2 arm on every host core
    cores = os.cpu_count() or 1
    with mp.get_context("spawn").Pool(cores) as pool:  # fresh processes: cv2's thread pool does not survive a fork
        pool.map(_cv2_pair, pairs[:cores])
        work_items = pairs * max(1, (2 * cores + len(pairs) - 1) // len(pairs))
        t0 = time.perf_counter()
        counts = pool.map(_cv2_pair, work_items, chunksize=1)
        cv2_rate = len(work_items) / (time.perf_counter() - t0)
    assert counts[: len(pairs)] == [len(h) for h in host]

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    line = {"workload": "twoway_sift", "frames": a.frames, "pairs": len(pairs), "max_kp": a.max_kp, "frame": [a.height, a.width], "ratio": 0.8,
            "mean_kp": float(np.mean([len(d) for d in desc])), "mean_matches": float(np.mean([len(h) for h in host])),
            "batched_dev_pairs_per_s": round(batched, 1), "plugin_host_pairs_per_s": round(plugin, 1),
            "cv2_pairs_per_s": round(cv2_rate, 2), "cv2_cores": cores, "batched_vs_cv2": round(batched / cv2_rate, 1),
            "k_mnn_top2_ms_per_pair": round(kern_ms_pair, 4), "k_mnn_top2_launches": launches,
            "k_mnn_top2_tops": round(work / (ms * 1e-3) / 1e12, 1) if ms > 0 else 0.0,
            "k_mnn_top2_share_int8_peak": round(share, 4),
            "k_mnn_top2_fp16_skip_ms_per_pair": round(ms_skip / (a.reps * len(pairs)), 4), "int8_peak_tops": INT8_PEAK_TOPS, "gpu": name, "power_limit": power}
    s = json.dumps(line)
    print(s)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(s + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
