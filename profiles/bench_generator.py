"""B200CorrespondenceGenerator throughput for the detector / matcher configs it serves besides SuperPoint + LightGlue, against
the same work done through the per-image and per-pair plugins.

Configs: SIFT + two-way (ratio 0.8; also what the MegaLoc + SIFT config runs), ORB + two-way, D2-Net + two-way (seeded
weights), SuperPoint + SuperGlue (seeded weights), all at 5000 keypoints.  Workloads: the 12 lund-door frames at loader
resolution (1135 x 760 gray) with all 66 pairs, and 12 seeded 480 x 640 RGB synthetic_sequence frames with all 66 pairs.

Arms, per config and workload (host arrays in, host results out, every call ending in a device synchronisation):
- generator pairs/s: `generate_correspondences` on the whole job, without and with `verify_with` (RANSAC under the matching);
- plugin pairs/s: what DetDescCorrespondenceGenerator issues, replayed in-process without Dask - `detect_and_describe` once per
  image, then `match` once per pair, and (with verification) B200Ransac.verify once per pair.
Each arm is warmed up once and timed over --reps repetitions; the median is reported.  The intrinsics are a pinhole guess
(f = 0.9 W, principal point at the centre) for lund-door and synthetic_sequence's own for the synthetic frames.  The card name
and power limit are read in the same run.  Writes one JSON line to --out.

    python profiles/bench_generator.py --out profiles/h100_generator.json
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

K = 5000
RATIO = 0.8
CONFIGS = ("sift", "orb", "d2net", "superpoint_superglue")


def _objects(config):
    """-> (generator, detector plugin, matcher plugin) sharing nothing: each builds its own device state."""
    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator
    from gtsfm_b200.detector_descriptor import (B200D2NetDetectorDescriptor, B200ORBDetectorDescriptor, B200SIFTDetectorDescriptor,
                                                B200SuperPointDetectorDescriptor)
    from gtsfm_b200.matcher import B200SuperGlueMatcher, B200TwoWayMatcher

    if config == "superpoint_superglue":
        sp, sg = syn.superpoint_state_dict(0), syn.superglue_state_dict(1, "sharp")
        return (B200CorrespondenceGenerator(sp, max_keypoints=K, matcher="superglue", superglue_weights=sg),
                B200SuperPointDetectorDescriptor(max_keypoints=K, weights_path=sp), B200SuperGlueMatcher(weights_path=sg))
    twoway = B200TwoWayMatcher(ratio_test_threshold=RATIO)
    if config == "d2net":
        d2 = syn.d2net_state_dict(7)
        return (B200CorrespondenceGenerator(max_keypoints=K, detector="d2net", matcher="twoway", d2net_weights=d2, ratio_test_threshold=RATIO),
                B200D2NetDetectorDescriptor(max_keypoints=K, model_path=d2), twoway)
    plugin = (B200SIFTDetectorDescriptor if config == "sift" else B200ORBDetectorDescriptor)(max_keypoints=K)
    return B200CorrespondenceGenerator(max_keypoints=K, detector=config, matcher="twoway", ratio_test_threshold=RATIO), plugin, twoway


def _median_s(fn, reps):
    fn()  # warm-up: module loads, workspaces, lanes
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return statistics.median(times)


def workload(name, frames, intr, config, reps):
    from gtsfm_b200.gtsfm_api import Cal3Bundler, Image
    from gtsfm_b200.verifier import B200Ransac

    images = [Image(f) for f in frames]
    pairs = [(i, j) for i in range(len(frames)) for j in range(i + 1, len(frames))]
    gen, det, mat = _objects(config)
    ver = B200Ransac(True, 4.0)
    cals = {i: Cal3Bundler(c[0], 0.0, 0.0, c[1], c[2]) for i, c in intr.items()}
    out = {}

    def generator(verify):
        out["gen"] = gen.generate_correspondences(None, images, pairs, verify_with=(intr, 4.0) if verify else None)

    def plugins(verify):
        feats = [det.detect_and_describe(im) for im in images]
        ms = {}
        for i1, i2 in pairs:
            (k1, d1), (k2, d2) = feats[i1], feats[i2]
            ms[(i1, i2)] = m = mat.match(k1, k2, d1, d2, frames[i1].shape, frames[i2].shape)
            if verify:
                ver.verify(k1, k2, m.reshape(-1, 2), cals[i1], cals[i2])
        out["plugin"] = ms

    row = {"workload": name, "config": config, "frames": len(frames), "frame": list(frames[0].shape), "pairs": len(pairs)}
    for verify in (False, True):
        tag = "match_verify" if verify else "match"
        row[f"generator_{tag}_pairs_per_s"] = round(len(pairs) / _median_s(lambda: generator(verify), reps), 1)
        row[f"plugin_{tag}_pairs_per_s"] = round(len(pairs) / _median_s(lambda: plugins(verify), reps), 1)
        row[f"generator_vs_plugin_{tag}"] = round(row[f"generator_{tag}_pairs_per_s"] / row[f"plugin_{tag}_pairs_per_s"], 2)
    kps, matches = out["gen"]
    row["mean_kp"] = float(np.mean([len(k) for k in kps]))
    row["mean_matches"] = float(np.mean([len(m) for m in matches.values()]))
    row["plugin_mean_matches"] = float(np.mean([len(m) for m in out["plugin"].values()]))
    row["verified_pairs"] = sum(r.i2Ri1 is not None for r in gen.last_two_view.values())
    row["generator_last_timing_s"] = {k: round(v, 4) for k, v in gen.last_timing.items()}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_generator.json"))
    a = ap.parse_args()

    import torch

    from gtsfm_b200 import synthetic as syn

    if not torch.cuda.is_available():
        raise SystemExit("bench_generator.py measures the GPU path and needs a CUDA device")
    lund = np.load(ROOT / "tests" / "golden" / "lund_door_images.npz")
    lund_frames = [lund[f"gray_{i}"] for i in range(1, 13)]
    h, w = lund_frames[0].shape
    lund_intr = {i: (0.9 * w, w / 2.0, h / 2.0) for i in range(12)}
    synth_frames, cal = syn.synthetic_sequence(12, 480, 640)
    synth_intr = {i: cal for i in range(12)}
    rows = []
    for config in a.configs.split(","):
        rows.append(workload("lund_door_loader", lund_frames, lund_intr, config, a.reps))
        rows.append(workload("synthetic_480x640", synth_frames, synth_intr, config, a.reps))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    line = {"workload": "correspondence_generator", "max_keypoints": K, "ratio": RATIO, "reps": a.reps, "results": rows,
            "gpu": name, "power_limit": power}
    s = json.dumps(line)
    print(s)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(s + "\n")


if __name__ == "__main__":
    main()
