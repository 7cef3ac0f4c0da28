"""Two-view refinement throughput (triangulation + two-view bundle adjustment + inlier support, csrc/twoview_ba.cu).

Workloads:
  * lund-door's 66 pairs (the reference-selected SuperPoint keypoints and LightGlue rows of tests/golden/, a stand-in focal
    length of 1.2 x the longer side): verification alone, verification + refinement (B200TwoViewBatch with
    bundle_adjust_2view), and the refinement alone (one b2_twoview_ba_batched_dev call over the verified pairs);
  * seeded 32-pair batches (oracle/make_golden_twoview_ba.synthetic_scene, 10 % outliers among the verified rows) at 200,
    1000 and 3000 verified rows: verification + refinement, and the refinement alone.
Each device arm is warmed and then timed `--reps` times with a host clock around work that ends in a synchronise (median
and spread).  The CPU arm is the NumPy oracle (oracle/twoview_ba_ref.py) on the host CPU, one process, on a few pairs
of each workload: gtsam is not a dependency of this project, so gtsam's own per-pair cost is NOT measured.  Launches per refinement call
are counted by the library.  The card's name and power limit are read in the same run.  Writes one JSON object to --out.

    python profiles/bench_twoview_ba.py --out profiles/h100_twoview_ba.json
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _timed(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def _rate(n, t):
    return dict(pairs_per_s=n / t[0], median_s=t[0], min_s=t[1], max_s=t[2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-pairs", type=int, default=4)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_twoview_ba.json"))
    a = ap.parse_args()
    import torch

    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd, RefineOptions
    from gtsfm_b200.two_view import B200TwoViewBatch
    from oracle import make_golden_twoview_ba as mg
    from oracle import twoview_ba_ref as ref

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), max_keypoints=64)
    out = dict(gpu=gpu, reps=a.reps, cpu_arm="NumPy oracle, one host process; gtsam's per-pair cost is not measured")

    # lund-door, 66 pairs
    golden = ROOT / "tests" / "golden"
    img = np.load(golden / "lund_door_images.npz")
    fx = np.load(golden / "lund_door_66pairs.npz")
    h, w = img["gray_1"].shape
    cal = (1.2 * max(h, w), w / 2.0, h / 2.0)
    feats, kps = {}, {}
    for i in range(1, 13):
        kp = img[f"kp_{i}"].astype(np.float32)[img[f"sel_{i}"]]
        kps[i] = kp
        feats[i] = DeviceFeatures(torch.from_numpy(kp).cuda(), torch.zeros(len(kp), device="cuda"),
                                  torch.zeros((len(kp), 1), device="cuda"), (h, w))
    pairs = [(p, q) for p in range(1, 13) for q in range(p + 1, 13)]
    put = {pq: torch.from_numpy(fx[f"m_{pq[0]}_{pq[1]}"].astype(np.int64)).cuda() for pq in pairs}
    intr = {i: cal for i in feats}
    off, on = B200TwoViewBatch(fe, 4.0), B200TwoViewBatch(fe, 4.0, bundle_adjust_2view=True)
    lund = dict(pairs=len(pairs), verify=_rate(len(pairs), _timed(lambda: off.run(feats, pairs, intr, put), a.reps)),
                verify_refine=_rate(len(pairs), _timed(lambda: on.run(feats, pairs, intr, put), a.reps)))
    items = [(feats[p], feats[q], put[(p, q)], cal, cal) for p, q in pairs]
    ver = fe.verify_many(items)
    torch.cuda.synchronize()
    opts = RefineOptions()
    ctx = fe.ctx
    n0 = ctx.launch_count()
    fe.refine_many(items, ver, opts)
    lund["launches_per_refine_call"] = ctx.launch_count() - n0
    lund["refine"] = _rate(len(pairs), _timed(lambda: fe.refine_many(items, ver, opts), a.reps))
    res = on.run(feats, pairs, intr, put)
    lund["pairs_kept"] = sum(r.i2Ri1 is not None for r in res.values())
    pre = off.run(feats, pairs, intr, put)
    done = 0
    for p in pairs[:: max(1, len(pairs) // a.oracle_pairs)][: a.oracle_pairs]:
        v = pre[p]
        if v.i2Ri1 is None:
            continue
        m = put[p].cpu().numpy()
        row_of = {tuple(x): j for j, x in enumerate(m)}
        verified = np.array(sorted(row_of[tuple(x)] for x in v.v_corr_idxs), np.int64)
        t1 = time.perf_counter()
        ref.refine_pair(kps[p[0]][m[:, 0]].astype(np.float64), kps[p[1]][m[:, 1]].astype(np.float64), verified, len(m), cal, cal,
                        v.i2Ri1.matrix(), v.i2Ui1.point3())
        done += 1
        lund.setdefault("oracle_s_per_pair", []).append(time.perf_counter() - t1)
    if done:
        lund["oracle_pairs_per_s"] = done / sum(lund["oracle_s_per_pair"])
    out["lund_door_66"] = lund

    # seeded 32-pair batches
    out["seeded"] = {}
    for n in (200, 1000, 3000):
        scenes = [mg.synthetic_scene(seed=100 + s, n=n, outlier_frac=0.1) for s in range(32)]
        items, vers = [], []
        for s in scenes:
            k = int(s["k"])
            fa = DeviceFeatures(torch.from_numpy(s["uv1"].astype(np.float32)).cuda(), torch.zeros(k, device="cuda"),
                                torch.zeros((k, 1), device="cuda"), (480, 640))
            fb = DeviceFeatures(torch.from_numpy(s["uv2"].astype(np.float32)).cuda(), torch.zeros(k, device="cuda"),
                                torch.zeros((k, 1), device="cuda"), (480, 640))
            m = torch.arange(k, device="cuda", dtype=torch.int64)[:, None].repeat(1, 2).contiguous()
            mask = torch.zeros(k, dtype=torch.uint8, device="cuda")
            mask[torch.from_numpy(s["verified"]).cuda()] = 1
            items.append((fa, fb, m, tuple(s["cal1"]), tuple(s["cal2"])))
            vers.append((np.eye(3), s["R0"], s["t0"], len(s["verified"]), mask))
        row = dict(refine=_rate(32, _timed(lambda: fe.refine_many(items, vers, opts), a.reps)))

        def both():
            v = fe.verify_many(items)
            return fe.refine_many(items, v, opts)

        row["verify_refine"] = _rate(32, _timed(both, a.reps))
        res = fe.refine_many(items, vers, opts)
        row["pairs_kept"] = sum(r[0] is not None for r in res)
        row["mean_iterations"] = float(np.mean([r[3].iterations for r in res if r[3] is not None]))
        ts = []
        for s in scenes[: max(1, a.oracle_pairs // (1 if n < 3000 else 2))]:
            t1 = time.perf_counter()
            mg.run_oracle(s)
            ts.append(time.perf_counter() - t1)
        row["oracle_pairs_per_s"] = len(ts) / sum(ts)
        out["seeded"][str(n)] = row
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
