"""Cost of the two-view reports' ground-truth evaluation on the GPU -> profiles/h100_twoview_report.json (or --out).

  * B200TwoViewBatch.run on lund-door's 66 pairs with and without ground-truth cameras, BA off and on, alternated in one
    process (the added cost of evaluation);
  * k_tv_eval alone (b2_twoview_eval_batched_dev) on 32-pair batches of 200, 1000 and 3000 rows, pre-BA stage;
  * the NumPy oracle per pair (the only CPU figure: gtsam is not a dependency, so gtsam's own cost is not measured).

    python profiles/bench_twoview_report.py [--out path] [--reps N]
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_twoview_report.json"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch

    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd, EvalUnit
    from gtsfm_b200.two_view import B200TwoViewBatch
    from oracle import make_golden_twoview_report as mg
    from oracle.make_golden_twoview_ba import lund_inputs, synthetic_scene

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    info = gpu_info()
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), max_keypoints=64)
    d = np.load(ROOT / "tests" / "golden" / "twoview_report_lund_door.npz")
    pairs = [tuple(int(x) for x in p) for p in d["pairs"]]
    feats = {}
    for i in range(1, 13):
        k = torch.from_numpy(np.ascontiguousarray(d[f"kp_{i}"])).cuda()
        feats[i] = DeviceFeatures(k, torch.zeros(len(k), device="cuda"), torch.zeros((len(k), 1), device="cuda"), (0, 0))
    putative = {p: torch.from_numpy(d[f"{p[0]}_{p[1]}/putative"]).cuda() for p in pairs}
    cams = {}
    for p in pairs:
        cams[p[0]], cams[p[1]] = mg.cam_from_vec(d[f"{p[0]}_{p[1]}/cam1"]), mg.cam_from_vec(d[f"{p[0]}_{p[1]}/cam2"])
    cal = lund_inputs()[3]
    intr = {i: cal for i in range(1, 13)}
    out = {"gpu": info, "pairs": len(pairs), "reps": a.reps}
    for ba in (False, True):
        tvb = B200TwoViewBatch(fe, 4.0, bundle_adjust_2view=ba)
        times = {"off": [], "on": []}
        for _ in range(3):
            tvb.run(feats, pairs, intr, putative)
            tvb.run(feats, pairs, intr, putative, gt_cameras=cams)
        for _ in range(a.reps):
            for mode in ("off", "on"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tvb.run(feats, pairs, intr, putative, gt_cameras=cams if mode == "on" else None)
                torch.cuda.synchronize()
                times[mode].append((time.perf_counter() - t0) * 1e3)
        out[f"run_ba_{'on' if ba else 'off'}_ms"] = {m: {"median": float(np.median(v)), "min": float(np.min(v))} for m, v in times.items()}
        out[f"run_ba_{'on' if ba else 'off'}_added_ms_median"] = float(np.median(times["on"]) - np.median(times["off"]))
    # k_tv_eval alone: 32 pairs of n rows (all verified), timed with CUDA events around the call
    kern = {}
    for n in (200, 1000, 3000):
        units = []
        for s in range(32):
            sc = synthetic_scene(100 + s, n, outlier_frac=0.1, n_unverified=0)
            kp1 = torch.from_numpy(sc["uv1"].astype(np.float32)).cuda()
            kp2 = torch.from_numpy(sc["uv2"].astype(np.float32)).cuda()
            m = torch.from_numpy(np.stack([np.arange(n), np.arange(n)], 1)).cuda()
            mask = torch.ones(n, dtype=torch.uint8, device="cuda")
            R, t = sc["R_true"], sc["t_true"]
            units.append(EvalUnit(kp1, kp2, m, mask, (sc["R0"], sc["t0"]), (np.eye(3), np.zeros(3), *sc["cal1"]),
                                  (R.T, -R.T @ t, *sc["cal2"])))
        for _ in range(5):
            fe.evaluate_many(units)
        ts = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fe.evaluate_many(units)
            ts.append((time.perf_counter() - t0) * 1e3)
        ctx = fe.ctx
        ctx.profile_start("k_tv_eval")
        for _ in range(a.reps):
            fe.evaluate_many(units)
        ms, launches, _ = ctx.profile_stop()
        kern[str(n)] = {"call_ms_median": float(np.median(ts)), "kernel_ms_per_launch": ms / max(1, launches), "launches": launches,
                        "pairs_per_s_call": 32 / (np.median(ts) / 1e3)}
    out["k_tv_eval_32_pairs"] = kern
    # the NumPy oracle per pair (pre + post stages of every lund-door pair)
    t0 = time.perf_counter()
    for name in (f"{p[0]}_{p[1]}" for p in pairs):
        mg.unit_reports(mg.load_unit(d, name))
    out["numpy_oracle_ms_per_pair"] = (time.perf_counter() - t0) * 1e3 / len(pairs)
    out["gpu_after"] = gpu_info()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
