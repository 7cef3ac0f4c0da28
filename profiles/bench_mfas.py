"""Cost of 1DSfM's outlier rejection on the device -> profiles/h100_mfas.json (or --out).

For seeded kNN scenes (oracle.make_golden_mfas.large_scene: k = 30, 20 % outlier camera directions, about 12 track
directions per camera) of 500, 2000 and 5000 cameras, with K = 2000 uniform projection directions:
  * call_ms: a host clock around outlier_weights_arrays (uploads, every launch, the copy back, the synchronisation), median
    of --reps after warm-up;
  * kernel_ms: the summed CUDA-event time of the k_mfas_order and of the k_mfas_sum launches of one call;
  * convert_ms: the host conversion of the {pair: Unit3} dicts into the call's arrays (dense_edges and the vectors);
  * the CPU arm: oracle/mfas_ref.order_vectorised (the restated greedy, one argmax per step) on --cpu-dirs directions, scaled
    to K (labelled as such).  gtsam's own C++ MFAS is not run here, and its time is not estimated.

    python profiles/bench_mfas.py [--out path] [--reps N] [--cpu-dirs D]
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


def gpu_info() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_mfas.json"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-dirs", type=int, default=4)
    ap.add_argument("--cameras", default="500,2000,5000")
    a = ap.parse_args()
    import torch

    from gtsfm_b200 import _lib
    from gtsfm_b200.gtsfm_api import Unit3
    from gtsfm_b200.translation_averaging import _vectors, dense_edges, outlier_weights_arrays
    from oracle import mfas_ref as mr
    from oracle.make_golden_mfas import large_scene

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"gpu": gpu_info(), "reps": a.reps, "directions": 2000, "scenes": {}}
    ctx = _lib.Context(0)
    for n in (int(x) for x in a.cameras.split(",")):
        cam, trk = large_scene(n)
        cu, tu = {k: Unit3(v) for k, v in cam.items()}, {k: Unit3(v) for k, v in trk.items()}
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            V, ea, eb, perm = dense_edges(cu, tu)
            meas = _vectors(list(cu.values()) + list(tu.values()))[perm]
            ts.append((time.perf_counter() - t0) * 1e3)
        m = {"cameras": n, "nodes": int(V), "camera_edges": len(cam), "track_edges": len(trk), "convert_ms": float(np.median(ts))}
        np.random.seed(0)
        dirs = mr.unit3(np.random.normal(size=(2000, 3)))
        for _ in range(2):
            s = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            s2 = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs)
            ts.append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(s.view(np.uint64), s2.view(np.uint64))
        m["call_ms_median"], m["call_ms_min"] = float(np.median(ts)), float(np.min(ts))
        for k in ("k_mfas_order", "k_mfas_sum"):
            ctx.profile_start(k)
            outlier_weights_arrays(ctx, V, ea, eb, meas, dirs)
            ms, launches, _ = ctx.profile_stop()
            m[k] = {"kernel_ms": ms, "launches": launches}
        m["outlier_edges"] = int((s / 2000 >= mr.OUTLIER_WEIGHT_THRESHOLD).sum())
        inc = mr.incidence(V, ea, eb)
        t0 = time.perf_counter()
        for d in dirs[:a.cpu_dirs]:
            mr.order_vectorised(V, ea, eb, meas, d, inc)
        sub = time.perf_counter() - t0
        m["cpu_restated_greedy"] = {"directions": a.cpu_dirs, "s": sub, "scaled_to_2000_s": sub * 2000 / a.cpu_dirs}
        out["scenes"][str(n)] = m
        print(n, json.dumps(m), flush=True)
    out["gpu_after"] = gpu_info()
    ctx.close()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
