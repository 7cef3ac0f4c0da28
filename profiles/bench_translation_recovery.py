"""Cost of 1DSfM's translation recovery on the device -> profiles/h100_translation_recovery.json (or --out).

For seeded kNN scenes (oracle.make_golden_mfas.large_scene: k = 30, 20 % outlier camera directions, about 12 track
directions per camera) of 500, 2000 and 5000 cameras, Huber on, scale 1, the initial values from a fresh std::mt19937(42):
  * call_ms: a host clock around recover_arrays (uploads, the structure sort, every trial, the copy back), median of
    --reps after one warm-up call, with the call's trials and iterations;
  * per_trial_kernel_ms: the CUDA-event time of each kernel of one call capped at 3 iterations, over its trials;
  * workspace_bytes: b2_translation_recovery_workspace_bytes;
  * the host arm: oracle/translation_recovery_ref.recover (the NumPy restatement, Schur then dense Cholesky) on the scenes
    of at most --host-max cameras.  gtsam's own TranslationRecovery is not run here, and its time is not estimated.

    python profiles/bench_translation_recovery.py [--out path] [--reps N] [--host-max C]
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

KERNELS = ("k_tr_lin", "k_tr_lmk", "k_tr_blocks", "k_tr_diag", "k_tr_rhs", "k_chol_diag", "k_chol_panel", "k_chol_update",
           "k_trsv_fwd", "k_trsv_bwd", "k_tr_nodes", "k_tr_edges", "k_tr_reduce")


def gpu_info() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_translation_recovery.json"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-max", type=int, default=500)
    ap.add_argument("--cameras", default="500,2000,5000")
    a = ap.parse_args()
    import torch

    from gtsfm_b200 import _lib
    from gtsfm_b200 import translation_averaging as ta
    from oracle import translation_recovery_ref as tr
    from oracle.make_golden_mfas import large_scene

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"gpu": gpu_info(), "reps": a.reps, "scenes": {}}
    ctx = _lib.Context(0)
    for n in (int(x) for x in a.cameras.split(",")):
        cam, trk = large_scene(n)
        cams, tracks, ea, eb, meas = ta.translation_graph(cam, trk)
        C, L = len(cams), len(tracks)
        ta.reseed_translation_rng()
        x0 = ta.initial_values(ea, eb, C + L)
        m = {"cameras": C, "landmarks": L, "camera_edges": len(cam), "track_edges": len(trk),
             "workspace_bytes": ta.recovery_workspace_bytes(C, L, ea, eb)}
        d = ta.recover_arrays(ctx, C, L, ea, eb, meas, x0, trace=True)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            d2 = ta.recover_arrays(ctx, C, L, ea, eb, meas, x0)
            ts.append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(d["x"], d2["x"])
        m.update(call_ms_median=float(np.median(ts)), call_ms_min=float(np.min(ts)), trials=len(d["trials"]),
                 iterations=d["iterations"], initial_error=float(d["trace"][0]), final_error=d["final_error"])
        per = {}
        for k in KERNELS:
            ctx.profile_start(k)
            p = ta.recover_arrays(ctx, C, L, ea, eb, meas, x0, max_iters=3, trace=True)
            ms, launches, _ = ctx.profile_stop()
            per[k] = {"ms_per_trial": ms / len(p["trials"]), "launches": launches, "trials": len(p["trials"])}
        m["per_trial_kernel_ms"] = per
        if n <= a.host_max:
            pr = tr.Problem(C, L, ea, eb, meas)
            t0 = time.perf_counter()
            r = tr.recover(pr, x0)
            m["host_numpy_restatement"] = {"s": time.perf_counter() - t0, "trials": len(r.trials),
                                           "same_trials_as_device": r.trials == list(d["trials"]),
                                           "final_error_rel_diff": abs(r.final_error - d["final_error"]) / abs(r.final_error)}
        out["scenes"][str(n)] = m
        print(n, json.dumps(m), flush=True)
    out["gpu_after"] = gpu_info()
    ctx.close()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
