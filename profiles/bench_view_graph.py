"""Cost of the cycle-consistent rotation view-graph filter -> profiles/h100_view_graph.json (or --out).

For seeded k-nearest-neighbour graphs (k = 50, N = 1000, 3000, 8000) and an exhaustive 300-image graph, both criteria:
  * call_ms: a host clock around B200CycleConsistentRotationViewGraphEstimator.filter_arrays (uploads, every launch,
    the copies back and the synchronisation), median of --reps after warm-up;
  * dict_to_arrays_ms: the Python conversion of the {(i1, i2): Rot3} dict `run` receives into the arrays the call takes;
  * kernel_ms: the summed CUDA-event time of the k_vg_* launches of one call, and their number;
  * the CPU figures: the reference's loop as oracle/view_graph_ref.py restates it (dict adjacency, set intersections, one
    scipy rotvec per triplet, one np.median per edge), timed on this host with the per-triplet part measured on a
    subsample of triplets and scaled to all of them (labelled as such), and the vectorised NumPy oracle on the whole graph.

    python profiles/bench_view_graph.py [--out path] [--reps N]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def gpu_info() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def reference_loop_cpu_s(edges, R, subsample: int = 20000) -> dict:
    """The restated reference loop: triplet extraction in full, the per-triplet cycle error on `subsample` triplets scaled
    to all, the per-edge np.median in full."""
    from oracle import view_graph_ref as ref

    pairs = [(int(a), int(b)) for a, b in edges]
    rot = {p: r for p, r in zip(pairs, R)}
    t0 = time.perf_counter()
    T = ref.triplets_literal(pairs)
    t_extract = time.perf_counter() - t0
    rng = np.random.default_rng(0)
    pick = rng.choice(len(T), min(subsample, len(T)), replace=False)
    per_edge = defaultdict(list)
    t0 = time.perf_counter()
    for i in pick:
        i0, i1, i2 = T[i]
        err = ref.cycle_error_deg(rot[(i0, i1)], rot[(i1, i2)], rot[(i0, i2)])
        per_edge[(i0, i1)].append(err)
        per_edge[(i1, i2)].append(err)
        per_edge[(i0, i2)].append(err)
    t_err = (time.perf_counter() - t0) * len(T) / len(pick)
    errs = rng.uniform(0.0, 180.0, len(T))  # the aggregation's cost does not depend on the values
    lists = defaultdict(list)
    for (i0, i1, i2), err in zip(T, errs):
        lists[(i0, i1)].append(err)
        lists[(i1, i2)].append(err)
        lists[(i0, i2)].append(err)
    t0 = time.perf_counter()
    for v in lists.values():
        np.median(v)
    t_agg = time.perf_counter() - t0
    return {"extract_s": t_extract, "errors_s_scaled": t_err, "errors_subsample": int(len(pick)), "median_s": t_agg,
            "total_s": t_extract + t_err + t_agg, "us_per_triplet": (t_extract + t_err + t_agg) / len(T) * 1e6}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_view_graph.json"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch

    from gtsfm_b200 import _lib
    from gtsfm_b200.gtsfm_api import Rot3
    from gtsfm_b200.view_graph import B200CycleConsistentRotationViewGraphEstimator as Est
    from oracle import make_golden_view_graph as mg
    from oracle import view_graph_ref as ref

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"gpu": gpu_info(), "reps": a.reps, "graphs": {}}
    ctx = _lib.Context(0)
    graphs = {f"knn_{n}_k50": mg.knn_edges(n, 50, 40 + n) for n in (1000, 3000, 8000)}
    graphs["exhaustive_300"] = mg.exhaustive_edges(300)
    for name, e in graphs.items():
        R = mg.relative_rotations(e, 7, outlier_frac=0.2)
        g = {"edges": int(len(e))}
        d = {(int(i1), int(i2)): Rot3(r) for (i1, i2), r in zip(e, R)}
        ts = []
        for _ in range(5):
            t0 = time.perf_counter()
            Est.arrays(d)
            ts.append((time.perf_counter() - t0) * 1e3)
        g["dict_to_arrays_ms"] = float(np.median(ts))
        for crit in (ref.MEDIAN, ref.MIN):
            est = Est(crit, ctx=ctx)
            for _ in range(3):
                keep, agg, ncyc = est.filter_arrays(e, R)
            g["triplets"] = int(ncyc.sum()) // 3
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                est.filter_arrays(e, R)
                ts.append((time.perf_counter() - t0) * 1e3)
            ctx.profile_start("k_vg")
            est.filter_arrays(e, R)
            ms, launches, _ = ctx.profile_stop()
            g[crit] = {"call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)), "kernel_ms": ms, "launches": launches,
                       "kept": int(keep.sum())}
        t0 = time.perf_counter()
        ref.run_vectorised(e, R)
        g["numpy_vectorised_oracle_s"] = time.perf_counter() - t0
        g["reference_loop_cpu_restated"] = reference_loop_cpu_s(e, R)
        out["graphs"][name] = g
        print(name, json.dumps(g), flush=True)
    out["gpu_after"] = gpu_info()
    ctx.close()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
