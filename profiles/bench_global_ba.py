"""Cost of the global bundle adjustment on the device -> profiles/h100_global_ba.json (or --out).

Seeded scenes (cameras on a ring looking inward, points in front, tracks of 2-6 views with 10 % outlier measurements,
cameras and points perturbed; HUBER, sigma 1, the Karcher gauge) of about 100 cameras / 50 000 tracks, 500 / 300 000
and 1 500 / 600 000, plus lund-door (tests/golden/global_ba_lund_door.npz):
  * call_ms: a host clock around adjust_arrays (uploads, every launch, the per-trial read-backs), median of --reps after one
    warm-up call, with max_iterations --iters (lund-door: the gtsam default, 100);
  * per trial: the summed CUDA-event time of the assembly kernels (k_gba_point, k_gba_blocks, k_gba_karcher, k_gba_diag,
    k_gba_rhs), of the Cholesky (k_chol_*), and of the rest (k_gba_lin, k_trsv_*, k_gba_cams, k_gba_points, k_gba_reduce,
    k_gba_cost) over one call, divided by its trials;
  * the Cholesky's achieved fp64 rate: (9C)^3 / 3 flops per trial over its time;
  * the host side of the plugin: building the call's arrays from per-track lists and the result's per-track lists, as
    to_values / from_values / filter_landmarks handle them (GtsfmData itself needs gtsam and is not run here);
  * the CPU arm: oracle/global_ba_ref.adjust on lund-door.  gtsam's own time is not measured here, and is not estimated.

    python profiles/bench_global_ba.py [--out path] [--reps N] [--iters K] [--scenes 100x50000,500x300000,1500x600000]
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

ASSEMBLY = ("k_gba_point", "k_gba_blocks", "k_gba_karcher", "k_gba_diag", "k_gba_rhs")
CHOL = ("k_chol_",)
REST = ("k_gba_lin", "k_trsv_", "k_gba_cams", "k_gba_points", "k_gba_reduce", "k_gba_cost")


def gpu_info() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def scene(C, N, seed=0, views=(2, 6)):
    """A large seeded scene, vectorised: -> cams (C, 17), points, track_off, meas_cam, meas_uv."""
    from oracle import global_ba_ref as gb
    from oracle import twoview_ba_ref as tv
    from oracle.make_golden_global_ba import look_at

    rng = np.random.default_rng(seed)
    cams = np.zeros((C, 17))
    ang = 2 * np.pi * np.arange(C) / C
    for a in range(C):
        eye = np.array([20 * np.sin(ang[a]), rng.normal(), -20 * np.cos(ang[a])])
        cams[a, :9], cams[a, 9:12] = look_at(eye, np.zeros(3)).ravel(), eye
        cams[a, 12:] = [rng.uniform(500, 700), 0.0, 0.0, 320.0, 240.0]
    # each track is seen by `k` consecutive cameras around a random one, its point in front of them
    k = rng.integers(views[0], views[1] + 1, size=N)
    a0 = rng.integers(0, C, size=N)
    off = np.zeros(N + 1, np.int64)
    np.cumsum(k, out=off[1:])
    trk = np.repeat(np.arange(N), k)
    step = np.arange(off[-1]) - off[trk]
    mcam = ((a0[trk] + step) % C).astype(np.int32)
    mid = (a0 + (k - 1) / 2.0) * 2 * np.pi / C
    pts = np.stack([8 * np.sin(mid), np.zeros(N), -8 * np.cos(mid)], 1) + rng.normal(size=(N, 3)) * 2.0
    pr = gb.Problem(cams, off, mcam, np.zeros((len(mcam), 2)), gb.Params())
    uv, z, _, _ = gb.project_meas(cams, pts, pr)
    uv += rng.normal(size=uv.shape) * 0.7
    out = rng.random(len(uv)) < 0.1
    uv[out] += rng.uniform(20, 60, size=(out.sum(), 1)) * rng.normal(size=(out.sum(), 2))
    cams_n = cams.copy()
    for a in range(C):
        R, t = tv.retract_pose(cams[a, :9].reshape(3, 3), cams[a, 9:12], rng.normal(size=6) * 0.003)
        cams_n[a, :9], cams_n[a, 9:12] = R.ravel(), t
        cams_n[a, 12] *= 1.0 + 0.005 * rng.normal()
    return cams_n, pts + rng.normal(size=pts.shape) * 0.01, off, mcam, uv


def timed(ctx, fn, prefixes):
    total = 0.0
    for p in prefixes:
        ctx.profile_start(p)
        fn()
        ms, _, _ = ctx.profile_stop()
        total += ms
    return total


def measure(ctx, C, N, iters, reps, label, data=None):
    from gtsfm_b200.bundle_adjustment import B200BundleAdjustmentOptimizer

    cams, pts, off, mcam, uv = data if data is not None else scene(C, N)
    o = B200BundleAdjustmentOptimizer(robust_ba_mode="HUBER", measurement_noise_sigma=1.0, max_iterations=iters, ctx=ctx)
    ctx.set_option("ba_workspace_mb", 16384)
    call = lambda: o.adjust_arrays(cams, pts, off, mcam, uv, trace=True)  # noqa: E731
    r = call()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = call()
        ts.append((time.perf_counter() - t0) * 1e3)
    trials = len(r["trials"])
    asm = timed(ctx, call, ASSEMBLY) / trials
    chol = timed(ctx, call, CHOL) / trials
    rest = timed(ctx, call, REST) / trials
    n = 9 * len(cams)
    # the host side of the plugin on per-track lists: packing the call's arrays and splitting the result back per track
    tracks = [(pts[j], [(int(mcam[m]), uv[m]) for m in range(off[j], off[j + 1])]) for j in range(min(len(pts), 100000))]
    t0 = time.perf_counter()
    lens = [len(t[1]) for t in tracks]
    np.array([m[0] for t in tracks for m in t[1]], np.int32), np.array([m[1] for t in tracks for m in t[1]]), np.cumsum(lens)
    pack_ms = (time.perf_counter() - t0) * 1e3 * len(pts) / len(tracks)
    t0 = time.perf_counter()
    from oracle import global_ba_ref as gb

    gb.valid_mask(r["reproj_err"], off, 3.0).tolist()
    [r["points"][j] for j in range(len(tracks))]
    unpack_ms = (time.perf_counter() - t0) * 1e3 * len(pts) / len(tracks)
    return dict(scene=label, cameras=len(cams), tracks=int(len(pts)), measurements=int(len(mcam)), max_iterations=iters,
                iterations=r["iterations"], trials=trials, final_error=r["final_error"], call_ms_median=float(np.median(ts)),
                call_ms_all=ts, trial_ms_assembly=asm, trial_ms_cholesky=chol, trial_ms_rest=rest,
                cholesky_fp64_tflops=(n ** 3 / 3.0) / (chol * 1e-3) / 1e12 if chol > 0 else None,
                host_pack_ms=pack_ms, host_unpack_filter_ms=unpack_ms)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_global_ba.json"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--scenes", default="100x50000,500x300000,1500x600000")
    a = ap.parse_args()
    from gtsfm_b200 import _lib
    from oracle import global_ba_ref as gb
    from oracle.make_golden_global_ba import params_from

    ctx = _lib.Context(0)
    rows = []
    z = np.load(ROOT / "tests/golden/global_ba_lund_door.npz")
    lund = tuple(z["lund_door/" + k] for k in ("cams", "points", "track_off", "meas_cam", "meas_uv"))
    rows.append(measure(ctx, 0, 0, 100, max(a.reps, 5), "lund_door", lund))
    t0 = time.perf_counter()
    gb.adjust(*lund, params_from(z["lund_door/params"]))
    cpu_lund_ms = (time.perf_counter() - t0) * 1e3
    for s in a.scenes.split(","):
        C, N = (int(x) for x in s.split("x"))
        rows.append(measure(ctx, C, N, a.iters, a.reps, s))
        print(json.dumps(rows[-1]), flush=True)
    res = dict(gpu=gpu_info(), rows=rows, oracle_cpu_ms_lund_door=cpu_lund_ms,
               gtsam_ms="not measured (gtsam is not run here)",
               note="call_ms: host clock around one adjust_arrays call; trial_ms_*: CUDA-event kernel time per LM trial")
    Path(a.out).write_text(json.dumps(res, indent=1))
    print(json.dumps(res, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
