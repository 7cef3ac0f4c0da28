"""Cost of data association's triangulation on the device -> profiles/h100_data_assoc.json (or --out).

For a seeded scene of 500 cameras (5 without a pose) and 500 000 tracks, lengths geometric (p 0.3) from 2 capped at 100,
10 % outlier measurements, with deep_front_end.yaml's options (RANSAC_SAMPLE_UNIFORM, 10 px, 100 hypotheses) and with
NO_RANSAC:
  * call_ms: a host clock around B200DataAssociation.triangulate_arrays (uploads, every launch, the copies back and the
    synchronisations), median of --reps after warm-up; tracks/s and hypotheses/s from it;
  * kernel_ms: the summed CUDA-event time of the k_da_hyp and of the k_da_track launches of one call, and their number;
  * pack_ms / unpack_ms: the host conversion of the SfmTrack2d list into the call's arrays, and of its results into the
    reference's three lists;
  * the CPU arm: the reference's per-track loop as oracle/data_assoc_ref.py restates it, timed on this host on a seeded
    subsample of tracks and scaled to all of them (labelled as such).

  * lund-door: the same figures (call and kernel time) for the 672 tracks of tests/golden/data_assoc_lund_door.npz.

    python profiles/bench_data_assoc.py [--out path] [--reps N] [--tracks T] [--cpu-subsample S]
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_data_assoc.json"))
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--tracks", type=int, default=500_000)
    ap.add_argument("--cpu-subsample", type=int, default=1000)
    a = ap.parse_args()
    import torch

    from gtsfm_b200 import _lib
    from gtsfm_b200.data_association import B200DataAssociation, pack_tracks, unpack
    from gtsfm_b200.gtsfm_api import SfmMeasurement, SfmTrack2d, TriangulationOptions, TriangulationSamplingMode
    from oracle import data_assoc_ref as da
    from oracle.make_golden_data_assoc import geometric_lengths, make_tracks, ring_cameras

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"gpu": gpu_info(), "reps": a.reps}
    rng = np.random.default_rng(5)
    cams = ring_cameras(rng, 500, radius=30.0)
    valid = np.ones(500, np.uint8)
    valid[rng.choice(500, 5, replace=False)] = 0
    lengths = geometric_lengths(rng, a.tracks, 0.3, 2, 100)
    raw = make_tracks(rng, cams, lengths, outlier_frac=0.1)
    tracks2d = [SfmTrack2d([SfmMeasurement(i, uv) for i, uv in t]) for t in raw]
    scene = {"cameras": 500, "cameras_without_pose": 5, "tracks": a.tracks, "measurements": int(lengths.sum()),
             "mean_length": float(lengths.mean()), "max_length": int(lengths.max()), "outlier_frac": 0.1}
    out["scene"] = scene
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        off, img, uv = pack_tracks(tracks2d)
        ts.append((time.perf_counter() - t0) * 1e3)
    out["pack_ms"] = float(np.median(ts))
    ctx = _lib.Context(0)
    modes = {"uniform_10px_100": (TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM, 10.0), "no_ransac_10px": (TriangulationSamplingMode.NO_RANSAC, 10.0)}
    for name, (mode, thr) in modes.items():
        pl = B200DataAssociation(min_track_len=2, triangulation_options=TriangulationOptions(mode, reproj_error_threshold=thr,
                                                                                              max_num_hypotheses=100), ctx=ctx)
        for _ in range(2):
            res = pl.triangulate_arrays(off, img, uv, cams, valid)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            pl.triangulate_arrays(off, img, uv, cams, valid)
            ts.append((time.perf_counter() - t0) * 1e3)
        hyps = int(np.minimum(lengths * (lengths - 1) // 2, 100).sum()) if mode == TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM else 0
        m = {"call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)), "hypotheses": hyps,
             "tracks_per_s": a.tracks / (np.median(ts) / 1e3), "hypotheses_per_s": hyps / (np.median(ts) / 1e3),
             "exit_codes": np.bincount(res[0].astype(np.int64), minlength=6).tolist()}
        for k in ("k_da_hyp", "k_da_track"):
            ctx.profile_start(k)
            pl.triangulate_arrays(off, img, uv, cams, valid)
            ms, launches, _ = ctx.profile_stop()
            m[k] = {"kernel_ms": ms, "launches": launches}
        t0 = time.perf_counter()
        unpack(tracks2d, off, *res)
        m["unpack_ms"] = (time.perf_counter() - t0) * 1e3
        # the CPU arm: the restated reference loop on a seeded subsample, scaled to every track
        pick = np.sort(np.random.default_rng(0).choice(a.tracks, a.cpu_subsample, replace=False))
        t0 = time.perf_counter()
        da.run_arrays(off, img, uv, cams, valid, da.SAMPLE_UNIFORM if hyps else da.NO_RANSAC, 100, thr, 0.0, 0, pick)
        sub = time.perf_counter() - t0
        m["cpu_restated_loop"] = {"subsample_tracks": int(a.cpu_subsample), "subsample_s": sub, "scaled_to_all_s": sub * a.tracks / a.cpu_subsample}
        out[name] = m
        print(name, json.dumps(m), flush=True)
    # lund-door's 672 tracks (tests/golden/data_assoc_lund_door.npz), both modes
    z = np.load(ROOT / "tests/golden/data_assoc_lund_door.npz")
    lund = {}
    for name, (mode, thr) in modes.items():
        pl = B200DataAssociation(min_track_len=2, triangulation_options=TriangulationOptions(mode, reproj_error_threshold=thr,
                                                                                              max_num_hypotheses=100), ctx=ctx)
        args = [z[f"{name}/{k}"] for k in ("track_off", "meas_cam", "meas_uv", "cams", "cam_valid")]
        for _ in range(3):
            pl.triangulate_arrays(*args)
        ts = []
        for _ in range(a.reps * 4):
            t0 = time.perf_counter()
            pl.triangulate_arrays(*args)
            ts.append((time.perf_counter() - t0) * 1e3)
        ctx.profile_start("k_da")
        pl.triangulate_arrays(*args)
        ms, launches, _ = ctx.profile_stop()
        lund[name] = {"tracks": int(len(args[0]) - 1), "call_ms_median": float(np.median(ts)), "kernel_ms": ms, "launches": launches}
    out["lund_door"] = lund
    print("lund_door", json.dumps(lund), flush=True)
    out["gpu_after"] = gpu_info()
    ctx.close()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
