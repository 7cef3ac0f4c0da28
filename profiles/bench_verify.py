"""RANSAC verification throughput: per pair against one batched call, on seeded oracle.verifier_ref.synthetic_two_view scenes
that are resident on the device.

Arms (E mode), each warmed on every shape and then timed `--reps` times in alternation: `DeviceFrontEnd.verify` in a loop,
the `verify_async` lane (one future per pair), `verify_many` at batch 8 / 32 / 128.  A host clock around work that ends in a
synchronise gives pairs/s; the spread over the repetitions is reported.  F mode (k = 2000): the per-pair host entry
(b2_ransac_fundamental_host + the host pose) against b2_ransac_verify_batched_dev at batch 32.  The outputs of all arms are
compared for equality before a number is printed.  Also: device time per stage of a 32-pair batch (CUDA events around the
k_rs_* launches), launches and stream synchronisations per pair for each arm, and the card's name and power limit read in the
same run.  Writes one JSON line to --out.

    python profiles/bench_verify.py --pairs 256 --out profiles/h100_verify.json
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

STAGES = ["k_rs_gather", "k_rs_hyp_E", "k_rs_score", "k_rs_select", "k_rs_refine", "k_rs_pick", "k_rs_mask", "k_rs_pose"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_verify.json"))
    a = ap.parse_args()

    import torch

    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd
    from gtsfm_b200.verifier import F_MAX_ITERS, RansacEngine, ransac_problem
    from oracle import verifier_ref as vr

    fe = DeviceFrontEnd(syn.superpoint_state_dict(0))
    vlane = fe._verify_lane()
    vctx = vlane.ctx

    def scenes(k, ratio):
        out = []
        for i in range(a.pairs):
            kp1, kp2, _, K, *_ = vr.synthetic_two_view(7000 + i, k, ratio)
            f = [DeviceFeatures(torch.from_numpy(kp.astype(np.float32)).cuda(), torch.zeros(k, device="cuda"), torch.zeros(k, 1, device="cuda"),
                                (960, 1280)) for kp in (kp1, kp2)]
            rows = torch.arange(k, device="cuda", dtype=torch.int64)[:, None].repeat(1, 2).contiguous()
            out.append((f[0], f[1], rows, K, K))
        return out

    def key(r):  # (E, R, t, n, mask) -> comparable bytes
        return None if r[0] is None else (r[0].tobytes(), r[1].tobytes(), r[2].tobytes(), r[3], r[4].cpu().numpy().tobytes())

    def arm_loop(items):
        return [fe.verify(*it, ctx=vctx, stream=vlane.stream) for it in items]

    def arm_async(items):
        return [f.result() for f in [fe.verify_async(*it) for it in items]]

    def arm_many(batch):
        def run(items):
            futs = [fe.verify_many_async(items[c:c + batch]) for c in range(0, len(items), batch)]
            return [r for f in futs for r in f.result()]
        return run

    arms = {"verify_loop": arm_loop, "verify_async": arm_async, "verify_many_8": arm_many(8), "verify_many_32": arm_many(32),
            "verify_many_128": arm_many(128)}
    rows_out = []
    for k in (500, 2000, 5000):
        for ratio in (0.3, 0.6):
            items = scenes(k, ratio)
            ref = [key(r) for r in arm_loop(items)]  # warm-up of every arm doubles as the equality check
            counts = {}
            for name, fn in arms.items():
                l0, s0 = vctx.launch_count(), vctx.ransac_sync_count()
                assert [key(r) for r in fn(items)] == ref, f"{name} differs from the per-pair results at k={k} ratio={ratio}"
                counts[name] = ((vctx.launch_count() - l0) / len(items), (vctx.ransac_sync_count() - s0) / len(items))
            rates = {name: [] for name in arms}
            for _ in range(a.reps):
                for name, fn in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn(items)  # every arm ends in the stream synchronisation of its last call
                    rates[name].append(len(items) / (time.perf_counter() - t0))
            row = {"mode": "E", "k": k, "inlier_ratio": ratio, "pairs": len(items),
                   "valid": sum(r is not None for r in ref)}
            for name in arms:
                row[name] = {"pairs_per_s": round(float(np.median(rates[name])), 1), "min": round(min(rates[name]), 1),
                             "max": round(max(rates[name]), 1), "launches_per_pair": round(counts[name][0], 3),
                             "syncs_per_pair": round(counts[name][1], 4)}
            print(row, flush=True)
            rows_out.append(row)
            if k == 2000 and ratio == 0.3:  # device time per stage of one 32-pair batch and of one pair
                stage = {}
                for s in STAGES:
                    ms = {}
                    for label, chunk in (("batch32", items[:32]), ("one_pair", items[:1])):
                        vctx.profile_start(s)
                        fe.verify_many(chunk, ctx=vctx, stream=vlane.stream)
                        ms[label] = round(vctx.profile_stop()[0], 4)
                    stage[s] = ms
                print(stage, flush=True)

    # F mode, k = 2000: host per-pair entry + host pose against the batched device call
    eng = RansacEngine(ctx=vctx)
    frow = []
    for ratio in (0.3, 0.6):
        n = min(a.pairs, 64)
        sc = [vr.synthetic_two_view(7000 + i, 2000, ratio) for i in range(n)]
        host = [(np.ascontiguousarray(s[0].astype(np.float32), np.float64), np.ascontiguousarray(s[1].astype(np.float32), np.float64)) for s in sc]
        dev = [(torch.from_numpy(p1).cuda(), torch.from_numpy(p2).cuda()) for p1, p2 in host]
        masks = torch.zeros(n, 2000, dtype=torch.uint8, device="cuda")

        def per_pair():
            out = []
            for (p1, p2), s in zip(host, sc):
                F, mask = eng.fundamental(p1, p2, 4.0)
                Kf = np.array([[s[3][0], 0, s[3][1]], [0, s[3][0], s[3][2]], [0, 0, 1.0]])
                inl = mask == 1
                R, t, _ = eng.recover_pose(Kf.T @ F @ Kf, vr.calibrate(p1[inl], *s[3]), vr.calibrate(p2[inl], *s[3]))
                out.append((F, mask, R, t))
            return out

        def many(batch=32):
            out = []
            for c in range(0, n, batch):
                probs = [ransac_problem(2000, 1, 4.0, F_MAX_ITERS, mask=masks[i], x1=dev[i][0], x2=dev[i][1], cal1=sc[i][3], cal2=sc[i][3])
                         for i in range(c, min(n, c + batch))]
                out += list(eng.verify_batched_dev(probs))
            return out

        torch.cuda.synchronize()
        ref, got = per_pair(), many()
        mh = masks.cpu().numpy()
        for i, ((F, mask, R, t), r) in enumerate(zip(ref, got)):
            assert np.array_equal(np.array(r.model), F.ravel()) and np.array_equal(mh[i], mask), "F batched differs from per pair"
            assert np.abs(np.array(r.R).reshape(3, 3) - R).max() < 1e-9
        rates = {"per_pair_host": [], "batched_32": []}
        s0 = vctx.ransac_sync_count()
        many()
        syncs = (vctx.ransac_sync_count() - s0) / n
        for _ in range(a.reps):
            for name, fn in (("per_pair_host", per_pair), ("batched_32", many)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                rates[name].append(n / (time.perf_counter() - t0))
        row = {"mode": "F", "k": 2000, "inlier_ratio": ratio, "pairs": n, "batched_syncs_per_pair": round(syncs, 4)}
        for name, v in rates.items():
            row[name] = {"pairs_per_s": round(float(np.median(v)), 1), "min": round(min(v), 1), "max": round(max(v), 1)}
        print(row, flush=True)
        frow.append(row)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    line = {"workload": "ransac_verify", "reps": a.reps, "threshold_px": 4.0, "E": rows_out, "F": frow,
            "stage_ms_k2000_ratio0.3": stage, "gpu": name, "power_limit": power}
    s = json.dumps(line)
    print(s)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(s + "\n")


if __name__ == "__main__":
    main()
