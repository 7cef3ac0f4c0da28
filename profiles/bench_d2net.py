"""D2-Net detector-descriptor throughput on two workloads: 12 seeded 480 x 640 gray synthetic frames and the 12 lund-door
frames at loader resolution (1135 x 760 gray).

Arms, per workload:
- images/s of the batched device path (D2NetEngine.extract_many, top 5000, images already on the GPU) and of the plugin on host
  arrays (B200D2NetDetectorDescriptor.detect_and_describe);
- images/s of the oracle's torch restatement (oracle/d2net_ref.py) in fp32 on the same GPU, TF32 off, and of the same
  restatement on the host cores (the reference algorithm on the CPU, all cores to torch's thread pool);
- pairs/s of device detect -> TwoWayEngine.match_batched_dev at ratio 0.8 on sequential pairs;
- device time per stage (CUDA events around the k_conv_ps<1>, k_conv_ps<2> and k_d2_* launches) and the convolutions' achieved
  TFLOP/s from the shape-computed FLOPs, against the 989 TFLOP/s dense peak: split-fp16 issues 3 MMAs per product, so 0.33 is
  the ceiling of that fraction.
Plus the cost of the dilated instance's two activation buffers: one 512 -> 512 layer at the lund feature-map size on
k_conv_ps<1> (three buffers) and k_conv_ps<2> (two buffers, larger halo), same FLOPs.
The card name and power limit are read in the same run.  Writes one JSON line to --out.

    python profiles/bench_d2net.py --out profiles/h100_d2net.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

PEAK_TFLOPS = 989.0  # H100 SXM dense bf16/fp16 data sheet
STAGES = ("k_conv_ps<1>", "k_conv_ps<2>", "k_d2_")
LAYERS = [(3, 64, 1, 0), (64, 64, 1, 0), (64, 128, 2, 0), (128, 128, 2, 0), (128, 256, 4, 0), (256, 256, 4, 0), (256, 256, 4, 0),
          (256, 512, 4, 1), (512, 512, 4, 1), (512, 512, 4, 1)]  # (Cin, Cout, input downscale, after the average pool)


def conv_flops(h: int, w: int):
    """(all convolutions, those on k_conv_ps<1>, those on k_conv_ps<2>) FLOPs of one image, from the shapes."""
    tot, pad1, dil = 0.0, 0.0, 0.0
    for n, (ci, co, s, after_avg) in enumerate(LAYERS):
        hh, ww = h // 2 // 2 if s == 4 else h // s, w // 2 // 2 if s == 4 else w // s
        if after_avg:
            hh, ww = hh - 1, ww - 1
        f = 2.0 * 9 * hh * ww * ci * co
        tot += f
        if after_avg:
            dil += f
        elif n:
            pad1 += f
    return tot, pad1, dil


def workload(name, frames, reps, ctx, sd):
    import torch

    from gtsfm_b200.detector_descriptor import B200D2NetDetectorDescriptor, D2NetEngine
    from gtsfm_b200.gtsfm_api import Image
    from gtsfm_b200.matcher import TwoWayEngine
    from oracle import d2net_ref

    eng, mt = D2NetEngine(sd, ctx=ctx), TwoWayEngine(ctx=ctx)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    n, npairs = len(frames), len(frames) - 1

    def front_end():
        out = eng.extract_many(dev, max_keypoints=5000)
        return out, mt.match_batched_dev([(out[i][2], out[i + 1][2]) for i in range(npairs)], 0.8)

    for _ in range(2):
        front_end()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = eng.extract_many(dev, max_keypoints=5000)
    torch.cuda.synchronize()
    dev_ips = reps * n / (time.perf_counter() - t0)
    t0 = time.perf_counter()
    for _ in range(reps):
        out, res = front_end()
    torch.cuda.synchronize()
    dev_pps = reps * npairs / (time.perf_counter() - t0)
    stage_ms, stage_flop = {}, {}
    for st in STAGES:
        ctx.profile_start(st)
        for _ in range(reps):
            eng.extract_many(dev, max_keypoints=5000)
        ms, launches, work = ctx.profile_stop()
        stage_ms[st] = round(ms / (reps * n), 4)
        stage_flop[st] = work / (reps * n)
    h, w = frames[0].shape[:2]
    tot, pad1, dil = conv_flops(h, w)
    assert abs(stage_flop["k_conv_ps<1>"] - pad1) < 1e-6 * pad1 and abs(stage_flop["k_conv_ps<2>"] - dil) < 1e-6 * dil
    tflops = {st: (pad1 if st.endswith("<1>") else dil) / (stage_ms[st] * 1e-3) / 1e12 for st in STAGES[:2]}
    conv_tflops = (pad1 + dil) / ((stage_ms["k_conv_ps<1>"] + stage_ms["k_conv_ps<2>"]) * 1e-3) / 1e12

    det = B200D2NetDetectorDescriptor(max_keypoints=5000, model_path=sd)
    det._engine = eng
    det.detect_and_describe(Image(frames[0]))
    plug_reps = max(1, reps // 4)
    t0 = time.perf_counter()
    for _ in range(plug_reps):
        for f in frames:
            det.detect_and_describe(Image(f))
    plugin_ips = plug_reps * n / (time.perf_counter() - t0)

    # the torch restatement in fp32 on the GPU (TF32 off), then the same on the host cores
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd_gpu = {k: torch.from_numpy(v).cuda() for k, v in sd.items()}

    def torch_gpu(f):
        x = torch.from_numpy(d2net_ref.preprocess(f)).cuda()
        dense = _dense_gpu(x, sd_gpu)
        return d2net_ref.detect(dense.cpu(), 5000)

    torch_gpu(frames[0])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in frames:
        torch_gpu(f)
    torch.cuda.synchronize()
    torch_gpu_ips = n / (time.perf_counter() - t0)
    torch.set_num_threads(os.cpu_count() or 1)
    ncpu = 2
    t0 = time.perf_counter()
    for f in frames[:ncpu]:
        d2net_ref.detect_and_describe(f, sd, 5000)
    cpu_ips = ncpu / (time.perf_counter() - t0)
    return {"workload": name, "frames": n, "frame": list(frames[0].shape), "mean_kp": float(np.mean([len(o[1]) for o in out])),
            "mean_total_kp": float(np.mean([o[3] for o in out])), "mean_matches": float(np.mean([len(m) for m in res])),
            "batched_dev_images_per_s": round(dev_ips, 1), "plugin_host_images_per_s": round(plugin_ips, 1),
            "torch_fp32_gpu_images_per_s": round(torch_gpu_ips, 1), "reference_cpu_images_per_s": round(cpu_ips, 3),
            "batched_vs_torch_gpu": round(dev_ips / torch_gpu_ips, 2), "batched_vs_cpu": round(dev_ips / cpu_ips, 1),
            "front_end_dev_pairs_per_s": round(dev_pps, 1), "stage_ms_per_image": stage_ms,
            "gflop_per_image": round(tot / 1e9, 1), "tflops": {k: round(v, 1) for k, v in tflops.items()},
            "conv_tflops": round(conv_tflops, 1), "conv_frac_of_peak": round(conv_tflops / PEAK_TFLOPS, 3)}


def _dense_gpu(x, sd_gpu):
    """oracle/d2net_ref.dense_features on device tensors (the same layer list, fp32)."""
    import torch
    import torch.nn.functional as F

    from oracle import d2net_ref

    t = x[None]
    with torch.no_grad():
        for idx in d2net_ref.CONV_IDX:
            if idx == d2net_ref.DILATED[0]:
                t = F.avg_pool2d(t, 2, stride=1)
            d = 2 if idx in d2net_ref.DILATED else 1
            t = F.relu(F.conv2d(t, sd_gpu[f"dense_feature_extraction.model.{idx}.weight"], sd_gpu[f"dense_feature_extraction.model.{idx}.bias"],
                                padding=d, dilation=d))
            if idx in d2net_ref.POOL_AFTER:
                t = F.max_pool2d(t, 2, stride=2)
    return t[0]


def buffer_cost(ctx, reps):
    """One 512 -> 512 layer at the lund feature-map size (282 x 189) on both instances: device ms and TFLOP/s."""
    import ctypes

    from gtsfm_b200 import _lib

    H, W, C = 282, 189, 512
    rng = np.random.default_rng(0)
    x = np.maximum(rng.standard_normal((H, W, C)), 0).astype(np.float32)
    wt = (rng.standard_normal((C, C, 3, 3)) * 0.02).astype(np.float32)
    b = np.zeros(C, np.float32)
    out = np.empty((H, W, C), np.float32)
    row = {}
    for dil in (1, 2):
        layer = _lib.ConvLayer(1, dil, 0, 1, 0, H, W, C, C, _lib.ptr(x).value, _lib.ptr(wt).value, _lib.ptr(b).value, _lib.ptr(out).value, None,
                               None)
        ctx.check(ctx.lib.b2_debug_conv_host(ctx.handle, ctypes.byref(layer)), "debug conv")
        ctx.profile_start(f"k_conv_ps<{dil}>")
        for _ in range(reps):
            ctx.check(ctx.lib.b2_debug_conv_host(ctx.handle, ctypes.byref(layer)), "debug conv")
        ms, _, work = ctx.profile_stop()
        row[f"dilation_{dil}"] = {"ms": round(ms / reps, 4), "tflops": round(work / reps / (ms / reps * 1e-3) / 1e12, 1),
                                  "activation_buffers": 3 if dil == 1 else 2}
    row["dilated_over_pad1_time"] = round(row["dilation_2"]["ms"] / row["dilation_1"]["ms"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_d2net.json"))
    a = ap.parse_args()

    from gtsfm_b200 import _lib
    from gtsfm_b200 import synthetic as syn

    lund = np.load(ROOT / "tests" / "golden" / "lund_door_images.npz")
    lund_frames = [lund[f"gray_{i}"] for i in range(1, 13)]
    vga = [syn.synthetic_frame(200 + i, 480, 640)[:, :, 0].copy() for i in range(12)]
    sd = syn.d2net_state_dict(7)
    ctx = _lib.Context(0)
    rows = [workload("synthetic_480x640", vga, a.reps, ctx, sd), workload("lund_door_loader", lund_frames, a.reps, ctx, sd)]
    cost = buffer_cost(ctx, a.reps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    line = {"workload": "d2net", "weights": "seeded synthetic (d2net_state_dict(7))", "max_keypoints": 5000, "ratio": 0.8,
            "cpu_cores": os.cpu_count(), "results": rows, "conv_buffer_cost": cost, "peak_tflops": PEAK_TFLOPS, "gpu": name,
            "power_limit": power}
    s = json.dumps(line)
    print(s)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(s + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
