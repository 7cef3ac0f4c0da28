"""MegaLoc global descriptor throughput: batches of 16 frames at 322 x 322 (megaloc_sift_frontend.yaml's batch_size).

Arms (seeded weights, synthetic frames):
  * dev        b2_megaloc_describe_dev on normalised fp32 device images
  * u8_dev     b2_megaloc_describe_u8_dev on 480 x 640 uint8 device frames: the resize to 322 x 322 and normalisation included
  * plugin     B200MegaLocGlobalDescriptor.describe_batch on the host tensor its batch transform returns
  * torch_gpu  oracle/megaloc_ref.py as torch fp32 on the same GPU (the reference runs its module on CUDA when it exists;
               torch's defaults leave TF32 off for matmuls and on for cuDNN convolutions - the patch embed here)
  * torch_cpu  the same on the host cores
Per-stage CUDA-event times come from the library's launch profiler (kernel-name prefixes); achieved TFLOP/s is the FLOP
count from shapes (`flops_per_image`) over the measured time.  The card name and power limit are read in the same run.
    python profiles/bench_megaloc.py --out profiles/h100_megaloc.json
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


def flops_per_image(h: int = 322, w: int = 322) -> dict:
    """Multiply-adds x 2 from the layer shapes."""
    n = (h // 14) * (w // 14)
    t = n + 1
    blocks = 12 * 2 * t * 768 * (3 * 768 + 768 + 3072 + 3072)
    attn = 12 * 12 * 2 * 2 * t * t * 64
    embed = 2 * n * 588 * 768
    salad = 2 * t * 768 * 1024 + 2 * t * 512 * (256 + 64) + 2 * 768 * 512 + 2 * 512 * 256 + 2 * n * 256 * 64
    head = 2 * 16640 * 8448
    return dict(blocks=blocks, attention=attn, embed=embed, salad=salad, head=head, total=blocks + attn + embed + salad + head)


def timed(fn, sync, reps):
    fn()
    sync()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    sync()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch

    from gtsfm_b200 import _lib, synthetic as syn
    from gtsfm_b200.global_descriptor import B200MegaLocGlobalDescriptor, MegaLocEngine
    from oracle import megaloc_ref

    B = 16
    sd = syn.megaloc_state_dict(5)
    ctx = _lib.Context(0)
    eng = MegaLocEngine(sd, ctx=ctx)
    frames = [syn.synthetic_frame(200 + i, 480, 640) for i in range(B)]
    u8 = [torch.from_numpy(f).cuda() for f in frames]
    x = torch.from_numpy(megaloc_ref.normalise(np.stack([megaloc_ref.resize_u8(f) for f in frames]))).cuda()
    sync = torch.cuda.synchronize
    fl = flops_per_image()
    res = {"workload": f"{B} frames 480x640 -> 322x322 per call", "flops_per_image": fl}
    res["dev_ms"] = 1e3 * timed(lambda: eng.describe_dev(x), sync, args.reps)
    res["u8_dev_ms"] = 1e3 * timed(lambda: eng.describe_u8_dev(u8), sync, args.reps)
    g = B200MegaLocGlobalDescriptor(weights_path=sd)
    g._engine = eng
    xh = x.cpu()
    res["plugin_ms"] = 1e3 * timed(lambda: g.describe_batch(xh), sync, args.reps)
    res["dev_images_per_s"] = B / res["dev_ms"] * 1e3
    res["dev_tflops"] = B * fl["total"] / (res["dev_ms"] * 1e-3) / 1e12
    # per-stage device time from the launch profiler
    stages = {}
    for prefix, key in (("k_gemm_ws", "gemm"), ("k_flash_ps", "attention"), ("k_ml_", "simt")):
        ctx.profile_start(prefix)
        eng.describe_dev(x)
        ms, launches, work = ctx.profile_stop()
        stages[key] = dict(ms=ms, launches=launches, tflops=(work / (ms * 1e-3) / 1e12) if work and ms else None)
    res["stages"] = stages
    # the torch restatement on the GPU and on the host
    t = {k: v.cuda() for k, v in megaloc_ref.tensors(sd).items()}

    def torch_fwd(tt, xx):
        with torch.no_grad():
            tok = megaloc_ref.backbone(tt, xx)
            return torch.nn.functional.normalize(torch.nn.functional.linear(megaloc_ref.salad(tt, tok), tt["aggregator.linear.weight"],
                                                                            tt["aggregator.linear.bias"]), dim=1)

    res["torch_gpu_ms"] = 1e3 * timed(lambda: torch_fwd(t, x), sync, args.reps)
    tc = megaloc_ref.tensors(sd)
    res["torch_cpu_threads"] = torch.get_num_threads()
    res["torch_cpu_ms"] = 1e3 * timed(lambda: torch_fwd(tc, xh), lambda: None, 1)
    res["torch_tf32_matmul"] = bool(torch.backends.cuda.matmul.allow_tf32)
    res["torch_tf32_cudnn"] = bool(torch.backends.cudnn.allow_tf32)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    res.update(gpu=name, power_limit=power)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
