#!/usr/bin/env python
"""Where a vga_lightglue step's matcher time goes, call site by call site.

    python profiles/lightglue_call_sites.py [--steps 2] [--warmup 3] [--out FILE.json]

Runs the step bench.py times for the default workload (two new synthetic 640x480 frames, each matched against the 20
frames before it with LightGlue in lock-step batches of 8 and verified on the verification stream) and times, one extra
step per row, every launch of one k_gemm_ws call site ("k_gemm_ws/<site>", the label run_linear hands the profiler) and
of every k_lg_* kernel with CUDA events on the launching stream.

Each row also gets the work its shapes imply: FLOP (split-fp16 counted as the 3 tensor-core products it issues) and the
HBM bytes of its operands and outputs, and the least time the hardware could take, max(FLOP / 989 TFLOP/s, bytes / 3.35
TB/s) (H100 SXM data sheet, dense fp16, 700 W).  The row count of every per-keypoint kernel comes from the FLOP the QKV
projection reported, so the model follows the keypoint counts the step really had.  The shapes of the model are
LightGlue's (d = 256, 4 heads of 64, feed-forward 512); weights are not counted (at most 1 MB per launch, L2-resident)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from collections import deque
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12
LOOKAHEAD, NEW_FRAMES, THR_PX = 20, 2, 4.0

GEMM_SITES = ["lg_self_qkv", "lg_self_out", "lg_self_ffn0", "lg_self_ffn3", "lg_cross_qk", "lg_cross_v", "lg_cross_qv",
              "lg_cross_out", "lg_cross_ffn0", "lg_cross_ffn3", "lg_assign_proj", "lg_assign_sim"]
LG_KERNELS = ["k_lg_load_desc", "k_lg_posenc", "k_lg_enc_copy", "k_lg_split_rotary", "k_lg_ln_gelu", "k_lg_rowheads", "k_lg_prune_plan", "k_lg_gather",
              "k_lg_assign", "k_lg_row_stats", "k_lg_col_stats", "k_lg_row_argmax", "k_lg_col_argmax", "k_lg_filter"]
# (N, K) of each GEMM site and its HBM bytes per output row: split-fp16 A planes are 4 B per element, plane outputs 4 B,
# fp32 outputs / residuals 4 B, the rotary table 2 x 32 x 4 B per row of each of q and k
GEMM_SHAPE = {
    "lg_self_qkv": (768, 256), "lg_self_out": (256, 256), "lg_self_ffn0": (512, 512), "lg_self_ffn3": (256, 512),
    "lg_cross_qk": (256, 256), "lg_cross_v": (256, 256), "lg_cross_qv": (512, 256), "lg_cross_out": (256, 256),
    "lg_cross_ffn0": (512, 512), "lg_cross_ffn3": (256, 512), "lg_assign_proj": (256, 256)}
GEMM_ROW_BYTES = {
    "lg_self_out": 256 * 4 + 256 * 4, "lg_self_ffn0": 512 * 4 + 512 * 4, "lg_self_ffn3": 512 * 4 + 256 * 4 * 3,
    "lg_cross_qk": 256 * 4 + 256 * 4, "lg_cross_v": 256 * 4 + 256 * 4, "lg_cross_qv": 256 * 4 + 512 * 4,
    "lg_cross_out": 256 * 4 + 256 * 4, "lg_cross_ffn0": 512 * 4 + 512 * 4, "lg_cross_ffn3": 512 * 4 + 256 * 4 * 3,
    "lg_assign_proj": 256 * 4 + 256 * 4 * 2}


def qkv_row_bytes(fused: bool) -> int:
    # A planes in; fused: q / k / v planes out + the rotary table for q and k; unfused: qkv fp32 out
    return 256 * 4 + (768 * 4 + 2 * 64 * 4 if fused else 768 * 4)


# k_lg_* bytes per keypoint row (R = rows of one attention block, summed over layers, sides and batches of the step)
LG_ROW_BYTES = {
    "k_lg_split_rotary": (768 * 4 + 64 * 4 + 768 * 4, 1.0),  # qkv fp32 + cos / sin in, q / k / v planes out; once per self block
    "k_lg_ln_gelu": (512 * 4 + 512 * 4, 2.0),                 # h fp32 in, planes out; once per self and per cross block
    "k_lg_rowheads": (256 * 4, 1.0 / 9 * 8),                  # x in, after every layer but the last
}


def gpu_name() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers are still the numbers; the card is then unknown
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2, help="steps per profiled row (their mean is reported)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()

    import torch

    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFrontEnd

    dev = torch.device("cuda", 0)
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "bench"), device=0, max_keypoints=5000)
    n_frames = LOOKAHEAD + NEW_FRAMES * (args.warmup + args.steps * (len(GEMM_SITES) + len(LG_KERNELS) + 2) + 2)
    frames, cal = syn.synthetic_sequence(n_frames, 480, 640, seed=77)
    frames_dev = [torch.from_numpy(f).to(dev) for f in frames]
    window = deque((fe.detect(frames_dev[i]) for i in range(LOOKAHEAD)), maxlen=LOOKAHEAD)
    cursor = [LOOKAHEAD]

    def step():
        pending = []
        for _ in range(NEW_FRAMES):
            f = fe.detect(frames_dev[cursor[0]])
            cursor[0] += 1
            prevs = list(window)

            def on_chunk(c0, res, prevs=prevs, f=f):
                for prev, (m, _) in zip(prevs[c0:c0 + len(res)], res):
                    pending.append(fe.verify_async(prev, f, m, cal, cal, THR_PX))

            fe.match_many([(p, f) for p in prevs], on_chunk=on_chunk)
            window.append(f)
        for fut in pending:
            fut.result()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps

    def profile(prefix):
        fe.profile_start(prefix)
        for _ in range(args.steps):
            step()
        ms, n, work = fe.profile_stop()
        return ms / args.steps, n / args.steps, work / args.steps

    rows = {}
    for site in GEMM_SITES:
        ms, n, work = profile(f"k_gemm_ws/{site}")
        if n:
            rows[site] = {"kernel": f"k_gemm_ws/{site}", "ms": ms, "launches": n, "work": work}
    for k in LG_KERNELS:
        ms, n, _ = profile(k)
        if n:
            rows[k] = {"kernel": k, "ms": ms, "launches": n, "work": 0.0}
    fam = {f: profile(f) for f in ("k_gemm_ws", "k_lg_", "k_flash_ps")}

    fused = "k_lg_split_rotary" not in rows
    R = rows["lg_self_qkv"]["work"] / (2 * 768 * 256)  # keypoint rows through one attention block, per step
    for name, r in rows.items():
        flop, nbytes = 0.0, None
        if name in GEMM_SHAPE:
            N, K = GEMM_SHAPE[name]
            M = r["work"] / (2 * N * K)
            flop = 3 * r["work"]
            nbytes = M * (qkv_row_bytes(fused) if name == "lg_self_qkv" else GEMM_ROW_BYTES[name])
        elif name == "lg_assign_sim":
            flop = 3 * r["work"]
            nbytes = r["work"] / (2 * 256) * 4  # the fp32 similarity (M x N); its operands are 2 x 1 KB per row, negligible
        elif name in LG_ROW_BYTES:
            per_row, mult = LG_ROW_BYTES[name]
            nbytes = per_row * mult * R
        r["gflop"] = flop / 1e9
        r["mb"] = None if nbytes is None else nbytes / 1e6
        if nbytes is not None:
            t_f, t_b = flop / PEAK_FLOPS * 1e3, nbytes / PEAK_BYTES * 1e3
            r["bound_ms"] = max(t_f, t_b)
            r["bound"] = "tensor" if t_f >= t_b else "HBM"
            r["frac_of_bound"] = r["bound_ms"] / r["ms"] if r["ms"] else None
    out = {"gpu": gpu_name(), "workload": "vga_lightglue (40 pairs per step, <= 5000 keypoints)", "steps_per_row": args.steps,
           "step_ms": step_ms, "rows_per_block": R, "families": {f: {"ms": v[0], "launches": v[1]} for f, v in fam.items()},
           "rows": rows}
    print(f"# {out['gpu']}; step {step_ms:.1f} ms (unprofiled); {R:.0f} keypoint rows per attention block per step")
    print(f"{'call site / kernel':<34}{'ms/step':>9}{'launch':>8}{'GFLOP':>9}{'MB':>9}{'bound ms':>10}  bound  of bound")
    for name, r in rows.items():
        mb = "-" if r["mb"] is None else f"{r['mb']:.0f}"
        b = "-" if "bound_ms" not in r else f"{r['bound_ms']:.2f}"
        frac = "-" if "bound_ms" not in r else f"{100 * r['frac_of_bound']:.0f}%"
        print(f"{r['kernel']:<34}{r['ms']:>9.2f}{r['launches']:>8.0f}{r['gflop']:>9.0f}{mb:>9}{b:>10}  {r.get('bound', '-'):<6} {frac:>5}")
    for f, (ms, n, _) in fam.items():
        print(f"{f + ' (family)':<34}{ms:>9.2f}{n:>8.0f}")
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
