"""Device JPEG decode throughput (b2_jpeg_decode_batched_dev through image_io.JpegEngine) on three inputs: the two lund-door
fixtures (1296 x 1936, h1v2), a 640 x 480 synthetic frame (quality 75, 4:2:0) and a 4000 x 3000 synthetic frame (quality 90,
4:2:0), each in batches of 16 and 64.

Arms:
- images/s and compressed GB/s of the device decode (host bytes in, device RGB out, one synchronisation per batch);
- device time per stage (CUDA events around the launches): unstuff (k_jpeg_markers / count / tiles / compact), synchronisation
  (k_jpeg_sync*, with the rounds taken), decode (k_jpeg_bases / write / dc), IDCT (k_jpeg_idct), colour (k_jpeg_color), and
  the share of the H100 SXM's 3.35 TB/s that the byte-bound IDCT and colour stages reach (bytes computed from the shapes);
- PIL (`np.asarray(Image.open(f).convert("RGB"))`) with one process per host core, and torchvision.io.decode_jpeg on the GPU
  (nvJPEG) as a yardstick;
- the chain JPEG bytes -> device RGB -> ingest resize (760) -> SIFT (top 5000) against PIL decode -> H2D -> ingest -> SIFT,
  on the lund fixtures, single process.
The card name and power limit are read in the same run.  Writes one JSON line to --out.

    python profiles/bench_jpeg.py --out profiles/h100_jpeg.json
"""
from __future__ import annotations

import argparse
import io
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HBM_TBS = 3.35  # H100 SXM data sheet
STAGES = {"unstuff": ("k_jpeg_markers", "k_jpeg_count", "k_jpeg_tiles", "k_jpeg_compact"), "sync": ("k_jpeg_sync",),
          "decode": ("k_jpeg_bases", "k_jpeg_write", "k_jpeg_dc"), "idct": ("k_jpeg_idct",), "color": ("k_jpeg_color",)}


def inputs():
    from oracle import jpeg_ref as J

    lund = [(ROOT / "tests/golden/jpeg" / n).read_bytes() for n in ("lund_door_DSC_0001.JPG", "lund_door_DSC_0002.JPG")]
    vga = J.encode(J.content("synthetic", 480, 640, seed=1), "420", quality=75)
    big = J.encode(J.content("synthetic", 3000, 4000, seed=2), "420", quality=90)
    return {"lund_1296x1936": lund, "synthetic_640x480_q75": [vga], "synthetic_4000x3000_q90": [big]}


def _pil_decode(d: bytes) -> int:
    from PIL import Image

    return int(np.asarray(Image.open(io.BytesIO(d)).convert("RGB")).shape[0])


def timed(fn, reps: int) -> float:
    import torch

    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def geometry_bytes(data: bytes):
    """Bytes the IDCT (coefficients read, samples written) and colour (planes read, RGB written) stages must move."""
    from oracle import jpeg_ref as J

    hd = J.parse(data)
    g = J.geometry(hd)
    blocks = g.mcux * g.mcuy * g.bpm
    planes = sum(g.comp_w[c] * g.comp_h[c] for c in range(len(hd.comps)))
    return blocks * (128 + 64), planes + 3 * hd.width * hd.height


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import torchvision

    from gtsfm_b200 import _lib
    from gtsfm_b200.detector_descriptor import SiftEngine
    from gtsfm_b200.image_io import JpegEngine
    from gtsfm_b200.pipeline import DeviceFrontEnd
    from gtsfm_b200 import synthetic as syn

    ctx = _lib.Context(0)
    eng = JpegEngine(0, ctx=ctx)
    res = {"workloads": {}}
    ncpu = os.cpu_count() or 1
    for name, files in inputs().items():
        w = {"compressed_bytes": [len(f) for f in files]}
        for batch in (16, 64):
            datas = [files[i % len(files)] for i in range(batch)]
            nbytes = sum(len(d) for d in datas)
            dt = timed(lambda: eng.decode_many(datas), args.reps)
            w[f"device_b{batch}_images_per_s"] = batch / dt
            w[f"device_b{batch}_compressed_GBps"] = nbytes / dt / 1e9
            w[f"device_b{batch}_rounds"] = sorted(set(eng.last_rounds))
            stages = {}
            for stage, prefixes in STAGES.items():
                ms = 0.0
                for p in prefixes:
                    ctx.profile_start(p)
                    eng.decode_many(datas)
                    ms += ctx.profile_stop()[0]
                stages[stage] = ms
            w[f"device_b{batch}_stage_ms"] = stages
            ib, cb = (sum(x) * batch // len(files) for x in zip(*[geometry_bytes(f) for f in files]))
            w[f"device_b{batch}_hbm_fraction"] = {"idct": ib / (stages["idct"] * 1e-3) / (HBM_TBS * 1e12),
                                                  "color": cb / (stages["color"] * 1e-3) / (HBM_TBS * 1e12)}
        # PIL on every host core
        datas = [files[i % len(files)] for i in range(max(64, 4 * ncpu) if "4000" not in name else max(16, ncpu))]
        with mp.get_context("spawn").Pool(ncpu) as pool:
            pool.map(_pil_decode, datas[:ncpu])
            t = time.perf_counter()
            pool.map(_pil_decode, datas, chunksize=1)
            w["pil_all_cores_images_per_s"] = len(datas) / (time.perf_counter() - t)
        t = time.perf_counter()
        _pil_decode(files[0])
        w["pil_one_core_ms"] = (time.perf_counter() - t) * 1e3
        # nvJPEG through torchvision
        batch = [torch.frombuffer(bytearray(files[i % len(files)]), dtype=torch.uint8) for i in range(64)]
        try:
            dt = timed(lambda: torchvision.io.decode_jpeg(batch, device="cuda"), args.reps)
            w["nvjpeg_b64_images_per_s"] = 64 / dt
        except Exception as e:  # noqa: BLE001 - a yardstick only
            w["nvjpeg_b64_error"] = str(e)[:200]
        w["device_over_pil_all_cores_b64"] = w["device_b64_images_per_s"] / w["pil_all_cores_images_per_s"]
        if "nvjpeg_b64_images_per_s" in w:
            w["device_over_nvjpeg_b64"] = w["device_b64_images_per_s"] / w["nvjpeg_b64_images_per_s"]
        res["workloads"][name] = w
        print(name, json.dumps(w), flush=True)

    # chain: bytes -> device RGB -> resize -> SIFT, against PIL -> H2D -> resize -> SIFT (lund, 16 frames)
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), ctx=ctx)
    sift = SiftEngine(ctx=ctx)
    lund = inputs()["lund_1296x1936"]
    datas = [lund[i % 2] for i in range(16)]

    def device_chain():
        frames = fe.ingest_jpeg(datas)
        return sift.extract_many(frames, max_keypoints=5000)

    def host_chain():
        from PIL import Image

        frames = [fe.ingest(torch.from_numpy(np.asarray(Image.open(io.BytesIO(d)).convert("RGB")).copy()).to(fe.device))
                  for d in datas]
        return sift.extract_many(frames, max_keypoints=5000)

    a, b = device_chain(), host_chain()
    host = lambda t: t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)  # noqa: E731
    same = all(np.array_equal(host(x[0]), host(y[0])) and np.array_equal(host(x[1]), host(y[1])) for x, y in zip(a, b))
    res["chain_lund_16"] = {"jpeg_bytes_device_images_per_s": 16 / timed(device_chain, args.reps),
                            "pil_h2d_images_per_s": 16 / timed(host_chain, args.reps), "same_descriptors": bool(same)}
    print("chain", json.dumps(res["chain_lund_16"]), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    res.update({"gpu": gpu, "power_limit": power, "host_cores": ncpu, "reps": args.reps})
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
