"""In-tree build of libgtsfm_b200.so (nvcc, sm_90a only).  `python -m gtsfm_b200.build` or __graft_entry__.build()."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG / "csrc" / "_obj"
LIB = PKG / "libgtsfm_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    # 5-point solver: null space by five Householder reflections (static indexing, registers) instead of Jacobi sweeps on the
    # 9 x 9 Gram matrix (run-time indexed local memory); tests/cpp/test_ransac_math.cpp
    # builds both variants on the host
    "-DB2_FIVEPT_QR",
]
# per-source additions: the LMedS verifier replays cv2's double arithmetic, so its products and sums are not contracted
# into FMAs (its solvers then round as the host build in tests/cpp/lmeds_shim.cpp does); the ORB detector likewise replays
# cv2's float arithmetic (Harris, angles, pattern rotation, resize coordinates) and writes its one FMA chain out explicitly
NVCC_FLAGS_FOR = {"lmeds.cu": ["-fmad=false"], "orb.cu": ["-fmad=false"]}


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(exe).exists():
        raise RuntimeError("nvcc not found; cannot build libgtsfm_b200.so")
    return exe


def _needs(src: Path, obj: Path, deps) -> bool:
    if not obj.exists():
        return True
    t = obj.stat().st_mtime
    return any(d.stat().st_mtime > t for d in [src, *deps])


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.inc")) + list((PKG.parent / "include").glob("*.h"))
    srcs = sorted(CSRC.glob("*.cu"))
    jobs = []
    for s in srcs:
        o = OBJ / (s.stem + ".o")
        if force or _needs(s, o, headers):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [nvcc(), *NVCC_FLAGS, *NVCC_FLAGS_FOR.get(s.name, []), "-c", str(s), "-o", str(o)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s.name}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr.strip():
            print(r.stderr, file=sys.stderr)
        return s.name

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    objs = [OBJ / (s.stem + ".o") for s in srcs]
    if jobs or not LIB.exists() or force:
        cmd = [nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print(p, os.path.getsize(p))
