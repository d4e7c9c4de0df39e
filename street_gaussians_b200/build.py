"""Builds street_gaussians_b200/libsgr.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

``python -m street_gaussians_b200.build`` or ``__graft_entry__.build()``.  nvcc cross-compiles without a GPU.
The .so and the objects under _obj/ are build products (git-ignored).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libsgr.so")
SOURCES = ["capi.cu", "preprocess_fwd.cu", "binning.cu", "blend_fwd.cu", "blend_bwd.cu", "blend_bwd2.cu", "preprocess_bwd.cu", "knn.cu", "peer_exchange.cu", "compose.cu", "corrections.cu", "losses.cu", "optim.cu", "densify.cu", "rebalance.cu", "layers.cu", "sky.cu", "actor_pose.cu", "features.cu", "metrics.cu"]
HEADERS = ["sgr_common.cuh", "ssim_tile.cuh", "gaussian_geom.cuh", "tile_visit.cuh", os.path.join("..", "..", "include", "sgr.h")]
# no --use_fast_math: parity with the reference needs IEEE division/sqrt and the accurate expf (DGR/setup.py:30 has none either)
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, extra_flags=()) -> str:
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    jobs = []
    for s in SOURCES:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s + ".o")
        if force or _stale(obj, [src] + hdrs):
            jobs.append([nvcc, "-c", src, "-o", obj] + NVCC_FLAGS + list(extra_flags))

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr, file=sys.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, s + ".o") for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        run([nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, extra_flags=["-Xptxas", "-v"] if "--ptxas" in sys.argv else ()))
