"""Builds libmagickb200.so (and the optional MagickCore shim) in-tree with nvcc for sm_90a.

    python -m imagemagick_b200.build [--force] [--verbose]

The shared library lands in imagemagick_b200/lib/ (git-ignored).  nvcc cross-compiles
without a GPU, so this runs anywhere the CUDA toolkit is installed.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
OBJDIR = LIBDIR / "obj"
LIB = LIBDIR / "libmagickb200.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden,-ffp-contract=off",
              "-Xptxas", "-v"]

SOURCES = ["runtime.cu", "kernel_info.cpp", "resize_filter.cpp", "resize_tables.cpp", "conv1d.cu", "conv_mma.cu",
           "morph2d.cu", "morph_stream.cu", "morph_direct.cu", "cache.cu", "resize.cu", "resize_stream.cu", "colorspace.cu", "hexcone.cu", "pointwise.cu", "stencils.cu", "hooks.cu", "enhance.cu", "layout.cu", "level.cu",
           "distort_plan.cpp", "distort.cu", "geometry_plan.cpp", "geometry.cu", "threshold.cu", "trim.cu", "api.cu"]
# distort.cu restates the reference's EWA sampler operation by operation: no contraction into fused multiply-adds.
FILE_FLAGS = {"distort.cu": ["-fmad=false"], "threshold.cu": ["-fmad=false"], "trim.cu": ["-fmad=false"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; libmagickb200 cannot be built")


def _stale(target: Path, deps: list[Path]) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps if d.exists())


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = _nvcc()
    OBJDIR.mkdir(parents=True, exist_ok=True)
    headers = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + list((ROOT / "include").glob("*.h"))
    jobs = []
    for name in SOURCES:
        src = CSRC / name
        obj = OBJDIR / (src.stem + ".o")
        if force or _stale(obj, [src] + headers):
            cmd = [nvcc, *ARCH, *NVCC_FLAGS, *FILE_FLAGS.get(name, []), "-x", "cu", "-c", str(src), "-o", str(obj)]
            jobs.append((name, cmd, obj))

    def run(job):
        name, cmd, obj = job
        p = subprocess.run(cmd, capture_output=True, text=True)
        log = OBJDIR / (Path(name).stem + ".log")
        log.write_text(" ".join(cmd) + "\n" + p.stdout + p.stderr)
        return name, p.returncode, p.stdout + p.stderr

    failed = False
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for name, rc, out in ex.map(run, jobs):
            if rc != 0:
                failed = True
                sys.stderr.write(f"[build] {name} FAILED\n{out}\n")
            elif verbose:
                sys.stderr.write(f"[build] {name} ok\n{out}\n")
    if failed:
        raise RuntimeError("libmagickb200 build failed")
    objs = [OBJDIR / (Path(n).stem + ".o") for n in SOURCES]
    if force or jobs or _stale(LIB, objs):
        cmd = [nvcc, *ARCH, "-shared", "-cudart", "static", "-o", str(LIB), *map(str, objs)]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("link failed:\n" + p.stdout + p.stderr)
    return LIB


if __name__ == "__main__":
    lib = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(lib)
