"""Build libmarigold_b200.so in-tree with nvcc for sm_90a (no torch extension machinery).

    python -m marigold_b200.build [--force] [--verbose]

One translation unit per .cu file, compiled in parallel, linked into
marigold_b200/libmarigold_b200.so. Objects are cached by source mtime.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
BUILD = PKG / "_build"
LIB = PKG / "libmarigold_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; libmarigold_b200 cannot be built (there is no CPU fallback)")


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _headers_mtime() -> float:
    hs = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "marigold_b200.h"]
    return max(h.stat().st_mtime for h in hs)


def _compile(src: Path, verbose: bool) -> tuple[Path, str]:
    obj = BUILD / (src.stem + ".o")
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{log}")
    (BUILD / (src.stem + ".ptxas.log")).write_text(log)
    if verbose:
        print(log)
    return obj, log


def build(force: bool = False, verbose: bool = False) -> Path:
    BUILD.mkdir(exist_ok=True)
    srcs = _sources()
    hm = _headers_mtime()
    todo = []
    for s in srcs:
        obj = BUILD / (s.stem + ".o")
        if force or not obj.exists() or obj.stat().st_mtime < max(s.stat().st_mtime, hm):
            todo.append(s)
    if todo:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(lambda s: _compile(s, verbose), todo))
    objs = [BUILD / (s.stem + ".o") for s in srcs]
    if todo or not LIB.exists() or any(o.stat().st_mtime > LIB.stat().st_mtime for o in objs):
        cmd = [_nvcc(), "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
               "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
