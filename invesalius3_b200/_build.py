"""In-tree build recipes: libb2v.so (CUDA, sm_90a) and the CPU oracle.

nvcc cross-compiles without a GPU; the resulting .so files are build products and stay
out of git.
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
LIB = PKG / "libb2v.so"
OBJ = PKG / "csrc" / "_obj"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",              # reference arithmetic (Rust, NumPy) never contracts to FMA
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; libb2v.so cannot be built")


def _newer(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a and link libb2v.so next to the package."""
    srcs = sorted(CSRC.glob("*.cu"))
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted((ROOT / "include").glob("*.h"))
    OBJ.mkdir(exist_ok=True)
    nvcc = _nvcc()
    jobs = []
    for s in srcs:
        o = OBJ / (s.stem + ".o")
        if force or _newer(o, [s, *hdrs, Path(__file__)]):   # this file holds the flags
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(s), "-o", str(o)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        (OBJ / (s.stem + ".ptxas.txt")).write_text(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return o

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    objs = [OBJ / (s.stem + ".o") for s in srcs]
    if force or jobs or _newer(LIB, objs):
        cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), *GENCODE,
               "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link of libb2v.so failed:\n{r.stdout}\n{r.stderr}")
    return LIB


def build_oracle(force: bool = False) -> Path:
    """Compile the CPU oracle (test infrastructure only) via oracle/Makefile, the 3-D mask
    editor's checker via oracle/editor.mk, the jump-flooding checker via oracle/voronoi.mk, the
    visible-faces checker via oracle/visibility.mk, the connectivity checker via
    oracle/connectivity.mk, the smoothing checker via oracle/smoothing.mk, the hole-filling checker via
    oracle/fill_holes.mk, the normals checker via oracle/normals.mk, the geodesic checker via oracle/geodesic.mk,
    the volume rendering's data-preparation checker via oracle/raycasting.mk and the clean and triangle filter's
    checker via oracle/clean.mk."""
    for makefile in ([], ["-f", "editor.mk"], ["-f", "voronoi.mk"], ["-f", "visibility.mk"],
                     ["-f", "connectivity.mk"], ["-f", "smoothing.mk"], ["-f", "fill_holes.mk"],
                     ["-f", "normals.mk"], ["-f", "geodesic.mk"], ["-f", "raycasting.mk"], ["-f", "clean.mk"]):
        r = subprocess.run(["make", "-C", str(ROOT / "oracle"), *makefile, *(["-B"] if force else [])],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"oracle build failed:\n{r.stdout}\n{r.stderr}")
    return ROOT / "oracle" / "liboracle.so"


if __name__ == "__main__":
    force = "--force" in sys.argv
    print(build_cuda(force=force, verbose="-v" in sys.argv))
    print(build_oracle(force=force))
