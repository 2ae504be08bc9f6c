"""In-tree build of libb200vit.so (sm_90a only) with plain nvcc.

    python -m vit_pytorch_b200.build            # build if sources are newer than the library
    python -m vit_pytorch_b200.build --force

The library lands in vit_pytorch_b200/lib/libb200vit.so (git-ignored build product).
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
OBJDIR = PKG / "lib" / "obj"
LIB = LIBDIR / "libb200vit.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; libb200vit.so must be prebuilt in-tree")
    return nvcc


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + \
        [PKG.parent / "include" / "b200vit.h"]
    return any(d.stat().st_mtime > t for d in deps)


def _compile(src: Path, verbose: bool) -> Path:
    obj = OBJDIR / (src.stem + ".o")
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    OBJDIR.mkdir(parents=True, exist_ok=True)
    srcs = sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
