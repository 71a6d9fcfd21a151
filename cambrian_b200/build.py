"""In-tree build of libcambrian_b200.so (sm_90a, H100, only).

`python -m cambrian_b200.build` cross-compiles every csrc/*.cu with nvcc (no GPU needed) and links one
shared library next to this file, where the ctypes loader (`_lib.py`) finds it.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "csrc" / "_obj"
LIB = HERE / "libcambrian_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC", "--use_fast_math", "-Xptxas", "-v",
]
# --use_fast_math would change erff/expf/division accuracy in the numerics-critical kernels; keep IEEE
FLAGS.remove("--use_fast_math")


def _newer(src: Path, dst: Path, deps: list[Path]) -> bool:
    if not dst.exists():
        return True
    t = dst.stat().st_mtime
    return any(p.stat().st_mtime > t for p in [src, *deps])


def _compile(src: Path, verbose: bool) -> Path:
    obj = OBJ / (src.stem + ".o")
    deps = list(CSRC.glob("*.cuh")) + [HERE.parent / "include" / "cambrian_b200.h"]
    if _newer(src, obj, deps):
        cmd = [NVCC, *FLAGS, *os.environ.get("CB_NVCC_EXTRA", "").split(), "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        (OBJ / (src.stem + ".ptxas.txt")).write_text(r.stderr)
        if verbose:
            print(f"[build] compiled {src.name}")
    return obj


def build(verbose: bool = True) -> Path:
    OBJ.mkdir(exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if not LIB.exists() or any(o.stat().st_mtime > LIB.stat().st_mtime for o in objs):
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[build] linked {LIB}")
    return LIB


if __name__ == "__main__":
    build()
    sys.exit(0)
