"""Build libivb200.so (in-tree) with nvcc for sm_90a.

The shared library is a plain C-ABI object (include/ivb200.h); it links only against the CUDA
runtime (cuTensorMapEncodeTiled is resolved at run time through cudaGetDriverEntryPoint), so it
cross-compiles without a GPU; the H100 only loads the built library.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OUT = PKG / "libivb200.so"
OBJ = PKG / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--use_fast_math", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def sources():
    return sorted(CSRC.glob("*.cu"))


def build(force: bool = False, verbose: bool = False) -> Path:
    srcs = sources()
    hdrs = sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "ivb200.h"]
    OBJ.mkdir(exist_ok=True)
    hdr_digest = _digest(hdrs)
    nvcc = _nvcc()

    def compile_one(src: Path):
        obj = OBJ / (src.stem + ".o")
        stamp = OBJ / (src.stem + ".stamp")
        dig = _digest([src]) + hdr_digest
        if not force and obj.exists() and stamp.exists() and stamp.read_text() == dig:
            return obj, ""
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        stamp.write_text(dig)
        return obj, r.stderr

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(compile_one, srcs))
    objs = [o for o, _ in results]
    log = "\n".join(l for _, l in results if l)
    (OBJ / "ptxas.log").write_text(log)
    if verbose and log:
        print(log)
    newest = max(o.stat().st_mtime for o in objs)
    if force or not OUT.exists() or OUT.stat().st_mtime < newest:
        cmd = [nvcc, "-shared", "-o", str(OUT), *map(str, objs), "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print("built", p)
