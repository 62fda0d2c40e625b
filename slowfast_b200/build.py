"""In-tree build of the native library (nvcc, sm_90a only).

The shared object lands next to the sources (``slowfast_b200/csrc/libsfb200.so``) so that it travels with the
repository snapshot to the GPU box; nothing is installed into site-packages and no JIT cache is used.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB_NAME = "libsfb200.so"
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
              "-Xptxas", "-v", "-DSFB_BUILD_ARCH=\"sm_90a\""]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (needed to build slowfast_b200's sm_90a kernels)")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(ARCH_FLAGS + NVCC_FLAGS).encode())
    return h.hexdigest()


def lib_path() -> Path:
    return CSRC / LIB_NAME


def build_native(force: bool = False, verbose: bool = False) -> Path:
    """Compile every ``csrc/*.cu`` for sm_90a and link ``libsfb200.so``. Returns the library path."""
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) +
                     list((CSRC.parent.parent / "include").glob("*.h")))
    stamp = CSRC / "build" / "stamp.txt"
    digest = _digest(sources + headers)
    out = lib_path()
    if not force and out.exists() and stamp.exists() and stamp.read_text().strip() == digest:
        return out
    nvcc = _nvcc()
    bdir = CSRC / "build"
    bdir.mkdir(exist_ok=True)

    def compile_one(src: Path) -> Path:
        obj = bdir / (src.stem + ".o")
        cmd = [nvcc, *ARCH_FLAGS, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        (bdir / (src.stem + ".ptxas.log")).write_text(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(sources))) as ex:
        objs = list(ex.map(compile_one, sources))
    cmd = [nvcc, *ARCH_FLAGS, "-shared", "-o", str(out), *map(str, objs), "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return out


if __name__ == "__main__":
    import sys
    print(build_native(force="--force" in sys.argv, verbose="-v" in sys.argv))
