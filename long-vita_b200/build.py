"""Build liblvb200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

The library has no Python / torch dependency: `nvcc -shared` over long-vita_b200/csrc/*.cu with the
static CUDA runtime.  The built artefact lives at long-vita_b200/lib/liblvb200.so (git-ignored).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "liblvb200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


if os.environ.get("LV_WATCHDOG") == "1":      # debug build: stuck waits report themselves and trap (csrc/ptx.cuh)
    NVCC_FLAGS.append("-DLV_WATCHDOG")
if os.environ.get("LV_EXTRA_DEFINES"):         # experiment builds: extra nvcc -D flags, space separated
    NVCC_FLAGS.extend(os.environ["LV_EXTRA_DEFINES"].split())


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; the CUDA extension cannot be built")
    return nvcc


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths) -> str:
    """Content hash of the sources (file names, not absolute paths: a copy of the tree in another directory
    accepts the library built here instead of rebuilding it)."""
    h = hashlib.sha256()
    for p in sorted(paths, key=os.path.basename):
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode())
            h.update(f.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = _sources()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "lvb200.h"))
    stamp = os.path.join(OBJDIR, "stamp")
    digest = _digest(srcs + headers)
    flags = " ".join(NVCC_FLAGS)
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        have = open(stamp).read().split("\n")
        # same sources; and the same flags unless the caller did not ask for a particular variant
        # (LV_WATCHDOG unset: keep whichever variant was shipped, e.g. a watchdog build made before gpurun)
        variant_asked = "LV_WATCHDOG" in os.environ or "LV_EXTRA_DEFINES" in os.environ
        if have[0] == digest and (not variant_asked or have[1:2] == [flags]):
            return LIB
    nvcc = _nvcc()

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".log")
        with open(log, "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-cudart", "static", "-Xlinker", "--no-undefined"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(digest + "\n" + flags)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
