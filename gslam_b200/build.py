"""In-tree build of the sm_90a (H100) CUDA library.

`python -m gslam_b200.build` (or __graft_entry__.build()) cross-compiles with nvcc for sm_90a — no GPU needed — into
gslam_b200/lib/.  The .so files are git-ignored; a content hash (.stamp) decides whether a rebuild is needed.
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(ROOT)
CSRC = os.path.join(ROOT, "csrc")
LIBDIR = os.path.join(ROOT, "lib")
OBJDIR = os.path.join(ROOT, "build")
KERNEL_LIB = os.path.join(LIBDIR, "libgslam_b200_kernels.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


# pnp.cu compares integer inlier counts across hypotheses and against the CPU checker: no FMA contraction there
# (host side too: gb_pnp_ransac re-derives the winner's inlier mask on the host and must count exactly what the device counted)
PER_FILE_FLAGS = {"pnp.cu": ["--fmad=false", "-Xcompiler", "-ffp-contract=off"]}


def _nvcc() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: the CUDA library cannot be built (there is no CPU fallback)")


def _hash(paths, extra="") -> str:
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(p.encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _sources():
    cu = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdr = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    hdr.append(os.path.join(REPO, "include", "gslam_b200.h"))
    return cu, hdr


def build_kernels(force: bool = False, verbose: bool = False) -> str:
    cu, hdr = _sources()
    stamp_path = os.path.join(LIBDIR, ".stamp_kernels")
    want = _hash(cu + hdr, " ".join(NVCC_FLAGS) + repr(sorted(PER_FILE_FLAGS.items())))
    if not force and os.path.exists(KERNEL_LIB) and os.path.exists(stamp_path) and open(stamp_path).read() == want:
        return KERNEL_LIB
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *PER_FILE_FLAGS.get(os.path.basename(src), []), "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".ptxas.log")
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr, file=sys.stderr)
        return obj

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(cu))) as ex:
        objs = list(ex.map(compile_one, cu))
    cmd = [nvcc, "-shared", "-o", KERNEL_LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp_path, "w") as f:
        f.write(want)
    return KERNEL_LIB


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_kernels(force, verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(KERNEL_LIB)
