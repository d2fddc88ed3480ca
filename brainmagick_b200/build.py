"""Builds libbm_b200.so in-tree with nvcc for sm_90a (H100) (cross-compiles without a GPU)."""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbm_b200.so")
STAMP = LIB + ".sha256"        # digest of the sources the library was built from (git-ignored, travels with the .so)
# one translation unit per subsystem, compiled in parallel; no relocatable device code, so each keeps its own kernels
SOURCES = ["api.cu", "gemm_simt.cu", "front_api.cu", "convseq_api.cu", "tc_conv_api.cu", "clip_api.cu", "losses_api.cu",
           "svd_api.cu", "prep_api.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _source_digest() -> str:
    """sha256 over the flags, every file under csrc/ and the public header: what the built library depends on.  Content, not
    mtimes -- a checkout, a snapshot copy to another box or a `touch` must not trigger (or hide the need for) a rebuild."""
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    paths = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC))
    paths.append(os.path.join(os.path.dirname(HERE), "include", "bm_b200.h"))
    for p in paths:
        if os.path.isfile(p):
            h.update(os.path.basename(p).encode())
            with open(p, "rb") as f:
                h.update(f.read())
    return h.hexdigest()


def is_current() -> bool:
    if not (os.path.isfile(LIB) and os.path.isfile(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _source_digest()


def compile_library(out: str, extra_flags: list[str] = (), verbose: bool = False, csrc: str = CSRC) -> str:
    """Compiles every SOURCES translation unit of `csrc` with `nvcc -c` in parallel, then links them with one
    `nvcc -shared` into `out`.  The objects live in a temporary directory: the tree receives the library alone."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    name = os.path.basename(out)

    def run(cmd):
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError(f"nvcc failed building {name}")
        if verbose:
            sys.stderr.write(res.stderr)

    with tempfile.TemporaryDirectory() as tmp:
        objs = [os.path.join(tmp, os.path.splitext(s)[0] + ".o") for s in SOURCES]
        cmds = [[nvcc] + NVCC_FLAGS + list(extra_flags) + ["-c", os.path.join(csrc, s), "-o", o]
                for s, o in zip(SOURCES, objs)]
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(cmds), os.cpu_count() or 1)) as pool:
            list(pool.map(run, cmds))
        run([nvcc, "-shared"] + objs + ["-o", out, "-lcudart"])
    return out


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and is_current():
        return LIB
    compile_library(LIB, (["-Xptxas", "-v"] if verbose else []), verbose)
    with open(STAMP, "w") as f:
        f.write(_source_digest() + "\n")
    return LIB


if __name__ == "__main__":
    print(build_library(force=True, verbose="-v" in sys.argv))
