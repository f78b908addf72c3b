"""Build libwts.so (hand-written sm_90a CUDA behind the C-ABI of include/wts.h) in-tree.

    python whisper-timestamped_b200/build.py [--force] [--verbose]

nvcc cross-compiles for sm_90a without a GPU; the resulting .so is git-ignored and rebuilt
from source whenever a source is newer.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "whisper_timestamped", "libwts.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC",
]


LINK_LIBS = []   # cudart is linked statically by nvcc; the driver API is reached through cudaGetDriverEntryPoint


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) \
        + [os.path.join(HERE, "..", "include", "wts.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, "-c", src, "-o", obj] + NVCC_FLAGS
        if verbose:
            cmd += ["-Xptxas", "-v"]
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd)))
        objs.append(obj)
    for src, p in procs:
        if p.wait() != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    link = [nvcc, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"] + LINK_LIBS
    if verbose:
        print(" ".join(link))
    subprocess.check_call(link)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
