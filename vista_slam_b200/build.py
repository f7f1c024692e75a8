"""Build libsta_b200.so (hand-written sm_90a CUDA, C ABI in include/sta_b200.h) in-tree with nvcc.

    python -m vista_slam_b200.build [--force]

nvcc cross-compiles without a GPU.  The shared object lands next to the sources
(vista_slam_b200/csrc/libsta_b200.so, git-ignored).  The nvcc flags it was built with are recorded in
csrc/build/nvcc_flags.txt, so that a library built with other flags (another GPU architecture) is rebuilt.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libsta_b200.so")
OBJDIR = os.path.join(CSRC, "build")
STAMP = os.path.join(OBJDIR, "nvcc_flags.txt")
SOURCES = ["host_util.cu", "gemm.cu", "attention.cu", "kernels.cu", "pointmap.cu", "preprocess.cu", "pose_graph.cu",
           "pose_graph_sparse.cu", "flow.cu", "orb.cu", "bow.cu", "slam_graph.cu", "recon.cu", "render.cu", "fusion.cu",
           "raycast.cu", "consistency.cu", "runtime.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-Wno-format-truncation",
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libsta_b200.so")
    return exe


def _stale():
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != " ".join(NVCC_FLAGS):
            return True
    t = os.path.getmtime(LIB)
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh", ".h")) and os.path.getmtime(os.path.join(CSRC, f)) > t:
            return True
    hdr = os.path.join(os.path.dirname(CSRC), "..", "include", "sta_b200.h")
    return os.path.exists(hdr) and os.path.getmtime(hdr) > t


def build(force=False, verbose=True):
    """Compile every .cu for sm_90a and link the shared library. Returns the library path."""
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    objdir = OBJDIR
    os.makedirs(objdir, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-cudart", "static", "-Wno-deprecated-gpu-targets"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(STAMP, "w") as f:
        f.write(" ".join(NVCC_FLAGS))
    if verbose:
        print("built", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
