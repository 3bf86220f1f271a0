"""Build libb2d.so (the C-ABI CUDA library) in-tree for sm_90a (H100) with nvcc.

Usage: ``python -m ray_lightning_b200.csrc.build`` or ``build_lib()``.  The shared object is
written next to the package (``ray_lightning_b200/lib/libb2d.so``, git-ignored), so the package
runs from the source tree.  nvcc cross-compiles without a GPU.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
LIB_DIR = os.path.join(PKG, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libb2d.so")
SOURCES = ["b2d.cu"]
HEADERS = ["b2d_device.cuh", "b2d_kernels.cuh", "b2d_tma.cuh", "b2d_staged.cuh", "b2d_owner.cuh", "b2d_syncbn.cuh", "b2d_clip.cuh", "b2d_launch.cuh", os.path.join("..", "..", "include", "b2d.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
    "-cudart", "static",
]


def find_nvcc():
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


def is_stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    for f in SOURCES + HEADERS:
        p = os.path.join(HERE, f)
        if os.path.exists(p) and os.path.getmtime(p) > t:
            return True
    return False


def build_lib(force=False, verbose=False):
    """Compile the library if it is missing or older than its sources. Returns its path."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = find_nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libb2d.so (expected /usr/local/cuda/bin/nvcc)")
    os.makedirs(LIB_DIR, exist_ok=True)
    tmp = LIB_PATH + ".tmp.%d" % os.getpid()
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + SOURCES + ["-ldl"]
    proc = subprocess.run(cmd, cwd=HERE, capture_output=True, text=True)
    if proc.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed (%d):\n%s\n%s" % (proc.returncode, proc.stdout, proc.stderr))
    os.replace(tmp, LIB_PATH)
    if verbose:
        sys.stderr.write(proc.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
