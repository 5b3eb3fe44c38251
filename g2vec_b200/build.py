"""Build libg2vec_b200.so (hand-written sm_90a CUDA + the C ABI of include/g2vec_b200.h).

nvcc cross-compiles without a GPU; the .so is built IN-TREE (g2vec_b200/libg2vec_b200.so,
git-ignored) so that it travels to the GPU box with the repo snapshot.
"""
import glob
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libg2vec_b200.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "--expt-relaxed-constexpr",
]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libg2vec_b200.so cannot be built")


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False, extra=()):
    """Compile into a temporary file and rename it over LIB while holding an exclusive file lock, so that the
    ranks of a torchrun launch that all find the library stale neither compile into the same output nor dlopen
    a half-written file: the first rank builds, the others wait on the lock and then find it fresh."""
    import fcntl
    if not force and not stale():
        return LIB
    with open(LIB + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not stale():          # another process built it while we waited
                return LIB
            tmp = "%s.tmp.%d" % (LIB, os.getpid())
            cmd = [nvcc_path()] + NVCC_FLAGS + list(extra) + ["-I", os.path.join(ROOT, "include"), "-I", CSRC,
                                                              "-o", tmp] + sources()
            if verbose:
                print(" ".join(cmd))
            try:
                subprocess.check_call(cmd)
                os.replace(tmp, LIB)
            finally:
                if os.path.exists(tmp):
                    os.remove(tmp)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    import sys
    build_library(force=True, verbose=True, extra=["-Xptxas", "-v"] if "-v" in sys.argv else [])
    print(LIB)
