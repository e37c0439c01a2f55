"""In-tree build of librnnt_b200.so for the H100 (nvcc cross-compiles sm_90a without a GPU).

The shared object is a build product: git ignores it, `build()` (or `load()` when it is missing) makes it.
"""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "rnnt_b200.cu")
OUT = os.environ.get("RNNTB200_BUILD_OUT") or os.path.join(HERE, "librnnt_b200.so")
DEPS = [SRC] + [os.path.join(HERE, "csrc", f) for f in sorted(os.listdir(os.path.join(HERE, "csrc"))) if f.endswith(".cuh")] + [
    os.path.join(os.path.dirname(HERE), "include", "rnnt_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC", "-diag-suppress", "177"]


def nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def is_stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    """Compile csrc/rnnt_b200.cu -> librnnt_b200.so for sm_90a.  Returns the .so path."""
    if not force and not is_stale():
        return OUT
    if not os.path.exists(nvcc()):
        raise RuntimeError("nvcc not found and %s is missing/stale" % OUT)
    flags = list(NVCC_FLAGS)
    if os.environ.get("RNNTB200_NO_TC") == "1":      # bring-up switch: CUDA-core kernels only
        flags += ["-DRNNTB200_NO_TC"]
    cmd = [nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + [SRC, "-o", OUT + ".tmp"]
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    os.replace(OUT + ".tmp", OUT)
    if verbose:
        print(r.stderr)
    return OUT


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
