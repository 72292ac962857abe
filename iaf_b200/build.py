"""Build libiaf_b200.so in-tree with nvcc for sm_90a (Hopper; no JIT cache, no torch extension)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libiaf_b200.so")
SOURCES = ["iaf_capi.cu", "iaf_pack.cu", "iaf_simt.cu", "iaf_tc.cu", "iaf_bwd.cu", "iaf_inv.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _stale(lib):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "iaf_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, lib=LIB, defines=()):
    """Compile the CUDA sources into `lib` (default iaf_b200/lib/libiaf_b200.so) with -D`defines`.  Returns the path."""
    if not force and not _stale(lib):
        return lib
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    cmd = ([_nvcc()] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) +
           ["-o", lib] + SOURCES)
    r = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return lib


if __name__ == "__main__":
    print(build(force=True, verbose=True))
