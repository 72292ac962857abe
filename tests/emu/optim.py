"""The host-emulated library with the fused Adamax step (TEST INFRASTRUCTURE ONLY): the sources of
tests/emu/build_emu.py plus iaf_b200/csrc/iaf_optim.cu, built into tests/emu/_build/libiaf_emu_optim.so.  The library
of build_emu.py is the C ABI without iaf_optim.cu, where iaf_adamax_step checks its arguments and then refuses; this one
registers the kernel, so the CPU suite executes it.  See cuda_emu.h for what the emulation is and is not."""
import ctypes as C
import os
import subprocess

from iaf_b200 import _lib as L
from . import build_emu as B

LIB = os.path.join(B.OUT, "libiaf_emu_optim.so")
SOURCES = B.SOURCES + [os.path.join(B.CSRC, "iaf_optim.cu")]

_lib = None


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(B.CSRC, f) for f in os.listdir(B.CSRC)] + \
           [os.path.join(B.HERE, f) for f in os.listdir(B.HERE) if f.endswith((".h", ".cc"))]
    deps.append(os.path.join(B.ROOT, "include", "iaf_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False):
    if not force and not _stale():
        return LIB
    os.makedirs(B.OUT, exist_ok=True)
    cmd = ["g++", "-std=c++20", "-O2", "-g", "-fPIC", "-shared", "-pthread", "-DIAF_EMU", "-Wno-unknown-pragmas",
           "-I", B.HERE, "-I", B.CSRC, "-o", LIB]
    for s in SOURCES:
        cmd += ["-x", "c++", s]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return LIB


def emu():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        for name, (res, args) in L.SYMBOLS.items():
            f = getattr(lib, name)
            f.restype = res
            f.argtypes = args
        _lib = lib
    return _lib
