"""Builds and loads tests/emu/libemu_oea.so: every product kernel source on the CPU warp emulator (test infrastructure)."""
import ctypes
import glob
import os
import subprocess

import pytest

from openea_b200 import lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "libemu_oea.so")
SRC = os.path.join(HERE, "emu_kernels.cpp")
CSRC = os.path.join(ROOT, "openea_b200", "csrc")
EMU_H = os.path.join(HERE, "cuda_host_emu.h")
# every kernel source and header: adding or editing one can never leave a stale library passing
DEPS = [SRC, EMU_H, os.path.join(ROOT, "include", "oea.h")] + sorted(glob.glob(os.path.join(CSRC, "*.cu"))) + \
    sorted(glob.glob(os.path.join(CSRC, "*.cuh")))


def cuda_include():
    for root in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if root and os.path.exists(os.path.join(root, "include", "cuda_runtime.h")):
            return os.path.join(root, "include")
    return None


def compile(main_cpp, out, extra_flags=()):
    """g++ the translation unit `main_cpp` (cuda_host_emu.h, then kernel sources) into the shared library `out`, written
    through a temporary file so that a concurrent builder (a runner subprocess, a gloo worker) never loads half of one.
    `extra_flags` come last, so they override the defaults (e.g. -O0 for a sanitizer build)."""
    inc = cuda_include()
    tmp = "%s.%d.tmp" % (out, os.getpid())
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DOEA_HOST_EMU", "-Wno-attributes",
           "-Wno-unknown-pragmas", *extra_flags, "-I", inc, "-I", HERE, "-o", tmp, main_cpp,
           "-L", os.path.join(os.path.dirname(inc), "lib64"), "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("emulator build failed:\n" + res.stderr[-4000:])
    os.replace(tmp, out)
    return out


def _fresh(out, deps):
    return os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps)


def build(force=False):
    """The emulated library's path; None without CUDA headers.  OEA_EMU_LIB names a prebuilt one instead (the
    AddressSanitizer build of scripts/emu_asan.sh)."""
    prebuilt = os.environ.get("OEA_EMU_LIB")
    if prebuilt:
        return prebuilt
    if cuda_include() is None:
        return None
    if force or not _fresh(OUT, DEPS):
        compile(SRC, OUT)
    return OUT


def build_selftest(force=False):
    """tests/emu/libemu_selftest.so: the emulator's own collectives checked against CUDA's documented behaviour."""
    if cuda_include() is None:
        return None
    src, out = os.path.join(HERE, "emu_selftest.cpp"), os.path.join(HERE, "libemu_selftest.so")
    if force or not _fresh(out, [src, EMU_H]):
        compile(src, out)
    return out


def load(path=None, names=None):
    """The emulated library at `path` (default: build()) with the signature of every entry point in `names` (default:
    all of openea_b200.lib.SIGNATURES) bound; a missing entry point raises.  Skips the calling test without CUDA
    headers."""
    path = path or build()
    if path is None:
        pytest.skip("no CUDA headers for the emulator build")
    lib = ctypes.CDLL(path)
    for name in L.SIGNATURES if names is None else names:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = L.SIGNATURES[name]
    return lib


def patch_engine(monkeypatch, lib):
    """Serves the product's host layer from `lib`: openea_b200.lib.load() returns it, and the engine, finding and gnn
    modules pass a NULL stream (the emulator's launches are synchronous)."""
    from openea_b200 import engine, finding, gnn
    monkeypatch.setattr(L, "load", lambda: lib)
    for module in (engine, finding, gnn):
        monkeypatch.setattr(module, "_stream_ptr", lambda: ctypes.c_void_p(0))


if __name__ == "__main__":
    print(build(force=True))
