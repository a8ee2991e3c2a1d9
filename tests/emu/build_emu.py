"""Builds tests/emu/libemu_oea.so: the product's kernel sources on the CPU warp emulator (test infrastructure)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "libemu_oea.so")
SRC = os.path.join(HERE, "emu_kernels.cpp")
CSRC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "openea_b200", "csrc")
DEPS = [SRC, os.path.join(HERE, "cuda_host_emu.h")] + [os.path.join(CSRC, f) for f in
                                                        ("oea_triple_ext.cu", "oea_sampler.cu", "oea_optim_ext.cu", "oea_triple_grouped.cu", "oea_triple_weighted.cu", "oea_spmm.cu", "oea_triple.cu", "oea_sim.cu", "oea_pipeline.cu", "oea_match.cu", "oea_p2p.cu", "oea_sampler.cuh", "oea_rowmath.cuh", "oea_common.cuh")]


def cuda_include():
    for root in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if root and os.path.exists(os.path.join(root, "include", "cuda_runtime.h")):
            return os.path.join(root, "include")
    return None


def build(force=False):
    prebuilt = os.environ.get("OEA_EMU_LIB")          # e.g. a build with -fsanitize=address,undefined (see DESIGN.md §2)
    if prebuilt:
        return prebuilt
    inc = cuda_include()
    if inc is None:
        return None
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DOEA_HOST_EMU",
           "-Wno-attributes", "-Wno-unknown-pragmas", "-I", inc, "-o", OUT, SRC,
           "-L", os.path.join(os.path.dirname(inc), "lib64"), "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("emulator build failed:\n" + res.stderr[-4000:])
    return OUT


def build_selftest(force=False):
    """tests/emu/libemu_selftest.so: the emulator's own collectives checked against CUDA's documented behaviour."""
    inc = cuda_include()
    if inc is None:
        return None
    src, out = os.path.join(HERE, "emu_selftest.cpp"), os.path.join(HERE, "libemu_selftest.so")
    deps = [src, os.path.join(HERE, "cuda_host_emu.h")]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-Wno-attributes", "-I", inc, "-o", out, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("emulator self-test build failed:\n" + res.stderr[-4000:])
    return out


if __name__ == "__main__":
    print(build(force=True))
