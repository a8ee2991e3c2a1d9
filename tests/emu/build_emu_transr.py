"""Builds tests/emu/libemu_transr.so: the warp-emulator library of build_emu.py plus TransR's kernel source
(emu_transr.cpp), with the same compiler flags (test infrastructure).

`OEA_EMU_LIB` names a prebuilt emulator library for build_emu.build(); the TransR tests point it at this one, so that
the shared runners (tests/emu/fake_cuda.py, the cpu_engine fixture) serve the TransR entry points too."""
import os
import subprocess

from tests.emu import build_emu

OUT = os.path.join(build_emu.HERE, "libemu_transr.so")
SRC = os.path.join(build_emu.HERE, "emu_transr.cpp")
DEPS = build_emu.DEPS + [SRC, os.path.join(build_emu.CSRC, "oea_triple_transr.cu")]


def build(force=False):
    inc = build_emu.cuda_include()
    if inc is None:
        return None
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    tmp = "%s.%d.tmp" % (OUT, os.getpid())          # concurrent builders never load a half-written library
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DOEA_HOST_EMU",
           "-Wno-attributes", "-Wno-unknown-pragmas", "-I", inc, "-o", tmp, SRC,
           "-L", os.path.join(os.path.dirname(inc), "lib64"), "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("emulator build failed:\n" + res.stderr[-4000:])
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    print(build(force=True))
