"""Builds tests/emu/libemu_proje.so: the warp-emulator library of build_emu.py plus ProjE's kernel source
(emu_proje.cpp), with the same compiler flags (test infrastructure).  The ProjE tests load it directly, and the lifecycle
test hands it to the engine in place of liboea.so."""
import os
import subprocess

from tests.emu import build_emu

OUT = os.path.join(build_emu.HERE, "libemu_proje.so")
SRC = os.path.join(build_emu.HERE, "emu_proje.cpp")
DEPS = build_emu.DEPS + [SRC, os.path.join(build_emu.CSRC, "oea_proje.cu")]


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
