"""CPU: the C-ABI library is built, loads without a GPU, and exports every symbol include/oea.h declares; so does the
emulated library of tests/emu."""
import ctypes
import glob
import os
import re

import pytest

from openea_b200 import lib as L


def test_header_symbols_all_bound_and_exported():
    declared = L.declared_symbols()
    assert declared, "no entry points parsed from include/oea.h"
    assert sorted(L.SIGNATURES) == declared, "openea_b200.lib.SIGNATURES must mirror include/oea.h exactly"
    assert os.path.exists(L.LIB_PATH), "liboea.so not built: run python -m openea_b200.build"
    raw = ctypes.CDLL(L.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), "liboea.so does not export " + name


def test_emulated_library_includes_every_kernel_source_and_exports_every_symbol():
    """tests/emu/emu_kernels.cpp includes every openea_b200/csrc/*.cu, so no entry point is out of the emulator's
    reach, and the library built from it exports every symbol include/oea.h declares."""
    from tests.emu import build_emu
    with open(build_emu.SRC) as f:
        included = set(re.findall(r'^#include "\.\./\.\./openea_b200/csrc/(\w+\.cu)"', f.read(), flags=re.M))
    sources = {os.path.basename(p) for p in glob.glob(os.path.join(build_emu.CSRC, "*.cu"))}
    assert included == sources, "emu_kernels.cpp misses %s" % sorted(sources - included)
    path = build_emu.build()
    if path is None:
        pytest.skip("no CUDA headers for the emulator build")
    raw = ctypes.CDLL(path)
    missing = [name for name in L.declared_symbols() if not hasattr(raw, name)]
    assert not missing, "the emulated library does not export " + ", ".join(missing)


def test_load_and_error_strings_without_gpu():
    lib = L.load()
    assert lib.oea_abi_version() == 1
    assert lib.oea_error_string(0) == b"ok"
    assert b"NULL" in lib.oea_error_string(1)
    # argument validation happens before any CUDA call: NULL tables are rejected with OEA_ERR_NULL
    rc = lib.oea_rowopt_apply(None, None, None)
    assert rc == 1


def test_sm90a_only():
    """The shared object carries sm_90a SASS (no multi-arch fatbin)."""
    import subprocess
    from openea_b200 import build
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")     # the toolkit's bin need not be on PATH
    out = subprocess.run([cuobjdump, "-lelf", L.LIB_PATH], capture_output=True, text=True).stdout
    archs = {line.split(".")[-2] for line in out.splitlines() if ".cubin" in line}
    assert archs == {"sm_90a"}, archs
