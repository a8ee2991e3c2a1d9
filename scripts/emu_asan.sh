#!/bin/bash
# Memory-safety audit of the kernels without a GPU: the emulated library (tests/emu) built with AddressSanitizer, the
# emulator suites run against it.  ~5 min to build at -O0, ~15 min to run.
set -e
cd "$(dirname "$0")/.."
OUT=${OEA_EMU_ASAN_LIB:-/tmp/libemu_oea_asan.so}
g++ -std=c++20 -O0 -pthread -fPIC -shared -DOEA_HOST_EMU -fsanitize=address -fno-omit-frame-pointer \
    -Wno-attributes -Wno-unknown-pragmas -I "${CUDA_HOME:-/usr/local/cuda}/include" -o "$OUT" tests/emu/emu_kernels.cpp \
    -L"${CUDA_HOME:-/usr/local/cuda}/lib64" -lcudart
OEA_EMU_LIB="$OUT" LD_PRELOAD="$(gcc -print-file-name=libasan.so)" ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 \
    python -m pytest tests/test_emu_triple_core.py tests/test_emu_triple_grouped.py tests/test_emu_triple_ext.py \
    tests/test_emu_sampler.py tests/test_emu_spmm.py tests/test_emu_finding.py tests/test_reference_graph_goldens.py \
    -q -m "not gpu" -p no:cacheprovider
