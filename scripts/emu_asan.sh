#!/bin/bash
# Memory-safety audit of the kernels without a GPU: the emulated library (tests/emu) built with AddressSanitizer, the
# emulator suites run against it.  ~5 min to build at -O0, ~15 min to run.
set -e
cd "$(dirname "$0")/.."
OUT=${OEA_EMU_ASAN_LIB:-/tmp/libemu_oea_asan.so}
python -c "import sys; from tests.emu import build_emu
build_emu.compile(build_emu.SRC, sys.argv[1], ('-O0', '-fsanitize=address', '-fno-omit-frame-pointer'))" "$OUT"
OEA_EMU_LIB="$OUT" LD_PRELOAD="$(gcc -print-file-name=libasan.so)" ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 \
    python -m pytest tests/test_emu_triple_core.py tests/test_emu_triple_grouped.py tests/test_emu_triple_ext.py \
    tests/test_emu_sampler.py tests/test_emu_spmm.py tests/test_emu_finding.py tests/test_reference_graph_goldens.py \
    tests/test_emu_transr.py tests/test_emu_proje.py tests/test_transr_goldens.py \
    -q -m "not gpu" -p no:cacheprovider
