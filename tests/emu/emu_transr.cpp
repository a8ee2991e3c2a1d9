// TEST INFRASTRUCTURE: the emulator library of emu_kernels.cpp plus TransR's relation-grouped kernels
// (openea_b200/csrc/oea_triple_transr.cu), so that the TransR tests can run the kernels alone and whole training steps
// (scorer + row optimiser) on the CPU warp emulator.  Built by tests/emu/build_emu_transr.py; nothing under openea_b200/
// loads it.
#include "emu_kernels.cpp"
#include "../../openea_b200/csrc/oea_triple_transr.cu"
