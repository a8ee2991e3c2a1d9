// TEST INFRASTRUCTURE: the emulator library of emu_kernels.cpp plus ProjE's sampler and step kernels
// (openea_b200/csrc/oea_proje.cu), so that the ProjE tests can run the kernels alone and whole training steps
// (sampler + step + row optimiser) on the CPU warp emulator.  Built by tests/emu/build_emu_proje.py; nothing under
// openea_b200/ loads it.
#include "emu_kernels.cpp"
#include <climits>

// the two device intrinsics the sampler uses beyond those of cuda_host_emu.h
inline int atomicMin(int* p, int v) { return emu_atomic_rmw<int>(p, [](int a, int b) { return a < b ? a : b; }, v); }
template <typename T>
inline T __ldcg(const T* p) { return std::atomic_ref<T>(*const_cast<T*>(p)).load(std::memory_order_relaxed); }

#include "../../openea_b200/csrc/oea_proje.cu"
