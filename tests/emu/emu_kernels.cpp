// TEST INFRASTRUCTURE: every product kernel source compiled for the CPU warp emulator (cuda_host_emu.h) into one
// library, which exports the C-ABI entry points of include/oea.h over host pointers ("device" pointers are host
// pointers).  tests/test_abi_exports.py checks that every openea_b200/csrc/*.cu is included here.  Nothing under
// openea_b200/ loads it.
#include "cuda_host_emu.h"
#include "../../openea_b200/csrc/oea_match.cu"
#include "../../openea_b200/csrc/oea_optim_ext.cu"
#include "../../openea_b200/csrc/oea_p2p.cu"
#include "../../openea_b200/csrc/oea_pipeline.cu"
#include "../../openea_b200/csrc/oea_proje.cu"
#include "../../openea_b200/csrc/oea_sampler.cu"
#include "../../openea_b200/csrc/oea_sim.cu"
#include "../../openea_b200/csrc/oea_sim_tc.cu"
#include "../../openea_b200/csrc/oea_spmm.cu"
#include "../../openea_b200/csrc/oea_triple.cu"
#include "../../openea_b200/csrc/oea_triple_ext.cu"
#include "../../openea_b200/csrc/oea_triple_grouped.cu"
#include "../../openea_b200/csrc/oea_triple_transr.cu"
#include "../../openea_b200/csrc/oea_triple_weighted.cu"
