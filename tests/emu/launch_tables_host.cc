// TEST INFRASTRUCTURE. launch_tables.cc compiled for the host emulations: the kernel headers it includes carry the
// device code of the entropy kernels, which needs cuda_shim.h's host stand-ins for the CUDA intrinsics under g++.
#include "cuda_shim.h"

#include "../../jxl_oxide_b200/csrc/launch_tables.cc"
