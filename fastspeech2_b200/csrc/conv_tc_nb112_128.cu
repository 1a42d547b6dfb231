// conv_tc_kernel<NB> instantiations for NB = 112 and 128 (see conv_tc_kernel.cuh); one translation unit per pair keeps the build parallel.
#include "conv_tc_kernel.cuh"

namespace fs2 {

FS2_CONV_TC_NB_DEF(112)
FS2_CONV_TC_NB_DEF(128)

}  // namespace fs2
