// conv_tc_kernel<NB> instantiations for NB = 80 and 96 (see conv_tc_kernel.cuh); one translation unit per pair keeps the build parallel.
#include "conv_tc_kernel.cuh"

namespace fs2 {

FS2_CONV_TC_NB_DEF(80)
FS2_CONV_TC_NB_DEF(96)

}  // namespace fs2
