// conv_tc_kernel<NB> instantiations for NB = 16 and 32 (see conv_tc_kernel.cuh); one translation unit per pair keeps the build parallel.
#include "conv_tc_kernel.cuh"

namespace fs2 {

FS2_CONV_TC_NB_DEF(16)
FS2_CONV_TC_NB_DEF(32)

}  // namespace fs2
