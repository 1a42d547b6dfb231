// conv_tc_kernel<NB> instantiations for NB = 48 and 64 (see conv_tc_kernel.cuh); one translation unit per pair keeps the build parallel.
#include "conv_tc_kernel.cuh"

namespace fs2 {

FS2_CONV_TC_NB_DEF(48)
FS2_CONV_TC_NB_DEF(64)

}  // namespace fs2
