// "3xFP16" instantiations of the wgmma implicit-GEMM kernel (conv_gemm_kernel.cuh, kModeF16x3): operands in the
// split-fp16 format (include/mega_b200.h), three f16 MMAs per k-step (hi.hi + hi.lo + lo.hi), fp32 accumulation in
// registers in segments folded round-to-nearest, output fp32 or split-fp16. Own translation unit: built in parallel.
#include "conv_gemm_kernel.cuh"

namespace mega {

template MEGA_LAUNCH_MODE(kModeF16x3);

}  // namespace mega
