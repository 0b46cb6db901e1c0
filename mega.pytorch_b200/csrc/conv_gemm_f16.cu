// fp16-operand instantiations of the wgmma implicit-GEMM kernel (conv_gemm_kernel.cuh): f16 MMAs,
// fp32 accumulation in registers, fp32 or fp16 output. Separate translation unit so nvcc builds it in parallel with
// the TF32 variants.
#include "conv_gemm_kernel.cuh"

namespace mega {

template MEGA_LAUNCH_MODE(kModeF16);

}  // namespace mega
