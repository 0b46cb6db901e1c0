// fp16-operand instantiations of the wgmma implicit-GEMM kernel (conv_gemm_kernel.cuh): f16 MMAs,
// fp32 accumulation in registers, fp32 or fp16 output. Separate translation unit so nvcc builds it in parallel with
// the TF32 variants.
#include "conv_gemm_kernel.cuh"

namespace mega {

int launch_conv_gemm_f16(int block_n, int out_f16, const CUtensorMap& tmA, const CUtensorMap& tmB,
                         const CUtensorMap& tmOut, const CUtensorMap& tmRes, const ConvGemmParams& p, dim3 grid,
                         cudaStream_t stream, int pdl) {
  if (out_f16 && block_n % 64 != 0) {
    mega_set_error("conv_gemm: fp16 output needs block_n %% 64 == 0 (got %d)", block_n);
    return MEGA_ERR_ARG;
  }
#define MEGA_F16_CASE(BN, ST)                                                                                  \
  case BN:                                                                                                     \
    return out_f16 ? launch_cfg<BN, ST, kModeF16, (BN % 64 == 0)>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl) \
                   : launch_cfg<BN, ST, kModeF16, false>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
  switch (block_n) {
    MEGA_F16_CASE(32, 6)
    MEGA_F16_CASE(64, 5)
    MEGA_F16_CASE(96, 4)
    MEGA_F16_CASE(128, 4)
    MEGA_F16_CASE(160, 3)
    MEGA_F16_CASE(192, 3)
    MEGA_F16_CASE(256, 2)
  }
#undef MEGA_F16_CASE
  mega_set_error("conv_gemm: unsupported block_n %d", block_n);
  return MEGA_ERR_ARG;
}

int launch_conv_gemm_f16_grouped(int gw, int out_f16, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                                 const CUtensorMap& tmRes, const ConvGemmParams& p, dim3 grid, cudaStream_t stream, int pdl) {
  return out_f16 ? launch_grouped<5, kModeF16, true>(gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl)
                 : launch_grouped<5, kModeF16, false>(gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
}

}  // namespace mega
