// "3xFP16" instantiations of the wgmma implicit-GEMM kernel (conv_gemm_kernel.cuh, kModeF16x3): operands in the
// split-fp16 format (include/mega_b200.h), three f16 MMAs per k-step (hi.hi + hi.lo + lo.hi), fp32 accumulation in
// registers in segments folded round-to-nearest, output fp32 or split-fp16. Own translation unit: built in parallel.
#include "conv_gemm_kernel.cuh"

namespace mega {

int launch_conv_gemm_f16x3(int block_n, int out_split, const CUtensorMap& tmA, const CUtensorMap& tmB,
                           const CUtensorMap& tmOut, const CUtensorMap& tmRes, const ConvGemmParams& p, dim3 grid,
                           cudaStream_t stream, int pdl) {
  if (block_n == 64) {
    return out_split ? launch_cfg<64, 5, kModeF16x3, true>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl)
                     : launch_cfg<64, 5, kModeF16x3, false>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
  }
  if (block_n == 128) {
    return out_split ? launch_cfg<128, 4, kModeF16x3, true>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl)
                     : launch_cfg<128, 4, kModeF16x3, false>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
  }
  mega_set_error("conv_gemm: 3xfp16 supports block_n 64 / 128 (got %d)", block_n);
  return MEGA_ERR_ARG;
}

int launch_conv_gemm_f16x3_grouped(int gw, int out_split, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                                   const CUtensorMap& tmRes, const ConvGemmParams& p, dim3 grid, cudaStream_t stream, int pdl) {
  return out_split ? launch_grouped<5, kModeF16x3, true>(gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl)
                   : launch_grouped<5, kModeF16x3, false>(gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
}

}  // namespace mega
