// Baseline JPEG decode, device stage and C entry points (SURVEY.md section 8f row 1): replaces
// `PIL.Image.open(path).convert("RGB")` in front of mega_image_transform_u8 with the same pixels. The host stage
// (jpeg_host.cuh) leaves quantised coefficients; two kernels serve a whole batch of images of different sizes:
//   jpeg_idct_kernel   coefficients -> uint8 component planes padded to whole MCUs. 8 threads per 8x8 block (a thread
//                      per column, then per row, exchanged through shared memory), 32 blocks per CTA. Reads 2 bytes and
//                      writes 1 byte per sample; quantisation tables come from the descriptor table through L1.
//   jpeg_color_kernel  per 4 pixels of a row: chroma upsampling, colour conversion, planar uint8 [3, H, W] cropped to
//                      the image, one 32-bit store per plane. Reads 1.5 and writes 3 bytes per pixel at 4:2:0.
// Both find their image by binary search in the device-side descriptor table, so the 23 frames that open a MEGA video
// cost two launches. Arithmetic: jpeg_decode.cuh.
#include "common.cuh"
#include "jpeg_decode.cuh"
#include "jpeg_host.cuh"
#include "mega_b200.h"

namespace mega {

constexpr int kIdctThreads = 256;   // 32 blocks of 8 threads

__global__ void __launch_bounds__(kIdctThreads) jpeg_idct_kernel(const mega_jpeg_desc* __restrict__ descs, int n,
                                                                 long long total_blocks,
                                                                 const int16_t* __restrict__ coef,
                                                                 uint8_t* __restrict__ planes) {
  __shared__ int ws[(kIdctThreads / 8) * mega_jpeg::kWsStride];
  const int sub = threadIdx.x >> 3, lane8 = threadIdx.x & 7;
  const long long b = static_cast<long long>(blockIdx.x) * (kIdctThreads / 8) + sub;
  const bool live = b < total_blocks;
  int* my = ws + sub * mega_jpeg::kWsStride;
  mega_jpeg::BlockPlace place;
  if (live) {
    place = mega_jpeg::place_block(descs, n, b);
    mega_jpeg::idct_column(coef + b * 64, place.d->quant[place.comp], lane8, my);
  }
  __syncwarp();                      // the 8 threads of a block sit in one warp
  if (live) {
    const uint64_t row = mega_jpeg::idct_row(my, lane8);
    *reinterpret_cast<uint2*>(planes + place.plane_off + static_cast<long long>(lane8) * place.stride) =
        make_uint2(static_cast<uint32_t>(row), static_cast<uint32_t>(row >> 32));
  }
}

__global__ void jpeg_color_kernel(const mega_jpeg_desc* __restrict__ descs, int n, long long total_quads,
                                  const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
  const long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (q < total_quads) mega_jpeg::color_item(descs, n, q, planes, out);
}

}  // namespace mega

extern "C" int mega_jpeg_probe(const unsigned char* data, long long size, mega_jpeg_info* info) {
  MEGA_ARG_CHECK(data && info && size >= 0, "jpeg_probe: null argument");
  const int st = mega_jpeg::decode_host(data, size, info, nullptr, 0);
  if (st != MEGA_OK) mega_set_error("jpeg_probe: %s", st == MEGA_JPEG_UNSUPPORTED ? "stream outside the supported baseline subset" : "damaged or truncated stream");
  return st;
}

extern "C" int mega_jpeg_entropy_decode(const unsigned char* data, long long size, mega_jpeg_info* info, short* coef,
                                        long long coef_capacity_blocks) {
  MEGA_ARG_CHECK(data && info && coef && size >= 0 && coef_capacity_blocks > 0, "jpeg_entropy_decode: null argument");
  const int st = mega_jpeg::decode_host(data, size, info, coef, coef_capacity_blocks);
  if (st != MEGA_OK)
    mega_set_error("jpeg_entropy_decode: %s", st == MEGA_JPEG_UNSUPPORTED ? "stream outside the supported baseline subset"
                                              : st == MEGA_JPEG_CORRUPT   ? "damaged or truncated stream"
                                                                          : "coefficient buffer smaller than the frame");
  return st;
}

extern "C" int mega_jpeg_plan_batch(const mega_jpeg_info* infos, int n, mega_jpeg_desc* descs, long long* totals) {
  MEGA_ARG_CHECK(infos && descs && totals && n > 0, "jpeg_plan_batch: null argument");
  MEGA_ARG_CHECK(mega_jpeg::plan_batch(infos, n, descs, totals) == 0, "jpeg_plan_batch: an image descriptor is inconsistent");
  return MEGA_OK;
}

extern "C" int mega_jpeg_decode_batch(const mega_jpeg_desc* descs_host, const mega_jpeg_desc* descs_dev, int n,
                                      const short* coef_dev, unsigned char* planes_dev, long long planes_bytes,
                                      unsigned char* out_dev, long long out_bytes, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(descs_host && descs_dev && coef_dev && planes_dev && out_dev && n > 0, "jpeg_decode_batch: null argument");
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(planes_dev) & 7) == 0 && (reinterpret_cast<uintptr_t>(out_dev) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(coef_dev) & 1) == 0 && (reinterpret_cast<uintptr_t>(descs_dev) & 7) == 0,
                 "jpeg_decode_batch: planes must be 8-byte, out 4-byte aligned");
  long long blocks = 0, quads = 0;
  MEGA_ARG_CHECK(mega_jpeg::batch_fits(descs_host, n, planes_bytes, out_bytes, &blocks, &quads),
                 "jpeg_decode_batch: descriptors do not fit the buffers (use mega_jpeg_plan_batch)");
  const long long g1 = (blocks + mega::kIdctThreads / 8 - 1) / (mega::kIdctThreads / 8), g2 = (quads + 255) / 256;
  MEGA_ARG_CHECK(g1 < (1LL << 31) && g2 < (1LL << 31), "jpeg_decode_batch: batch too large");
  mega::jpeg_idct_kernel<<<static_cast<unsigned>(g1), mega::kIdctThreads, 0, stream>>>(descs_dev, n, blocks, coef_dev, planes_dev);
  MEGA_CUDA_CHECK(cudaGetLastError());
  mega::jpeg_color_kernel<<<static_cast<unsigned>(g2), 256, 0, stream>>>(descs_dev, n, quads, planes_dev, out_dev);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
