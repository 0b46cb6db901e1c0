// Host build of csrc/jpeg_host.cuh + csrc/jpeg_decode.cuh -- TEST INFRASTRUCTURE ONLY (see train_ops_host.cpp): the
// library's own entropy decoder (also built with -fsanitize=address,undefined for the damaged-stream tests) and the
// very bodies the two CUDA kernels run, block by block and item by item, under the C-ABI prototypes of
// include/mega_b200.h with host pointers; `stream` is ignored.
// Build: g++ -O2 -fPIC -shared -std=c++17 -I mega.pytorch_b200/csrc -I include -o libjpeg_decode_host.so jpeg_decode_host.cpp
#include "mega_b200.h"
#include "jpeg_decode.cuh"
#include "jpeg_host.cuh"

extern "C" int mega_jpeg_probe(const unsigned char* data, long long size, mega_jpeg_info* info) {
  return mega_jpeg::decode_host(data, size, info, nullptr, 0);
}

extern "C" int mega_jpeg_entropy_decode(const unsigned char* data, long long size, mega_jpeg_info* info, short* coef,
                                        long long coef_capacity_blocks) {
  if (!coef || coef_capacity_blocks <= 0) return 1;
  return mega_jpeg::decode_host(data, size, info, coef, coef_capacity_blocks);
}

extern "C" int mega_jpeg_plan_batch(const mega_jpeg_info* infos, int n, mega_jpeg_desc* descs, long long* totals) {
  return mega_jpeg::plan_batch(infos, n, descs, totals);
}

extern "C" int mega_jpeg_decode_batch(const mega_jpeg_desc* descs_host, const mega_jpeg_desc* descs_dev, int n,
                                      const short* coef_dev, unsigned char* planes_dev, long long planes_bytes,
                                      unsigned char* out_dev, long long out_bytes, void* stream) {
  (void)stream;
  long long blocks = 0, quads = 0;
  if (!mega_jpeg::batch_fits(descs_host, n, planes_bytes, out_bytes, &blocks, &quads)) return 1;
  int ws[mega_jpeg::kWsStride];
  for (long long b = 0; b < blocks; ++b) {
    const mega_jpeg::BlockPlace place = mega_jpeg::place_block(descs_dev, n, b);
    for (int col = 0; col < 8; ++col) mega_jpeg::idct_column(coef_dev + b * 64, place.d->quant[place.comp], col, ws);
    for (int row = 0; row < 8; ++row) {
      const uint64_t v = mega_jpeg::idct_row(ws, row);
      for (int k = 0; k < 8; ++k) planes_dev[place.plane_off + static_cast<long long>(row) * place.stride + k] = static_cast<unsigned char>(v >> (8 * k));
    }
  }
  for (long long q = 0; q < quads; ++q) mega_jpeg::color_item(descs_dev, n, q, planes_dev, out_dev);
  return 0;
}
