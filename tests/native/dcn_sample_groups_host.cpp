// Host build of the grouped deformable sampling of csrc/dcn_sample.cu -- TEST INFRASTRUCTURE ONLY.
// g++ compiles the shared geometry / interpolation of csrc/dcn_sample.cuh and walks (pixel, group, tap, channel)
// serially in the kernel's arithmetic, so the CPU tests check it against oracle/train_ops_oracle.py with several
// deformable groups and the GPU tests check the kernel against this build bit for bit. Same name and prototype as the
// C ABI entry point (the header is included, so a drifting signature does not compile); pointers are host pointers,
// `stream` is ignored, MEGA_DCN_FP32 only.
// Build: g++ -O2 -fPIC -shared -std=c++17 -I mega.pytorch_b200/csrc -I include -o libdcn_sample_groups_host.so \
//        dcn_sample_groups_host.cpp
#include "mega_b200.h"
#include "dcn_sample.cuh"

using namespace mega;

extern "C" int mega_dcn_sample_nhwc_groups(const void* input, int format, int batch, int height, int width,
                                           int channels, int deformable_groups, const float* offset, int offset_ld,
                                           int modulated, int stride, int dil, void* cols, void* stream) {
  (void)stream;
  const int dg = deformable_groups;
  if (format != MEGA_DCN_FP32 || channels % 32 != 0 || dg < 1 || channels % dg != 0 || (channels / dg) % 8 != 0 ||
      (modulated && dg != 1) || offset_ld < (modulated ? 27 : 18 * dg))
    return 1;
  const float* in = static_cast<const float*>(input);
  float* out = static_cast<float*>(cols);
  const int ho = (height - 1) / stride + 1, wo = (width - 1) / stride + 1, cpg = channels / dg;
  const long long plane = static_cast<long long>(height) * width;
  for (long long pix = 0; pix < static_cast<long long>(batch) * ho * wo; ++pix) {
    const int w_col = static_cast<int>(pix % wo), h_col = static_cast<int>((pix / wo) % ho);
    const long long img = pix / (static_cast<long long>(ho) * wo) * plane;
    const float* o = offset + pix * offset_ld;
    for (int g = 0; g < dg; ++g) {
      for (int tap = 0; tap < 9; ++tap) {
        const int i = tap / 3, j = tap - 3 * i;
        const float h_im = h_col * stride - dil + i * dil + o[18 * g + 2 * tap];
        const float w_im = w_col * stride - dil + j * dil + o[18 * g + 2 * tap + 1];
        const DcnTap t = dcn_tap_geometry(h_im, w_im, height, width);
        const float m = modulated ? dcn_sigmoid(o[18 + tap]) : 1.f;
        float* row = out + pix * 9 * channels + tap * channels;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
          if (t.i00 == kDcnOutside) {
            row[c] = 0.f;
            continue;
          }
          const float v00 = t.i00 >= 0 ? in[(img + t.i00) * channels + c] : 0.f;
          const float v01 = t.i01 >= 0 ? in[(img + t.i01) * channels + c] : 0.f;
          const float v10 = t.i10 >= 0 ? in[(img + t.i10) * channels + c] : 0.f;
          const float v11 = t.i11 >= 0 ? in[(img + t.i11) * channels + c] : 0.f;
          row[c] = dcn_blend(t, v00, v01, v10, v11) * m;
        }
      }
    }
  }
  return 0;
}
