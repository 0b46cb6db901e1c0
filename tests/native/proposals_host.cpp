// Host build of csrc/box_head.cuh and csrc/iou.cuh -- TEST INFRASTRUCTURE ONLY.
// g++ compiles the per-element bodies the proposal and post-processing kernels run: decode + clip, the class soft-max
// and the IoU threshold decision, one call per element, for the exact-order fp32 restatement of
// tests/proposals_ref.py to be compared against bit for bit (expf is the host libm's).
// Build: g++ -O2 -fPIC -shared -std=c++17 -ffp-contract=off -I mega.pytorch_b200/csrc -o libproposals_host.so
//            proposals_host.cpp
#include "box_head.cuh"

using namespace mega;

extern "C" {

// out[i] = decode_clip_box(d + 4 i, box i) with weights w[4]
void proposals_decode_clip(const float* d, const float* box, int n, const float* w, float im_w, float im_h,
                           float* out) {
  const BoxCoderW bw{w[0], w[1], w[2], w[3]};
  for (int i = 0; i < n; ++i) {
    const float4 b{box[4 * i], box[4 * i + 1], box[4 * i + 2], box[4 * i + 3]};
    const float4 o = decode_clip_box(d + 4 * i, b, bw, im_w, im_h);
    out[4 * i] = o.x, out[4 * i + 1] = o.y, out[4 * i + 2] = o.z, out[4 * i + 3] = o.w;
  }
}

// out[r, j] = class_softmax_prob(row r, nc, j)
void proposals_softmax(const float* l, int rows, int nc, float* out) {
  for (int r = 0; r < rows; ++r)
    for (int j = 0; j < nc; ++j) out[r * nc + j] = class_softmax_prob(l + r * nc, nc, j);
}

// out[i] = iou_plus1_gt(a_i, b_i) at thresh, with the kernels' t_lo / t_hi band
void proposals_iou_gt(const float* a, const float* b, int n, float thresh, unsigned char* out) {
  const float t_lo = thresh * (1.f - 9.5367431640625e-07f), t_hi = thresh * (1.f + 9.5367431640625e-07f);
  for (int i = 0; i < n; ++i) {
    const float4 x{a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]};
    const float4 y{b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]};
    out[i] = iou_plus1_gt(x, box_area_plus1(x), y, box_area_plus1(y), thresh, t_lo, t_hi) ? 1 : 0;
  }
}

}  // extern "C"
