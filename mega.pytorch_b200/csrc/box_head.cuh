// Per-(proposal, class) arithmetic of the box-head post-processor, shared by box_class_nms_kernel (postprocess.cu) and
// the test-time augmentation collect kernel (bbox_aug.cu): softmax probability of one class, BoxCoder.decode with the
// BBOX_REG_WEIGHTS (box_coder.py:52-95) and clip_to_image(remove_empty=False) (bounding_box.py). Every fp32 operation
// is a separately rounded IEEE operation in the reference's order; __host__ __device__ so the g++ builds under
// tests/native run the same code (expf is the one libm call: host and device may differ in its last bit).
#pragma once
#include "iou.cuh"

namespace mega {

struct BoxCoderW {
  float wx, wy, ww, wh;
};

// F.softmax(class_logits, -1)[j] of one row of nc logits
MEGA_IOU_HD float class_softmax_prob(const float* l, int nc, int j) {
  float mx = l[0];
  for (int c = 1; c < nc; ++c) mx = fmaxf(mx, l[c]);
  float sum = 0.f;
  for (int c = 0; c < nc; ++c) sum = MEGA_IOU_ADD(sum, expf(MEGA_IOU_SUB(l[c], mx)));
  return MEGA_IOU_DIV(expf(MEGA_IOU_SUB(l[j], mx)), sum);
}

// decode deltas d[0..3] against proposal `box`, then clip to an im_w x im_h image
MEGA_IOU_HD float4 decode_clip_box(const float* d, const float4 box, const BoxCoderW w, float im_w, float im_h) {
  const float widths = MEGA_IOU_ADD(MEGA_IOU_SUB(box.z, box.x), 1.f), heights = MEGA_IOU_ADD(MEGA_IOU_SUB(box.w, box.y), 1.f);
  const float ctr_x = MEGA_IOU_ADD(box.x, MEGA_IOU_MUL(0.5f, widths)), ctr_y = MEGA_IOU_ADD(box.y, MEGA_IOU_MUL(0.5f, heights));
  const float clipv = 4.135166556742356f;
  const float dx = MEGA_IOU_DIV(d[0], w.wx), dy = MEGA_IOU_DIV(d[1], w.wy);
  const float dw = fminf(MEGA_IOU_DIV(d[2], w.ww), clipv), dh = fminf(MEGA_IOU_DIV(d[3], w.wh), clipv);
  const float pcx = MEGA_IOU_ADD(MEGA_IOU_MUL(dx, widths), ctr_x), pcy = MEGA_IOU_ADD(MEGA_IOU_MUL(dy, heights), ctr_y);
  const float pw = MEGA_IOU_MUL(expf(dw), widths), ph = MEGA_IOU_MUL(expf(dh), heights);
  float4 o;
  o.x = MEGA_IOU_SUB(pcx, MEGA_IOU_MUL(0.5f, pw));
  o.y = MEGA_IOU_SUB(pcy, MEGA_IOU_MUL(0.5f, ph));
  o.z = MEGA_IOU_SUB(MEGA_IOU_ADD(pcx, MEGA_IOU_MUL(0.5f, pw)), 1.f);
  o.w = MEGA_IOU_SUB(MEGA_IOU_ADD(pcy, MEGA_IOU_MUL(0.5f, ph)), 1.f);
  o.x = fminf(fmaxf(o.x, 0.f), MEGA_IOU_SUB(im_w, 1.f));
  o.y = fminf(fmaxf(o.y, 0.f), MEGA_IOU_SUB(im_h, 1.f));
  o.z = fminf(fmaxf(o.z, 0.f), MEGA_IOU_SUB(im_w, 1.f));
  o.w = fminf(fmaxf(o.w, 0.f), MEGA_IOU_SUB(im_h, 1.f));
  return o;
}

#if defined(__CUDACC__)
// inputs of box_final_kernel (postprocess.cu): class-major staging [num_classes][r_max] -> the frame's detections
struct FinalParams {
  const float4* cls_boxes;
  const float* cls_scores;
  const unsigned char* cls_keep;
  int r_max, num_classes, max_det, out_cap;
  float* out_boxes;        // [out_cap,4]
  float* out_scores;       // [out_cap]
  long long* out_labels;   // [out_cap]
  int* out_count;
};

// threshold at the max_det-th kept score (ties kept) + ordered compaction, one CTA on `stream`
void launch_box_final(const FinalParams& f, cudaStream_t stream);
#endif

}  // namespace mega
