// Per-item bodies of test-time box augmentation (TEST.BBOX_AUG; reference engine/bbox_aug.py:11-68), shared by the
// kernels of bbox_aug.cu and the g++ build under tests/native:
//   * collect: one (proposal, class) of one pass -> softmax, decode, clip in the pass's own image size (the
//     post-processor with bbox_aug_enabled, box_head/inference.py:84-86), flip back (BoxList.transpose
//     FLIP_LEFT_RIGHT) and scale to the identity pass's size (BoxList.resize), written to the pass's slot of a
//     class-major staging area [num_classes][num_passes * r_max];
//   * merge primitives: the candidate sort key (score descending, merged row ascending) and the exact early stop of a
//     class's greedy NMS sweep.
#pragma once
#include <stdint.h>
#include <string.h>

#include "box_head.cuh"

namespace mega {

constexpr int kAugMaxCand = 8192;   // merged rows (passes x proposals) per class: 18 passes x 300 fit, as does _C.nms

struct AugCollectArgs {
  const float* logits;     // [r_max, ld_logits]
  int ld_logits;
  const float* deltas;     // [r_max, ld_deltas], 4 * num_classes valid columns
  int ld_deltas;
  const float* proposals;  // [r_max, 4]
  int r_max, num_classes, slot, rows;   // rows = num_passes * r_max: the staging row pitch of one class
  float im_w, im_h;        // this pass's image size
  int hflip;               // the pass ran on the flipped image
  float ratio_w, ratio_h;  // fp32 of the Python ratios identity size / pass size (1 for the identity pass)
  float score_thresh;
  BoxCoderW w;
  float4* boxes;           // [num_classes][rows]
  float* scores;           // [num_classes][rows]
  unsigned char* cand;     // [num_classes][rows]: score > SCORE_THRESH
};

// pass frame -> identity frame. transpose: x1' = (W - x2) - 1, x2' = (W - x1) - 1 with W the pass's int width, each
// subtraction rounded to fp32 (bounding_box.py transpose); resize: fp32 tensor * Python float == x * fl32(ratio). When
// the two ratios are equal the reference multiplies all four by one ratio: the same products.
MEGA_IOU_HD float4 aug_to_identity(float4 b, int hflip, float im_w, float ratio_w, float ratio_h) {
  if (hflip) {
    const float x1 = MEGA_IOU_SUB(MEGA_IOU_SUB(im_w, b.z), 1.f);
    const float x2 = MEGA_IOU_SUB(MEGA_IOU_SUB(im_w, b.x), 1.f);
    b.x = x1;
    b.z = x2;
  }
  b.x = MEGA_IOU_MUL(b.x, ratio_w);
  b.y = MEGA_IOU_MUL(b.y, ratio_h);
  b.z = MEGA_IOU_MUL(b.z, ratio_w);
  b.w = MEGA_IOU_MUL(b.w, ratio_h);
  return b;
}

// item i = (class j = 1 + i / r_max, proposal r = i % r_max); rows >= count are no candidates
MEGA_IOU_HD void aug_collect_item(const AugCollectArgs& a, int count, long long i) {
  const int j = 1 + static_cast<int>(i / a.r_max), r = static_cast<int>(i % a.r_max);
  const long long o = static_cast<long long>(j) * a.rows + static_cast<long long>(a.slot) * a.r_max + r;
  if (r >= count) {
    a.boxes[o] = float4{0.f, 0.f, 0.f, 0.f};
    a.scores[o] = 0.f;
    a.cand[o] = 0;
    return;
  }
  const float prob = class_softmax_prob(a.logits + static_cast<long long>(r) * a.ld_logits, a.num_classes, j);
  const float* p = a.proposals + static_cast<long long>(r) * 4;
  const float4 box = decode_clip_box(a.deltas + static_cast<long long>(r) * a.ld_deltas + j * 4,
                                     float4{p[0], p[1], p[2], p[3]}, a.w, a.im_w, a.im_h);
  a.boxes[o] = aug_to_identity(box, a.hflip, a.im_w, a.ratio_w, a.ratio_h);
  a.scores[o] = prob;
  a.cand[o] = prob > a.score_thresh ? 1 : 0;
}

// sort key of a candidate: ascending key == score descending, then merged row ascending
MEGA_IOU_HD uint64_t aug_key(float score, int row) {
  uint32_t b;
  memcpy(&b, &score, 4);
  const uint32_t ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return (static_cast<uint64_t>(~ord) << 32) | static_cast<uint32_t>(row);
}

MEGA_IOU_HD int aug_key_row(uint64_t key) { return static_cast<int>(key & 0xffffffffu); }

// Exact early stop of one class's sweep. Once the class has kept max_det boxes, the max_det-th of them scoring s, the
// kthvalue cap over all classes is >= s: every later box scoring below s is cut by the cap whatever NMS decides, and
// dropping such boxes leaves the max_det-th largest kept score unchanged. Boxes tying s still go through NMS.
// cap_key_hi: the upper key half (score order) of the max_det-th kept box.
MEGA_IOU_HD bool aug_past_cap(int kept, int max_det, uint32_t cap_key_hi, uint64_t key) {
  return max_det > 0 && kept >= max_det && static_cast<uint32_t>(key >> 32) != cap_key_hi;
}

}  // namespace mega
