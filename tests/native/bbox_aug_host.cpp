// Host build of csrc/bbox_aug.cuh -- TEST INFRASTRUCTURE ONLY.
// g++ compiles the bodies the kernels of csrc/bbox_aug.cu run: the collect item, the pass -> identity mapping, the
// candidate key, the exact cap stop and the IoU decision (iou.cuh). The merge is the same greedy sweep done one
// candidate at a time (the kernel does it 64 at a time; both keep box o iff no earlier kept box overlaps it), followed by
// the cap and the ordered compaction of box_final_kernel. Entry points carry the prototypes of include/mega_b200.h;
// pointers are host pointers, `count_ptr` points to host memory, `stream` is ignored.
// Build: g++ -O2 -fPIC -shared -std=c++17 -ffp-contract=off -I mega.pytorch_b200/csrc -I include
//            -o libbbox_aug_host.so bbox_aug_host.cpp
#include <algorithm>
#include <vector>

#include "bbox_aug.cuh"
#include "mega_b200.h"

using namespace mega;

namespace {

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

struct Staging {
  float4* boxes;
  float* scores;
  unsigned char* flags;
};

Staging staging(void* ws, int rows, int num_classes) {
  const size_t slots = static_cast<size_t>(rows) * num_classes;
  char* w = static_cast<char*>(ws);
  return {reinterpret_cast<float4*>(w), reinterpret_cast<float*>(w + align256(sizeof(float4) * slots)),
          reinterpret_cast<unsigned char*>(w + align256(sizeof(float4) * slots) + align256(sizeof(float) * slots))};
}

}  // namespace

extern "C" {

long long mega_bbox_aug_workspace_bytes(int num_passes, int r_max, int num_classes) {
  if (num_passes < 1 || r_max < 1 || num_classes < 2) return -1;
  if (static_cast<long long>(num_passes) * r_max > kAugMaxCand) return -1;
  const size_t slots = static_cast<size_t>(num_passes) * r_max * num_classes;
  return static_cast<long long>(align256(sizeof(float4) * slots) + align256(sizeof(float) * slots) + align256(slots));
}

int mega_bbox_aug_collect(const float* logits, int ld_logits, const float* deltas, int ld_deltas, const float* proposals,
                          const int* count_ptr, int r_max, int num_classes, int pass, int num_passes, int im_w,
                          int im_h, int hflip, double ratio_w, double ratio_h, float score_thresh, float wx, float wy,
                          float ww, float wh, void* workspace, long long workspace_bytes, void* stream) {
  (void)stream;
  const long long need = mega_bbox_aug_workspace_bytes(num_passes, r_max, num_classes);
  if (need < 0 || workspace_bytes < need || pass < 0 || pass >= num_passes) return 1;
  const Staging s = staging(workspace, num_passes * r_max, num_classes);
  AugCollectArgs a;
  a.logits = logits, a.ld_logits = ld_logits, a.deltas = deltas, a.ld_deltas = ld_deltas, a.proposals = proposals;
  a.r_max = r_max, a.num_classes = num_classes, a.slot = pass, a.rows = num_passes * r_max;
  a.im_w = static_cast<float>(im_w), a.im_h = static_cast<float>(im_h), a.hflip = hflip ? 1 : 0;
  a.ratio_w = static_cast<float>(ratio_w), a.ratio_h = static_cast<float>(ratio_h);
  a.score_thresh = score_thresh;
  a.w = BoxCoderW{wx, wy, ww, wh};
  a.boxes = s.boxes, a.scores = s.scores, a.cand = s.flags;
  const int count = std::min(*count_ptr, r_max);
  for (long long i = 0; i < static_cast<long long>(num_classes - 1) * r_max; ++i) aug_collect_item(a, count, i);
  return 0;
}

// test entry: stage a pass's raw post-processor BoxList as the reference returns it (rows proposal-major, class-minor;
// boxes already decoded and clipped in the pass frame) through the mapping the collect item applies
int bbox_aug_stage_raw_host(const float* boxes, const float* scores, int count, int r_max, int num_classes, int pass,
                            int num_passes, int im_w, int hflip, double ratio_w, double ratio_h, float score_thresh,
                            void* workspace) {
  if (count > r_max || pass < 0 || pass >= num_passes) return 1;
  const int rows = num_passes * r_max;
  const Staging s = staging(workspace, rows, num_classes);
  for (int j = 1; j < num_classes; ++j) {
    for (int r = 0; r < r_max; ++r) {
      const long long o = static_cast<long long>(j) * rows + static_cast<long long>(pass) * r_max + r;
      if (r >= count) {
        s.boxes[o] = float4{0.f, 0.f, 0.f, 0.f};
        s.scores[o] = 0.f;
        s.flags[o] = 0;
        continue;
      }
      const float* b = boxes + (static_cast<long long>(r) * num_classes + j) * 4;
      const float sc = scores[static_cast<long long>(r) * num_classes + j];
      s.boxes[o] = aug_to_identity(float4{b[0], b[1], b[2], b[3]}, hflip, static_cast<float>(im_w),
                                   static_cast<float>(ratio_w), static_cast<float>(ratio_h));
      s.scores[o] = sc;
      s.flags[o] = sc > score_thresh ? 1 : 0;
    }
  }
  return 0;
}

int mega_bbox_aug_merge(int num_passes, int r_max, int num_classes, float nms_thresh, int max_det, void* workspace,
                        long long workspace_bytes, float* out_boxes, float* out_scores, long long* out_labels,
                        int out_cap, int* out_count, void* stream) {
  (void)stream;
  const long long need = mega_bbox_aug_workspace_bytes(num_passes, r_max, num_classes);
  if (need < 0 || workspace_bytes < need) return 1;
  const int rows = num_passes * r_max;
  const Staging s = staging(workspace, rows, num_classes);
  const float t_lo = nms_thresh * (1.f - 9.5367431640625e-07f), t_hi = nms_thresh * (1.f + 9.5367431640625e-07f);
  for (int j = 1; j < num_classes; ++j) {
    const float4* boxes = s.boxes + static_cast<long long>(j) * rows;
    const float* scores = s.scores + static_cast<long long>(j) * rows;
    unsigned char* flags = s.flags + static_cast<long long>(j) * rows;
    std::vector<uint64_t> keys;
    for (int i = 0; i < rows; ++i) {
      if (flags[i]) keys.push_back(aug_key(scores[i], i));
      flags[i] = 0;
    }
    std::sort(keys.begin(), keys.end());
    std::vector<float4> kept;
    uint32_t cap = 0;
    for (const uint64_t key : keys) {
      if (aug_past_cap(static_cast<int>(kept.size()), max_det, cap, key)) break;
      const float4 b = boxes[aug_key_row(key)];
      const float ab = box_area_plus1(b);
      bool hit = false;
      for (const float4& k : kept) {
        if (iou_plus1_gt(k, box_area_plus1(k), b, ab, nms_thresh, t_lo, t_hi)) {
          hit = true;
          break;
        }
      }
      if (hit) continue;
      kept.push_back(b);
      flags[aug_key_row(key)] = 1;
      if (static_cast<int>(kept.size()) == max_det) cap = static_cast<uint32_t>(key >> 32);
    }
  }
  // box_final_kernel: the max_det-th largest kept score, ties kept, class-major in merged-row order
  std::vector<float> kept_scores;
  for (long long i = rows; i < static_cast<long long>(rows) * num_classes; ++i)
    if (s.flags[i]) kept_scores.push_back(s.scores[i]);
  const int total = static_cast<int>(kept_scores.size());
  uint64_t thr = ~0ULL;   // keep a box iff aug_key(score, 0) <= thr
  if (total > max_det && max_det > 0) {
    std::nth_element(kept_scores.begin(), kept_scores.begin() + (max_det - 1), kept_scores.end(),
                     [](float a, float b) { return aug_key(a, 0) < aug_key(b, 0); });
    thr = aug_key(kept_scores[max_det - 1], 0);
  }
  int n = 0;
  for (long long i = rows; i < static_cast<long long>(rows) * num_classes; ++i) {
    if (!s.flags[i] || aug_key(s.scores[i], 0) > thr) continue;
    if (n < out_cap) {
      out_boxes[4 * n + 0] = s.boxes[i].x;
      out_boxes[4 * n + 1] = s.boxes[i].y;
      out_boxes[4 * n + 2] = s.boxes[i].z;
      out_boxes[4 * n + 3] = s.boxes[i].w;
      out_scores[n] = s.scores[i];
      out_labels[n] = i / rows;
    }
    ++n;
  }
  *out_count = std::min(n, out_cap);
  return 0;
}

}  // extern "C"
