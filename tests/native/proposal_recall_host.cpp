// Host build of csrc/proposal_recall.cuh -- TEST INFRASTRUCTURE ONLY.
// g++ compiles the very per-image body the kernel of csrc/proposal_recall.cu runs, with a single lane (the block arg-max
// becomes a no-op: one lane scans every entry), over the images in order, so the CPU suite checks the kernel's sort,
// IoU arithmetic and greedy rounds against the reference's eval_proposals_vid without a GPU. The entry points carry the
// names and prototypes of include/mega_b200.h (the header is included, so a drifting signature does not compile);
// pointers are host pointers, `stream` is ignored.
// Build: g++ -O2 -fPIC -shared -std=c++17 -ffp-contract=off -I mega.pytorch_b200/csrc -I include
//            -o libproposal_recall_host.so proposal_recall_host.cpp
#include <vector>

#include "mega_b200.h"
#include "proposal_recall.cuh"

using namespace mega_pr;

struct HostLanes {
  int lane() const { return 0; }
  int count() const { return 1; }
  void sync() const {}
  void argmax(float&, unsigned&) const {}
};

extern "C" {

long long mega_proposal_recall_workspace_bytes(int num_images, int max_props, int max_gt, int limit) {
  PrLayout l;
  return pr_layout(num_images, max_props, max_gt, limit, &l) ? l.workspace_bytes : -1;
}

int mega_proposal_recall(const float* prop_boxes, const float* prop_scores, const long long* prop_offsets,
                         const float* gt_boxes, const long long* gt_offsets, int num_images, int max_props, int max_gt,
                         int limit, float iou_thresh, void* workspace, long long workspace_bytes, float* gt_overlaps,
                         unsigned long long* stats, void* stream) {
  (void)stream;
  PrLayout l;
  if (!pr_layout(num_images, max_props, max_gt, limit, &l) || workspace_bytes < l.workspace_bytes) return 1;
  PrArgs a;
  a.prop_boxes = reinterpret_cast<const float4*>(prop_boxes);
  a.prop_scores = prop_scores;
  a.prop_off = prop_offsets;
  a.gt_boxes = reinterpret_cast<const float4*>(gt_boxes);
  a.gt_off = gt_offsets;
  a.num_images = num_images;
  a.max_props = max_props;
  a.max_gt = max_gt;
  a.limit = limit;
  a.thresh = iou_thresh;
  a.smem_matrix_floats = static_cast<int>(l.smem_matrix_bytes / 4);
  a.gmatrix = l.workspace_bytes ? static_cast<float*>(workspace) : nullptr;
  a.slot_floats = l.slot_bytes / 4;
  a.gt_overlaps = gt_overlaps;
  std::vector<PrItem> keys(l.keys_bytes / 8);
  std::vector<float> smat(l.smem_matrix_bytes / 4 + 1);
  PrCounts c = {0, 0, 0};
  for (int img = 0; img < num_images; ++img) pr_image(a, HostLanes(), img, keys.data(), smat.data(), a.gmatrix, c);
  stats[0] = c.hits;
  stats[1] = c.num_pos;
  stats[2] = c.rejected;
  return 0;
}

}  // extern "C"
