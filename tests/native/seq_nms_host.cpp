// Host build of csrc/seq_nms.cuh -- TEST INFRASTRUCTURE ONLY.
// g++ compiles the very bodies the kernels of csrc/seq_nms.cu run: the bucket and link items one by one, and the
// per-(video, class) select / rescore / suppress loop with a single lane (the warp's reductions become no-ops), so the
// CPU suite checks the kernels' arithmetic and control flow -- incremental DP, early exit, root-search blocks -- against
// tests/seq_nms_oracle.py without a GPU. The entry points carry the names and prototypes of include/mega_b200.h (the
// header is included, so a drifting signature does not compile); pointers are host pointers, `stream` is ignored.
// Build: g++ -O2 -fPIC -shared -std=c++17 -ffp-contract=off -I mega.pytorch_b200/csrc -I include
//            -o libseq_nms_host.so seq_nms_host.cpp
#include "mega_b200.h"
#include "seq_nms.cuh"

using namespace mega_seq;

struct HostLanes {
  int lane() const { return 0; }
  int count() const { return 1; }
  void sync() const {}
  bool any(bool p) const { return p; }
  void argmax(double&, int&) const {}
};

extern "C" {

long long mega_seq_nms_workspace_bytes(int num_frames, int max_det, int num_classes) {
  if (num_frames < 1 || max_det < 1 || max_det > kMaxDet || num_classes < 1) return -1;
  return seq_workspace_layout(num_frames, max_det, num_classes, nullptr, nullptr);
}

int mega_seq_nms(const float* boxes, const float* scores, const int* labels, const int* counts, int num_frames,
                 int max_det, const int* video_offsets, int num_videos, int num_classes, float link_iou, float nms_iou,
                 int rescore, void* workspace, long long workspace_bytes, float* out_scores, unsigned char* keep,
                 void* stream) {
  (void)stream;
  const long long need = mega_seq_nms_workspace_bytes(num_frames, max_det, num_classes);
  if (need < 0 || workspace_bytes < need || num_videos < 1 || (rescore != 0 && rescore != 1)) return 1;
  const SeqArgs a = seq_make_args(boxes, scores, labels, counts, num_frames, max_det, video_offsets, num_classes,
                                  link_iou, nms_iou, rescore, workspace, out_scores, keep);
  for (long long i = 0; i < static_cast<long long>(num_frames) * num_classes; ++i) seq_bucket_item(a, i);
  for (long long i = 0; i < static_cast<long long>(num_frames) * max_det * a.words; ++i) seq_link_item(a, i);
  for (int v = 0; v < num_videos; ++v)
    for (int c = 0; c < num_classes; ++c) seq_video_class(a, HostLanes(), v, c);
  return 0;
}

}  // extern "C"
