// Host build of csrc/vid_eval.cuh -- TEST INFRASTRUCTURE ONLY.
// g++ compiles the bodies the kernels of csrc/vid_eval.cu run (ve_match, ve_fp_weight / ve_tp_flag, ve_cumsum,
// ve_prec / ve_rec, ve_steps) and drives them in the kernels' order: the same sort keys written at the same positions
// and sorted by std::stable_sort (the device's CUB radix sort is stable as well), the images and (class, range) lists
// in turn. So the CPU suite checks the device evaluator's order, matching and arithmetic against the host evaluator
// without a GPU. The entry points carry the names and prototypes of include/mega_b200.h (the header is included, so a
// drifting signature does not compile); pointers are host pointers, the workspace is unused, `stream` is ignored.
// Build: g++ -O2 -fPIC -shared -std=c++17 -ffp-contract=off -I mega.pytorch_b200/csrc -I include
//            -o libvid_eval_host.so vid_eval_host.cpp
#include <algorithm>
#include <vector>

#include "mega_b200.h"
#include "vid_eval.cuh"

using namespace mega_ve;

namespace {

struct HostSeg {
  const float* boxes;
  const int* perm;
  long long q0, g0;
  int n, ng, label;
  float sw, sh;
  const float* gt_boxes;
  const int* gt_labels;
  const double* gt_motion;
  const VeRange* ranges;
  unsigned char* sel;             // [nr][G] at this image's GT
  long long G, P;
  signed char* match;
  double* weight;
  int n_pred() const { return n; }
  int n_gt_all() const { return ng; }
  float4 pred(int j) const {
    const float* b = boxes + 4LL * perm[q0 + j];
    return {b[0] * sw, b[1] * sh, b[2] * sw, b[3] * sh};
  }
  float4 gt(int k) const {
    const float* b = gt_boxes + 4 * (g0 + k);
    return {b[0], b[1], b[2], b[3]};
  }
  bool in_class(int k) const { return gt_labels[g0 + k] == label; }
  bool ignored(int k, int r) const { return ve_ignored(gt_motion[g0 + k], ranges[r]); }
  double empty_weight(int r) const { return ranges[r].empty_weight; }
  unsigned char* selec(int r) const { return sel + r * G; }
  void put(int j, int r, signed char m, double w) const {
    const long long g = perm[q0 + j];
    match[r * P + g] = m;
    weight[r * P + g] = w;
  }
};

int bits(long long n) {
  int b = 0;
  while ((1LL << b) < n) ++b;
  return b;
}

void stable_sort_pairs(std::vector<unsigned long long>& keys, std::vector<int>& vals) {
  std::vector<long long> idx(keys.size());
  for (size_t i = 0; i < idx.size(); ++i) idx[i] = static_cast<long long>(i);
  std::stable_sort(idx.begin(), idx.end(), [&](long long a, long long b) { return keys[a] < keys[b]; });
  std::vector<unsigned long long> k2(keys.size());
  std::vector<int> v2(vals.size());
  for (size_t i = 0; i < idx.size(); ++i) k2[i] = keys[idx[i]], v2[i] = vals[idx[i]];
  keys.swap(k2);
  vals.swap(v2);
}

}  // namespace

extern "C" {

long long mega_vid_eval_workspace_bytes(long long num_dets, long long num_gt, int num_images, int num_classes,
                                        int num_ranges) {
  if (num_dets < 0 || num_gt < 0 || num_images < 0 || num_classes < 1 || num_ranges < 1 || num_ranges > kMaxRanges ||
      bits(num_images) + bits(num_classes) > 32)
    return -1;
  return 0;
}

int mega_vid_eval(const float* det_boxes, const float* det_scores, const int* det_labels, const long long* det_offsets,
                  const float* det_scale, long long num_dets, const float* gt_boxes, const int* gt_labels,
                  const double* gt_motion, const long long* gt_offsets, long long num_gt, int num_images,
                  int num_classes, const double* ranges, int num_ranges, float iou_thresh,
                  const long long* step_offsets, long long num_steps, void* workspace, long long workspace_bytes,
                  double* prec, double* rec, long long* stats, double* steps, void* stream) {
  (void)workspace, (void)workspace_bytes, (void)stream;
  if (mega_vid_eval_workspace_bytes(num_dets, num_gt, num_images, num_classes, num_ranges) < 0) return 1;
  const long long P = num_dets, G = num_gt, S = num_steps;
  const int C = num_classes, nr = num_ranges, cs = bits(C);
  VeRange rg[kMaxRanges];
  for (int r = 0; r < nr; ++r) rg[r] = {ranges[3 * r], ranges[3 * r + 1], ranges[3 * r + 2]};
  long long *present = stats, *begin = stats + C, *end = stats + 2 * C, *n_pos = stats + 3 * C,
            *n_steps = stats + 3 * C + nr * C, *rejected = stats + 3 * C + 2 * nr * C;
  std::fill(stats, stats + 3 * C + 2 * nr * C + 1, 0LL);
  for (long long i = 0; i < P; ++i)
    if (det_labels[i] < 0 || det_labels[i] >= C) return 1;
  for (long long i = 0; i < G; ++i)
    if (gt_labels[i] < 0 || gt_labels[i] >= C) return 1;
  // 1. (image, class, score descending), fed in reverse index order
  std::vector<unsigned long long> keys(P);
  std::vector<int> vals(P);
  for (int img = 0; img < num_images; ++img)
    for (long long g = det_offsets[img]; g < det_offsets[img + 1]; ++g) {
      keys[P - 1 - g] = (static_cast<unsigned long long>(img) << (cs + 32)) |
                        (static_cast<unsigned long long>(det_labels[g]) << 32) | ve_desc_key(det_scores[g]);
      vals[P - 1 - g] = static_cast<int>(g);
    }
  stable_sort_pairs(keys, vals);
  // 2. per image and class segment
  std::vector<signed char> match(nr * P);
  std::vector<double> weight(nr * P);
  std::vector<unsigned char> sel(nr * G + 1);
  const unsigned long long cmask = (1ULL << cs) - 1ULL;
  for (int img = 0; img < num_images; ++img) {
    const long long p0 = det_offsets[img], p1 = det_offsets[img + 1], g0 = gt_offsets[img];
    const long long ng = gt_offsets[img + 1] - g0;
    for (long long k = 0; k < ng; ++k) {
      present[gt_labels[g0 + k]] = 1;
      for (int r = 0; r < nr; ++r) n_pos[r * C + gt_labels[g0 + k]] += ve_ignored(gt_motion[g0 + k], rg[r]) ? 0 : 1;
    }
    for (long long q = p0; q < p1;) {
      const int l = static_cast<int>((keys[q] >> 32) & cmask);
      long long e = q + 1;
      while (e < p1 && static_cast<int>((keys[e] >> 32) & cmask) == l) ++e;
      present[l] = 1;
      const HostSeg s = {det_boxes, vals.data(), q, g0, static_cast<int>(e - q), static_cast<int>(ng), l,
                         det_scale[2 * img], det_scale[2 * img + 1], gt_boxes, gt_labels, gt_motion, rg,
                         sel.data() + g0, G, P, match.data(), weight.data()};
      ve_match(s, nr, iou_thresh);
      q = e;
    }
  }
  // 3. (class, score descending), fed image-descending, index-ascending
  for (int img = 0; img < num_images; ++img)
    for (long long g = det_offsets[img]; g < det_offsets[img + 1]; ++g) {
      const long long pos = P - det_offsets[img + 1] + (g - det_offsets[img]);
      keys[pos] = (static_cast<unsigned long long>(det_labels[g]) << 32) | ve_desc_key(det_scores[g]);
      vals[pos] = static_cast<int>(g);
    }
  stable_sort_pairs(keys, vals);
  // 4.
  for (long long i = 0; i < P; ++i) {
    const int c = static_cast<int>(keys[i] >> 32);
    if (i == 0 || static_cast<int>(keys[i - 1] >> 32) != c) begin[c] = i;
    if (i == P - 1 || static_cast<int>(keys[i + 1] >> 32) != c) end[c] = i + 1;
    for (int r = 0; r < nr; ++r) {
      prec[r * P + i] = ve_fp_weight(match[r * P + vals[i]], weight[r * P + vals[i]]);
      rec[r * P + i] = ve_tp_flag(match[r * P + vals[i]], weight[r * P + vals[i]]);
    }
  }
  for (int r = 0; r < nr; ++r)
    for (int c = 0; c < C; ++c)
      if (end[c] > begin[c]) ve_cumsum(prec + r * P + begin[c], rec + r * P + begin[c], end[c] - begin[c]);
  for (long long i = 0; i < P; ++i) {
    const int c = static_cast<int>(keys[i] >> 32);
    for (int r = 0; r < nr; ++r) {
      const double f = prec[r * P + i], tp = rec[r * P + i];
      prec[r * P + i] = ve_prec(f, tp);
      rec[r * P + i] = n_pos[r * C + c] > 0 ? ve_rec(tp, n_pos[r * C + c]) : 0.0;
    }
  }
  for (int r = 0; r < nr; ++r)
    for (int c = 0; c < C; ++c) {
      long long cnt = -1;
      if (present[c] && n_pos[r * C + c] > 0) {
        const long long o = step_offsets[c];
        double* base = steps + 3LL * r * S + o;
        cnt = ve_steps(prec + r * P + begin[c], rec + r * P + begin[c], end[c] - begin[c], step_offsets[c + 1] - o,
                       base, base + S, base + 2 * S);
        if (cnt < 0) ++*rejected;
      }
      n_steps[r * C + c] = cnt;
    }
  return 0;
}

}  // extern "C"
