// ImageNet VID detection AP (SURVEY.md section 8f row 2).
//
// mega_vid_match_host: the host-side greedy matching of one (image, class), one native call per (image, class) from
// the host evaluator (data/datasets/evaluation/vid/vid_eval.py:201-262 of the reference).
//
// mega_vid_eval: the whole evaluation of a dataset, every motion range at once, in one sequence of launches on the
// caller's stream (include/mega_b200.h). The bodies are those of vid_eval.cuh; what this file adds is the order:
//   1. keys (image, class, score descending) over the detections fed in reverse index order, and a stable CUB radix
//      sort: per image and class the detections in the order of argsort(kind="stable")[::-1];
//   2. one CTA per image (images blockIdx.x, + gridDim.x, ...): one thread per class segment of the image runs
//      ve_match for all ranges; the CTA's threads count n_pos and the classes present (integer atomics);
//   3. keys (class, score descending) over the detections fed image-descending, index-ascending, and a second stable
//      sort: per class the order of argsort(kind="stable")[::-1] over the per-image lists concatenated in image order;
//   4. in that order: the fps / tps of every (range, detection) gathered (parallel), cumulated per (class, range) by
//      one thread each (ve_cumsum: the fp64 sum runs strictly left to right, as np.cumsum does), prec / rec
//      (parallel), and the envelope and recall steps per (class, range) by one thread each (ve_steps).
// Every result is independent of scheduling: the only atomics add integers, and the stores of `present` all write 1.
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "vid_eval.cuh"
#include "mega_b200.h"

using namespace mega_ve;

namespace {

// host-pointer source of mega_vid_match_host: one class, all GT in the class, one range
struct HostMatch {
  const float* pb;
  const float* gb;
  const unsigned char* gi;
  int np, ng;
  double ew;
  unsigned char* sel;
  signed char* match_out;
  double* ign_out;
  int n_pred() const { return np; }
  int n_gt_all() const { return ng; }
  float4 pred(int j) const { return {pb[4 * j], pb[4 * j + 1], pb[4 * j + 2], pb[4 * j + 3]}; }
  float4 gt(int k) const { return {gb[4 * k], gb[4 * k + 1], gb[4 * k + 2], gb[4 * k + 3]}; }
  bool in_class(int) const { return true; }
  bool ignored(int k, int) const { return gi[k] != 0; }
  double empty_weight(int) const { return ew; }
  unsigned char* selec(int) const { return sel; }
  void put(int j, int, signed char m, double w) const {
    match_out[j] = m;
    ign_out[j] = w;
  }
};

}  // namespace

extern "C" int mega_vid_match_host(const float* pred_boxes, int n_pred, const float* gt_boxes,
                                   const unsigned char* gt_ignore, int n_gt, float iou_thresh, double empty_weight,
                                   signed char* match_out, double* pred_ignore_out) {
  MEGA_ARG_CHECK(n_pred >= 0 && n_gt >= 0, "vid_match: negative sizes");
  std::vector<unsigned char> selec(n_gt > 0 ? n_gt : 1, 0);
  const HostMatch s = {pred_boxes, gt_boxes, gt_ignore, n_pred, n_gt, empty_weight, selec.data(), match_out,
                       pred_ignore_out};
  ve_match(s, 1, iou_thresh);
  return MEGA_OK;
}

namespace {

constexpr int kThreads = 256;
constexpr int kMaxCtas = 2048;

struct VeArgs {
  const float4* det_boxes;
  const float* det_scores;
  const int* det_labels;
  const long long* det_off;
  const float2* det_scale;
  const float4* gt_boxes;
  const int* gt_labels;
  const double* gt_motion;
  const long long* gt_off;
  int num_images, num_classes, nr, cls_shift;
  long long P, G, S;
  VeRange ranges[kMaxRanges];
  float iou_thresh;
  const long long* step_off;
  unsigned long long* keys;       // sort buffers
  int* vals;
  signed char* match;             // [nr][P], by input index
  double* weight;                 // [nr][P], by input index
  unsigned char* selec;           // [nr][G]
  double* prec;                   // [nr][P], global class order
  double* rec;
  long long* present;             // stats sections
  long long* cls_begin;
  long long* cls_end;
  long long* n_pos;               // [nr][C]
  long long* n_steps;             // [nr][C]
  unsigned long long* rejected;
  double* steps;                  // [nr][3][S]
};

__device__ __forceinline__ int label_ok(int l, int c) { return l >= 0 && l < c; }

// 1. (image, class, score descending), detections fed in reverse index order so that ties end later-index-first
__global__ void __launch_bounds__(kThreads) ve_keys_image(VeArgs a) {
  for (int img = blockIdx.x; img < a.num_images; img += gridDim.x) {
    const long long p0 = a.det_off[img], p1 = a.det_off[img + 1];
    for (long long g = p0 + threadIdx.x; g < p1; g += blockDim.x) {
      int l = a.det_labels[g];
      if (!label_ok(l, a.num_classes)) {
        atomicAdd(a.rejected, 1ULL);
        l = 0;
      }
      const long long pos = a.P - 1 - g;
      a.keys[pos] = (static_cast<unsigned long long>(img) << (a.cls_shift + 32)) |
                    (static_cast<unsigned long long>(l) << 32) | ve_desc_key(a.det_scores[g]);
      a.vals[pos] = static_cast<int>(g);
    }
  }
}

// device source of ve_match: one class segment [q0, q0 + n) of the image's sorted detections
struct DevMatch {
  const VeArgs* a;
  const int* perm;
  long long q0, g0;
  int n, ng, label;
  float2 scale;
  __device__ int n_pred() const { return n; }
  __device__ int n_gt_all() const { return ng; }
  __device__ float4 pred(int j) const {
    const float4 b = a->det_boxes[perm[q0 + j]];     // BoxList.resize: bbox * tensor([rw, rh, rw, rh]) in fp32
    return {__fmul_rn(b.x, scale.x), __fmul_rn(b.y, scale.y), __fmul_rn(b.z, scale.x), __fmul_rn(b.w, scale.y)};
  }
  __device__ float4 gt(int k) const { return a->gt_boxes[g0 + k]; }
  __device__ bool in_class(int k) const { return a->gt_labels[g0 + k] == label; }
  __device__ bool ignored(int k, int r) const { return ve_ignored(a->gt_motion[g0 + k], a->ranges[r]); }
  __device__ double empty_weight(int r) const { return a->ranges[r].empty_weight; }
  __device__ unsigned char* selec(int r) const { return a->selec + r * a->G + g0; }
  __device__ void put(int j, int r, signed char m, double w) const {
    const long long g = perm[q0 + j];
    a->match[r * a->P + g] = m;
    a->weight[r * a->P + g] = w;
  }
};

// 2. per image: matching per class segment, n_pos and the classes present
__global__ void __launch_bounds__(kThreads) ve_match_images(const __grid_constant__ VeArgs a,
                                                            const unsigned long long* keys, const int* perm) {
  const unsigned long long cmask = (1ULL << a.cls_shift) - 1ULL;
  for (int img = blockIdx.x; img < a.num_images; img += gridDim.x) {
    const long long p0 = a.det_off[img], p1 = a.det_off[img + 1];
    const long long g0 = a.gt_off[img], ng = a.gt_off[img + 1] - g0;
    for (long long k = threadIdx.x; k < ng; k += blockDim.x) {
      const int l = a.gt_labels[g0 + k];
      if (!label_ok(l, a.num_classes)) {
        atomicAdd(a.rejected, 1ULL);
        continue;
      }
      a.present[l] = 1;
      for (int r = 0; r < a.nr; ++r)
        if (!ve_ignored(a.gt_motion[g0 + k], a.ranges[r]))
          atomicAdd(reinterpret_cast<unsigned long long*>(a.n_pos + r * a.num_classes + l), 1ULL);
    }
    for (long long q = p0 + threadIdx.x; q < p1; q += blockDim.x) {
      const int l = static_cast<int>((keys[q] >> 32) & cmask);
      if (q > p0 && static_cast<int>((keys[q - 1] >> 32) & cmask) == l) continue;   // not a segment start
      long long e = q + 1;
      while (e < p1 && static_cast<int>((keys[e] >> 32) & cmask) == l) ++e;
      a.present[l] = 1;
      const DevMatch s = {&a, perm, q, g0, static_cast<int>(e - q), static_cast<int>(ng), l, a.det_scale[img]};
      ve_match(s, a.nr, a.iou_thresh);
    }
  }
}

// 3. (class, score descending), detections fed image-descending, index-ascending
__global__ void __launch_bounds__(kThreads) ve_keys_class(VeArgs a) {
  for (int img = blockIdx.x; img < a.num_images; img += gridDim.x) {
    const long long p0 = a.det_off[img], p1 = a.det_off[img + 1];
    for (long long g = p0 + threadIdx.x; g < p1; g += blockDim.x) {
      const int l = a.det_labels[g];
      const long long pos = a.P - p1 + (g - p0);
      a.keys[pos] = (static_cast<unsigned long long>(label_ok(l, a.num_classes) ? l : 0) << 32) |
                    ve_desc_key(a.det_scores[g]);
      a.vals[pos] = static_cast<int>(g);
    }
  }
}

// 4a. class bounds in the sorted order; tps / fps of every (range, detection)
__global__ void ve_gather(VeArgs a, const unsigned long long* keys, const int* perm) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < a.P; i += stride) {
    const int c = static_cast<int>(keys[i] >> 32);
    if (i == 0 || static_cast<int>(keys[i - 1] >> 32) != c) a.cls_begin[c] = i;
    if (i == a.P - 1 || static_cast<int>(keys[i + 1] >> 32) != c) a.cls_end[c] = i + 1;
    const long long g = perm[i];
    for (int r = 0; r < a.nr; ++r) {
      const signed char m = a.match[r * a.P + g];
      const double w = a.weight[r * a.P + g];
      a.prec[r * a.P + i] = ve_fp_weight(m, w);
      a.rec[r * a.P + i] = ve_tp_flag(m, w);
    }
  }
}

// 4b. one thread per (range, class): the sequential cumulative sums
__global__ void ve_cumsum_classes(VeArgs a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.nr * a.num_classes) return;
  const int r = t / a.num_classes, c = t - r * a.num_classes;
  const long long b = a.cls_begin[c], e = a.cls_end[c];
  if (e > b) ve_cumsum(a.prec + r * a.P + b, a.rec + r * a.P + b, e - b);
}

// 4c. prec / rec
__global__ void ve_prec_rec(VeArgs a, const unsigned long long* keys) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < a.P; i += stride) {
    const int c = static_cast<int>(keys[i] >> 32);
    for (int r = 0; r < a.nr; ++r) {
      const double f = a.prec[r * a.P + i], tp = a.rec[r * a.P + i];
      const long long npos = a.n_pos[r * a.num_classes + c];
      a.prec[r * a.P + i] = ve_prec(f, tp);
      a.rec[r * a.P + i] = npos > 0 ? ve_rec(tp, npos) : 0.0;
    }
  }
}

// 4d. one thread per (range, class): envelope and recall steps
__global__ void ve_steps_classes(VeArgs a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.nr * a.num_classes) return;
  const int r = t / a.num_classes, c = t - r * a.num_classes;
  long long cnt = -1;
  if (a.present[c] && a.n_pos[t] > 0) {
    const long long b = a.cls_begin[c], n = a.cls_end[c] - b, o = a.step_off[c];
    double* base = a.steps + 3LL * r * a.S + o;
    cnt = ve_steps(a.prec + r * a.P + b, a.rec + r * a.P + b, n, a.step_off[c + 1] - o, base, base + a.S,
                   base + 2 * a.S);
    if (cnt < 0) atomicAdd(a.rejected, 1ULL);
  }
  a.n_steps[t] = cnt;
}

struct VeLayout {
  int cls_shift, img_bits;
  size_t sort_temp;
  long long keys0, keys1, vals0, vals1, temp, match, weight, selec, total;
};

long long ve_align(long long x) { return (x + 255) & ~255LL; }

int ve_bits(long long n) {
  int b = 0;
  while ((1LL << b) < n) ++b;
  return b;
}

bool ve_layout(long long P, long long G, int num_images, int num_classes, int nr, VeLayout* l) {
  if (P < 0 || P > 0x7fffffffLL || G < 0 || num_images < 0 || num_classes < 1 || nr < 1 || nr > kMaxRanges)
    return false;
  l->cls_shift = ve_bits(num_classes);
  l->img_bits = ve_bits(num_images);
  if (l->cls_shift + l->img_bits > 32) return false;
  size_t t1 = 0, t2 = 0;
  cub::DoubleBuffer<unsigned long long> dk(nullptr, nullptr);
  cub::DoubleBuffer<int> dv(nullptr, nullptr);
  const int n = static_cast<int>(P);
  if (cub::DeviceRadixSort::SortPairs(nullptr, t1, dk, dv, n, 0, 32 + l->cls_shift + l->img_bits) != cudaSuccess ||
      cub::DeviceRadixSort::SortPairs(nullptr, t2, dk, dv, n, 0, 32 + l->cls_shift) != cudaSuccess)
    return false;
  l->sort_temp = t1 > t2 ? t1 : t2;
  long long o = 0;
  l->keys0 = o, o += ve_align(8 * P);
  l->keys1 = o, o += ve_align(8 * P);
  l->vals0 = o, o += ve_align(4 * P);
  l->vals1 = o, o += ve_align(4 * P);
  l->temp = o, o += ve_align(static_cast<long long>(l->sort_temp));
  l->match = o, o += ve_align(nr * P);
  l->weight = o, o += ve_align(8 * nr * P);
  l->selec = o, o += ve_align(nr * G);
  l->total = o;
  return true;
}

}  // namespace

extern "C" long long mega_vid_eval_workspace_bytes(long long num_dets, long long num_gt, int num_images,
                                                   int num_classes, int num_ranges) {
  VeLayout l;
  return ve_layout(num_dets, num_gt, num_images, num_classes, num_ranges, &l) ? l.total : -1;
}

extern "C" int mega_vid_eval(const float* det_boxes, const float* det_scores, const int* det_labels,
                             const long long* det_offsets, const float* det_scale, long long num_dets,
                             const float* gt_boxes, const int* gt_labels, const double* gt_motion,
                             const long long* gt_offsets, long long num_gt, int num_images, int num_classes,
                             const double* ranges, int num_ranges, float iou_thresh, const long long* step_offsets,
                             long long num_steps, void* workspace, long long workspace_bytes, double* prec,
                             double* rec, long long* stats, double* steps, void* stream_) {
  VeLayout l;
  MEGA_ARG_CHECK(ve_layout(num_dets, num_gt, num_images, num_classes, num_ranges, &l),
                 "vid_eval: out of range: %lld detections, %lld GT, %d images, %d classes, %d ranges (at most %d "
                 "ranges, 2^31 - 1 detections, and ceil(log2 images) + ceil(log2 classes) <= 32)",
                 num_dets, num_gt, num_images, num_classes, num_ranges, kMaxRanges);
  MEGA_ARG_CHECK(ranges && stats && det_offsets && gt_offsets && step_offsets && num_steps >= 0,
                 "vid_eval: null ranges, stats or offsets pointer, or negative num_steps");
  MEGA_ARG_CHECK(reinterpret_cast<uintptr_t>(det_boxes) % 16 == 0 && reinterpret_cast<uintptr_t>(gt_boxes) % 16 == 0 &&
                     reinterpret_cast<uintptr_t>(det_scale) % 8 == 0,
                 "vid_eval: boxes must be 16-byte aligned, scales 8-byte aligned");
  MEGA_ARG_CHECK(workspace && workspace_bytes >= l.total && reinterpret_cast<uintptr_t>(workspace) % 256 == 0,
                 "vid_eval: workspace must be 256-byte aligned and hold %lld bytes (got %lld)", l.total,
                 workspace_bytes);
  MEGA_ARG_CHECK((num_dets == 0 || (prec && rec)) && (num_steps == 0 || steps), "vid_eval: null prec, rec or steps");
  const int C = num_classes, nr = num_ranges;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  char* ws = static_cast<char*>(workspace);
  VeArgs a = {};
  a.det_boxes = reinterpret_cast<const float4*>(det_boxes);
  a.det_scores = det_scores;
  a.det_labels = det_labels;
  a.det_off = det_offsets;
  a.det_scale = reinterpret_cast<const float2*>(det_scale);
  a.gt_boxes = reinterpret_cast<const float4*>(gt_boxes);
  a.gt_labels = gt_labels;
  a.gt_motion = gt_motion;
  a.gt_off = gt_offsets;
  a.num_images = num_images;
  a.num_classes = C;
  a.nr = nr;
  a.cls_shift = l.cls_shift;
  a.P = num_dets;
  a.G = num_gt;
  a.S = num_steps;
  for (int r = 0; r < nr; ++r) a.ranges[r] = {ranges[3 * r], ranges[3 * r + 1], ranges[3 * r + 2]};
  a.iou_thresh = iou_thresh;
  a.step_off = step_offsets;
  a.match = reinterpret_cast<signed char*>(ws + l.match);
  a.weight = reinterpret_cast<double*>(ws + l.weight);
  a.selec = reinterpret_cast<unsigned char*>(ws + l.selec);
  a.prec = prec;
  a.rec = rec;
  a.present = stats;
  a.cls_begin = stats + C;
  a.cls_end = stats + 2 * C;
  a.n_pos = stats + 3 * C;
  a.n_steps = stats + 3 * C + nr * C;
  a.rejected = reinterpret_cast<unsigned long long*>(stats + 3 * C + 2 * nr * C);
  a.steps = steps;
  MEGA_CUDA_CHECK(cudaMemsetAsync(stats, 0, sizeof(long long) * (3 * C + 2 * nr * C + 1), stream));
  const int grid_img = num_images < kMaxCtas ? (num_images > 0 ? num_images : 1) : kMaxCtas;
  const int grid_pc = mega_ceil_div(nr * C, 32);
  const int n = static_cast<int>(num_dets);
  auto* k0 = reinterpret_cast<unsigned long long*>(ws + l.keys0);
  auto* k1 = reinterpret_cast<unsigned long long*>(ws + l.keys1);
  auto* v0 = reinterpret_cast<int*>(ws + l.vals0);
  auto* v1 = reinterpret_cast<int*>(ws + l.vals1);
  void* temp = ws + l.temp;
  size_t temp_bytes = l.sort_temp;
  // 1-2
  a.keys = k0, a.vals = v0;
  if (num_images > 0) {
    ve_keys_image<<<grid_img, kThreads, 0, stream>>>(a);
    MEGA_CUDA_CHECK(cudaGetLastError());
  }
  cub::DoubleBuffer<unsigned long long> dk(k0, k1);
  cub::DoubleBuffer<int> dv(v0, v1);
  if (n > 0)
    MEGA_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, dk, dv, n, 0, 32 + l.cls_shift + l.img_bits,
                                                    stream));
  if (num_images > 0) {
    ve_match_images<<<grid_img, kThreads, 0, stream>>>(a, dk.Current(), dv.Current());
    MEGA_CUDA_CHECK(cudaGetLastError());
  }
  // 3
  a.keys = k0, a.vals = v0;
  if (num_images > 0) {
    ve_keys_class<<<grid_img, kThreads, 0, stream>>>(a);
    MEGA_CUDA_CHECK(cudaGetLastError());
  }
  cub::DoubleBuffer<unsigned long long> ck(k0, k1);
  cub::DoubleBuffer<int> cv(v0, v1);
  if (n > 0) {
    MEGA_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, ck, cv, n, 0, 32 + l.cls_shift, stream));
    // 4
    const int grid_el = n / kThreads + 1 < 132 * 8 ? n / kThreads + 1 : 132 * 8;
    ve_gather<<<grid_el, kThreads, 0, stream>>>(a, ck.Current(), cv.Current());
    MEGA_CUDA_CHECK(cudaGetLastError());
    ve_cumsum_classes<<<grid_pc, 32, 0, stream>>>(a);
    MEGA_CUDA_CHECK(cudaGetLastError());
    ve_prec_rec<<<grid_el, kThreads, 0, stream>>>(a, ck.Current());
    MEGA_CUDA_CHECK(cudaGetLastError());
  }
  ve_steps_classes<<<grid_pc, 32, 0, stream>>>(a);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
