// Test-time box augmentation (TEST.BBOX_AUG) on the device: per pass a collect launch stages the pass's raw
// post-processor output, mapped to the identity pass's frame, in a class-major area; one merge launch pair then does
// what filter_results does on the concatenation (box_head/inference.py:108-149): per foreground class, score >
// SCORE_THRESH, NMS, concatenation, and the DETECTIONS_PER_IMG kthvalue cap. The reference runs that merge on the host
// as 30 boxlist_nms calls with a host sync each (engine/bbox_aug.py:57-66).
//
// Merge: one CTA per class. The class's candidates (<= kAugMaxCand merged rows) are bitonic-sorted in shared memory
// (score descending, merged row ascending), then swept by the chunked greedy NMS of rpn_nms_greedy_kernel
// (proposals.cu): 64 candidates at a time are tested against the kept list in shared memory and then against each
// other, and warp 0 resolves the chunk in order. The kept list holds every candidate, so it cannot overflow; the sweep
// ends early at the exact cap stop of aug_past_cap. Kept rows are flagged in place and box_final_kernel
// (postprocess.cu), unchanged, applies the cap and compacts class-major in merged-row order.
#include "bbox_aug.cuh"
#include "common.cuh"
#include "mega_b200.h"

namespace mega {

constexpr int kAugCollectThreads = 256;
constexpr int kAugMergeThreads = 512;

__global__ void bbox_aug_collect_kernel(const AugCollectArgs a, const int* __restrict__ count_ptr) {
  const int count = min(*count_ptr, a.r_max);
  const long long total = static_cast<long long>(a.num_classes - 1) * a.r_max;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    aug_collect_item(a, count, i);
}

struct AugMergeParams {
  const float4* boxes;
  const float* scores;
  unsigned char* flags;    // in: candidate flags, out: kept flags
  int rows, key_cap, max_det;
  float thresh;
};

// dynamic shared memory: keys [key_cap] (power of two >= rows), kept boxes [rows]
__global__ void __launch_bounds__(kAugMergeThreads, 1) bbox_aug_merge_kernel(const AugMergeParams p) {
  extern __shared__ __align__(16) unsigned char aug_smem[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(aug_smem);
  float4* kept_b = reinterpret_cast<float4*>(keys + p.key_cap);
  __shared__ float4 cand[64];
  __shared__ float cand_a[64];
  __shared__ uint64_t cand_k[64];
  __shared__ unsigned long long diag[64];
  __shared__ unsigned long long sup_s;
  __shared__ int n_s, nk_s, stop_s;
  __shared__ uint32_t cap_s;
  const int j = blockIdx.x + 1;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float4* boxes = p.boxes + static_cast<long long>(j) * p.rows;
  const float* scores = p.scores + static_cast<long long>(j) * p.rows;
  unsigned char* flags = p.flags + static_cast<long long>(j) * p.rows;
  if (tid == 0) n_s = 0, nk_s = 0, stop_s = 0, cap_s = 0;
  __syncthreads();
  // 1. candidates -> keys (any order), flags cleared
  for (int i = tid; i < p.rows; i += blockDim.x) {
    if (flags[i]) {
      keys[atomicAdd(&n_s, 1)] = aug_key(scores[i], i);
      flags[i] = 0;
    }
  }
  __syncthreads();
  const int n = n_s;
  int np2 = 1;
  while (np2 < n) np2 <<= 1;
  for (int i = n + tid; i < np2; i += blockDim.x) keys[i] = ~0ULL;
  __syncthreads();
  // 2. bitonic sort of np2 keys, ascending
  for (int k = 2; k <= np2; k <<= 1) {
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int t = tid; t < np2 / 2; t += blockDim.x) {
        const int i = ((t & ~(jj - 1)) << 1) | (t & (jj - 1));
        const int l = i | jj;
        const bool up = ((i & k) == 0);
        const uint64_t a = keys[i], b = keys[l];
        if ((a > b) == up) {
          keys[i] = b;
          keys[l] = a;
        }
      }
      __syncthreads();
    }
  }
  // 3. chunked greedy NMS (rpn_nms_greedy_kernel's sweep)
  const float thresh = p.thresh;
  const float t_lo = __fmul_rn(thresh, 1.f - 9.5367431640625e-07f), t_hi = __fmul_rn(thresh, 1.f + 9.5367431640625e-07f);
  const int chunks = (n + 63) / 64;
  for (int c = 0; c < chunks; ++c) {
    const int base = c * 64;
    const int csz = min(64, n - base);
    if (tid < 64) {
      const uint64_t key = tid < csz ? keys[base + tid] : ~0ULL;
      const float4 b = tid < csz ? boxes[aug_key_row(key)] : make_float4(0.f, 0.f, 0.f, 0.f);
      cand[tid] = b;
      cand_a[tid] = box_area_plus1(b);
      cand_k[tid] = key;
      diag[tid] = 0ULL;
    }
    if (tid == 0) sup_s = csz < 64 ? (~0ULL << csz) : 0ULL;     // positions past the end count as suppressed
    __syncthreads();
    const int nk = nk_s;
    // ---- against the kept list: warp w owns candidates 4w .. 4w+3, lanes stride over the kept boxes
#pragma unroll
    for (int qq = 0; qq < 64 / (kAugMergeThreads / 32); ++qq) {
      const int q = warp * (64 / (kAugMergeThreads / 32)) + qq;
      const float4 cq = cand[q];
      const float aq = cand_a[q];
      bool hit = false;
      for (int k = lane; k < nk; k += 32) {
        const float4 kb = kept_b[k];
        hit |= iou_plus1_gt(kb, box_area_plus1(kb), cq, aq, thresh, t_lo, t_hi);
      }
      if (__any_sync(0xffffffffu, hit) && lane == 0) atomicOr(&sup_s, 1ULL << q);
    }
    // ---- the chunk against itself: thread (q, part) evaluates 8 later candidates
    {
      const int q = tid >> 3, part = tid & 7;
      const float4 cq = cand[q];
      const float aq = cand_a[q];
      unsigned long long bits = 0;
#pragma unroll
      for (int jx = 0; jx < 8; ++jx) {
        const int o = part * 8 + jx;
        if (o > q && o < csz && iou_plus1_gt(cq, aq, cand[o], cand_a[o], thresh, t_lo, t_hi)) bits |= 1ULL << o;
      }
      if (bits) atomicOr(&diag[q], bits);
    }
    __syncthreads();
    // ---- warp 0 resolves the chunk in order (every lane tracks the same removed set); stops at the exact cap stop
    if (warp == 0) {
      const unsigned long long d0 = diag[lane], d1 = diag[lane + 32];
      unsigned long long r = sup_s;
      int cnt = nk;
      uint32_t cap = cap_s;
      int stop = 0;
      while (r != ~0ULL) {
        const int i = __ffsll(static_cast<long long>(~r)) - 1;
        const uint64_t key = cand_k[i];
        if (aug_past_cap(cnt, p.max_det, cap, key)) {
          stop = 1;
          break;
        }
        const unsigned long long di_lo = __shfl_sync(0xffffffffu, d0, i & 31);
        const unsigned long long di_hi = __shfl_sync(0xffffffffu, d1, i & 31);
        r |= ((i < 32) ? di_lo : di_hi) | (1ULL << i);
        if (lane == 0) {
          kept_b[cnt] = cand[i];
          flags[aug_key_row(key)] = 1;
        }
        ++cnt;
        if (cnt == p.max_det) cap = static_cast<uint32_t>(key >> 32);
      }
      if (lane == 0) nk_s = cnt, cap_s = cap, stop_s = stop;
    }
    __syncthreads();
    if (stop_s) break;
  }
}

static size_t aug_align(size_t v) { return (v + 255) / 256 * 256; }

static int aug_key_cap(int rows) {
  int np2 = 1;
  while (np2 < rows) np2 <<= 1;
  return np2;
}

static size_t aug_merge_smem(int rows) { return static_cast<size_t>(aug_key_cap(rows)) * 8 + static_cast<size_t>(rows) * 16; }

}  // namespace mega

using namespace mega;

extern "C" long long mega_bbox_aug_workspace_bytes(int num_passes, int r_max, int num_classes) {
  if (num_passes < 1 || r_max < 1 || num_classes < 2) return -1;
  if (static_cast<long long>(num_passes) * r_max > kAugMaxCand) return -1;
  const size_t slots = static_cast<size_t>(num_passes) * r_max * num_classes;
  return static_cast<long long>(aug_align(sizeof(float4) * slots) + aug_align(sizeof(float) * slots) + aug_align(slots));
}

static int aug_check(const char* what, int num_passes, int r_max, int num_classes, const void* workspace,
                     long long workspace_bytes) {
  MEGA_ARG_CHECK(num_passes >= 1 && r_max >= 1 && num_classes >= 2,
                 "%s: need num_passes >= 1, r_max >= 1 and num_classes >= 2 (got %d, %d, %d)", what, num_passes, r_max,
                 num_classes);
  MEGA_ARG_CHECK(static_cast<long long>(num_passes) * r_max <= kAugMaxCand,
                 "%s: num_passes * r_max = %lld exceeds %d merged rows per class", what,
                 static_cast<long long>(num_passes) * r_max, kAugMaxCand);
  const long long need = mega_bbox_aug_workspace_bytes(num_passes, r_max, num_classes);
  MEGA_ARG_CHECK(workspace && workspace_bytes >= need, "%s: workspace too small (%lld < %lld)", what, workspace_bytes,
                 need);
  return MEGA_OK;
}

extern "C" int mega_bbox_aug_collect(const float* logits, int ld_logits, const float* deltas, int ld_deltas,
                                     const float* proposals, const int* count_ptr, int r_max, int num_classes, int pass,
                                     int num_passes, int im_w, int im_h, int hflip, double ratio_w, double ratio_h,
                                     float score_thresh, float wx, float wy, float ww, float wh, void* workspace,
                                     long long workspace_bytes, void* stream_v) {
  const int st = aug_check("bbox_aug_collect", num_passes, r_max, num_classes, workspace, workspace_bytes);
  if (st != MEGA_OK) return st;
  MEGA_ARG_CHECK(pass >= 0 && pass < num_passes, "bbox_aug_collect: pass %d outside [0, %d)", pass, num_passes);
  MEGA_ARG_CHECK(count_ptr != nullptr && logits && deltas && proposals, "bbox_aug_collect: null input");
  MEGA_ARG_CHECK(ld_logits >= num_classes && ld_deltas >= 4 * num_classes, "bbox_aug_collect: row pitch too small");
  MEGA_ARG_CHECK(im_w > 0 && im_h > 0, "bbox_aug_collect: empty image");
  const int rows = num_passes * r_max;
  const size_t slots = static_cast<size_t>(rows) * num_classes;
  char* w = static_cast<char*>(workspace);
  AugCollectArgs a;
  a.logits = logits, a.ld_logits = ld_logits, a.deltas = deltas, a.ld_deltas = ld_deltas, a.proposals = proposals;
  a.r_max = r_max, a.num_classes = num_classes, a.slot = pass, a.rows = rows;
  a.im_w = static_cast<float>(im_w), a.im_h = static_cast<float>(im_h), a.hflip = hflip ? 1 : 0;
  a.ratio_w = static_cast<float>(ratio_w), a.ratio_h = static_cast<float>(ratio_h);
  a.score_thresh = score_thresh;
  a.w = BoxCoderW{wx, wy, ww, wh};
  a.boxes = reinterpret_cast<float4*>(w);
  a.scores = reinterpret_cast<float*>(w + aug_align(sizeof(float4) * slots));
  a.cand = reinterpret_cast<unsigned char*>(w + aug_align(sizeof(float4) * slots) + aug_align(sizeof(float) * slots));
  const long long total = static_cast<long long>(num_classes - 1) * r_max;
  const int blocks = static_cast<int>((total + kAugCollectThreads - 1) / kAugCollectThreads);
  bbox_aug_collect_kernel<<<blocks, kAugCollectThreads, 0, static_cast<cudaStream_t>(stream_v)>>>(a, count_ptr);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_bbox_aug_merge(int num_passes, int r_max, int num_classes, float nms_thresh, int max_det,
                                   void* workspace, long long workspace_bytes, float* out_boxes, float* out_scores,
                                   long long* out_labels, int out_cap, int* out_count, void* stream_v) {
  const int st = aug_check("bbox_aug_merge", num_passes, r_max, num_classes, workspace, workspace_bytes);
  if (st != MEGA_OK) return st;
  MEGA_ARG_CHECK(out_boxes && out_scores && out_labels && out_count && out_cap >= 0, "bbox_aug_merge: null output");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int rows = num_passes * r_max;
  const size_t slots = static_cast<size_t>(rows) * num_classes;
  char* w = static_cast<char*>(workspace);
  AugMergeParams p;
  p.boxes = reinterpret_cast<const float4*>(w);
  p.scores = reinterpret_cast<const float*>(w + aug_align(sizeof(float4) * slots));
  p.flags = reinterpret_cast<unsigned char*>(w + aug_align(sizeof(float4) * slots) + aug_align(sizeof(float) * slots));
  p.rows = rows;
  p.key_cap = aug_key_cap(rows);
  p.max_det = max_det;
  p.thresh = nms_thresh;
  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(bbox_aug_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(aug_merge_smem(kAugMaxCand))));
    configured = true;
  }
  bbox_aug_merge_kernel<<<num_classes - 1, kAugMergeThreads, aug_merge_smem(rows), stream>>>(p);
  FinalParams f;
  f.cls_boxes = p.boxes;
  f.cls_scores = p.scores;
  f.cls_keep = p.flags;
  f.r_max = rows;
  f.num_classes = num_classes;
  f.max_det = max_det;
  f.out_cap = out_cap;
  f.out_boxes = out_boxes;
  f.out_scores = out_scores;
  f.out_labels = out_labels;
  f.out_count = out_count;
  launch_box_final(f, stream);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
