// Proposal recall over a whole dataset (mega_proposal_recall, include/mega_b200.h) in one launch: each CTA takes images
// blockIdx.x, blockIdx.x + gridDim.x, ... (one CTA per image up to kMaxCtas images) and runs the per-image body of
// proposal_recall.cuh with its 256 threads: shared-memory sort (one lane), IoU matrix, greedy rounds with a block-wide arg-max.
// The counts reach the output through one integer atomic per CTA and counter, so the result does not depend on
// scheduling.
#include "common.cuh"
#include "proposal_recall.cuh"
#include "mega_b200.h"

namespace {

using namespace mega_pr;

struct CtaLanes {
  float* red_v;
  unsigned* red_k;
  __device__ __forceinline__ int lane() const { return threadIdx.x; }
  __device__ __forceinline__ int count() const { return kThreads; }
  __device__ __forceinline__ void sync() const { __syncthreads(); }
  // every thread ends with the CTA's best (value, key). The scratch is read again only after the caller's next barrier.
  __device__ __forceinline__ void argmax(float& v, unsigned& key) const {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, off);
      const unsigned ok = __shfl_xor_sync(0xffffffffu, key, off);
      if (pr_better(ov, ok, v, key)) {
        v = ov;
        key = ok;
      }
    }
    if ((threadIdx.x & 31) == 0) {
      red_v[threadIdx.x >> 5] = v;
      red_k[threadIdx.x >> 5] = key;
    }
    __syncthreads();
    v = red_v[0];
    key = red_k[0];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) {
      if (pr_better(red_v[w], red_k[w], v, key)) {
        v = red_v[w];
        key = red_k[w];
      }
    }
  }
};

__global__ void __launch_bounds__(kThreads) proposal_recall_kernel(PrArgs a, long long keys_bytes,
                                                                   unsigned long long* stats) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float red_v[kThreads / 32];
  __shared__ unsigned red_k[kThreads / 32];
  PrItem* keys = reinterpret_cast<PrItem*>(smem);
  float* smat = reinterpret_cast<float*>(smem + keys_bytes);
  float* gslot = a.gmatrix ? a.gmatrix + blockIdx.x * a.slot_floats : nullptr;
  const CtaLanes lanes = {red_v, red_k};
  PrCounts c = {0, 0, 0};
  for (int img = blockIdx.x; img < a.num_images; img += gridDim.x) pr_image(a, lanes, img, keys, smat, gslot, c);
  if (threadIdx.x == 0) {
    if (c.hits) atomicAdd(&stats[0], c.hits);
    if (c.num_pos) atomicAdd(&stats[1], c.num_pos);
    if (c.rejected) atomicAdd(&stats[2], c.rejected);
  }
}

}  // namespace

extern "C" long long mega_proposal_recall_workspace_bytes(int num_images, int max_props, int max_gt, int limit) {
  PrLayout l;
  return pr_layout(num_images, max_props, max_gt, limit, &l) ? l.workspace_bytes : -1;
}

extern "C" int mega_proposal_recall(const float* prop_boxes, const float* prop_scores, const long long* prop_offsets,
                                    const float* gt_boxes, const long long* gt_offsets, int num_images, int max_props,
                                    int max_gt, int limit, float iou_thresh, void* workspace, long long workspace_bytes,
                                    float* gt_overlaps, unsigned long long* stats, void* stream_) {
  MEGA_ARG_CHECK(max_props >= 0 && max_props <= kMaxProps,
                 "proposal_recall: at most %d proposals per image are supported (max_props = %d)", kMaxProps, max_props);
  MEGA_ARG_CHECK(num_images >= 0 && max_gt >= 0 && limit >= 0,
                 "proposal_recall: need num_images, max_gt and limit >= 0 (got %d, %d, %d)", num_images, max_gt, limit);
  PrLayout l;
  MEGA_ARG_CHECK(pr_layout(num_images, max_props, max_gt, limit, &l),
                 "proposal_recall: IoU matrix of min(max_props, limit) x max_gt = %d x %d entries is too large",
                 max_props < limit ? max_props : limit, max_gt);
  MEGA_ARG_CHECK(stats && prop_offsets && gt_offsets, "proposal_recall: null stats or offsets pointer");
  MEGA_ARG_CHECK(reinterpret_cast<uintptr_t>(prop_boxes) % 16 == 0 && reinterpret_cast<uintptr_t>(gt_boxes) % 16 == 0,
                 "proposal_recall: boxes must be 16-byte aligned");
  MEGA_ARG_CHECK(l.workspace_bytes == 0 ||
                     (workspace && workspace_bytes >= l.workspace_bytes && reinterpret_cast<uintptr_t>(workspace) % 256 == 0),
                 "proposal_recall: workspace must be 256-byte aligned and hold %lld bytes (got %lld)", l.workspace_bytes,
                 workspace_bytes);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MEGA_CUDA_CHECK(cudaMemsetAsync(stats, 0, 3 * sizeof(unsigned long long), stream));
  if (num_images == 0) return MEGA_OK;
  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(proposal_recall_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         8 * kMaxProps + kSmemMatrixBytes));
    configured = true;
  }
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
  const size_t smem = static_cast<size_t>(l.keys_bytes + l.smem_matrix_bytes);
  proposal_recall_kernel<<<l.grid, kThreads, smem, stream>>>(a, l.keys_bytes, stats);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
