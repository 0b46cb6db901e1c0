// Seq-NMS over whole videos (mega_seq_nms, include/mega_b200.h); the per-item bodies and the contract are in
// seq_nms.cuh. Three launches on the caller's stream:
//   bucket  : one thread per (frame, class), binary search of the class's slot range in the frame's ascending labels;
//   links   : one thread per (frame, slot, 64-slot word of the next frame): the link bits, all pairs independent;
//   iterate : one warp per (video, class) runs the select / rescore / suppress loop with the DP values in global
//             memory (L2-resident: a long video's values do not fit in shared memory). Warps are independent, so a CTA
//             holds four of them and never synchronises beyond its warps.
// Every result is written by exactly one thread, no atomics: the output does not depend on scheduling.
#include "common.cuh"
#include "seq_nms.cuh"
#include "mega_b200.h"

namespace {

using namespace mega_seq;

constexpr int kWarpsPerCta = 4;

struct WarpLanes {
  __device__ __forceinline__ int lane() const { return threadIdx.x & 31; }
  __device__ __forceinline__ int count() const { return 32; }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ bool any(bool p) const { return __any_sync(0xffffffffu, p) != 0; }
  // every lane ends with the best (value, key) of the warp: larger value, ties to the smaller key
  __device__ __forceinline__ void argmax(double& v, int& key) const {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, v, off);
      const int ok = __shfl_xor_sync(0xffffffffu, key, off);
      if (seq_better(ov, ok, v, key)) {
        v = ov;
        key = ok;
      }
    }
  }
};

__global__ void __launch_bounds__(256) seq_bucket_kernel(SeqArgs a, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    seq_bucket_item(a, i);
}

__global__ void __launch_bounds__(256) seq_link_kernel(SeqArgs a, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    seq_link_item(a, i);
}

__global__ void __launch_bounds__(32 * kWarpsPerCta) seq_iterate_kernel(SeqArgs a, int num_items) {
  const int item = blockIdx.x * kWarpsPerCta + static_cast<int>(threadIdx.x >> 5);
  if (item >= num_items) return;   // uniform per warp
  seq_video_class(a, WarpLanes(), item / a.num_classes, item % a.num_classes);
}

int grid_for(long long n) {
  const long long g = (n + 255) / 256;
  return static_cast<int>(g < 65536 ? (g > 0 ? g : 1) : 65536);
}

}  // namespace

extern "C" long long mega_seq_nms_workspace_bytes(int num_frames, int max_det, int num_classes) {
  if (num_frames < 1 || max_det < 1 || max_det > kMaxDet || num_classes < 1) return -1;
  return seq_workspace_layout(num_frames, max_det, num_classes, nullptr, nullptr);
}

extern "C" int mega_seq_nms(const float* boxes, const float* scores, const int* labels, const int* counts,
                            int num_frames, int max_det, const int* video_offsets, int num_videos, int num_classes,
                            float link_iou, float nms_iou, int rescore, void* workspace, long long workspace_bytes,
                            float* out_scores, unsigned char* keep, void* stream_) {
  MEGA_ARG_CHECK(num_frames >= 1 && max_det >= 1 && max_det <= kMaxDet,
                 "seq_nms: need num_frames >= 1 and 1 <= max_det <= %d (got %d, %d)", kMaxDet, num_frames, max_det);
  MEGA_ARG_CHECK(num_videos >= 1 && num_classes >= 1, "seq_nms: need num_videos >= 1 and num_classes >= 1");
  MEGA_ARG_CHECK(static_cast<long long>(num_videos) * num_classes <= 0x7fffffffLL, "seq_nms: too many (video, class) pairs");
  MEGA_ARG_CHECK(rescore == 0 || rescore == 1, "seq_nms: rescore must be 0 (avg) or 1 (max), got %d", rescore);
  MEGA_ARG_CHECK(boxes && scores && labels && counts && video_offsets && out_scores && keep,
                 "seq_nms: null tensor pointer");
  MEGA_ARG_CHECK(reinterpret_cast<uintptr_t>(boxes) % 16 == 0, "seq_nms: boxes must be 16-byte aligned");
  const long long need = mega_seq_nms_workspace_bytes(num_frames, max_det, num_classes);
  MEGA_ARG_CHECK(workspace && workspace_bytes >= need && reinterpret_cast<uintptr_t>(workspace) % 256 == 0,
                 "seq_nms: workspace must be 256-byte aligned and hold %lld bytes (got %lld)", need, workspace_bytes);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SeqArgs a = seq_make_args(boxes, scores, labels, counts, num_frames, max_det, video_offsets, num_classes,
                                  link_iou, nms_iou, rescore, workspace, out_scores, keep);
  const long long n_bucket = static_cast<long long>(num_frames) * num_classes;
  seq_bucket_kernel<<<grid_for(n_bucket), 256, 0, stream>>>(a, n_bucket);
  MEGA_CUDA_CHECK(cudaGetLastError());
  const long long n_link = static_cast<long long>(num_frames) * max_det * a.words;
  seq_link_kernel<<<grid_for(n_link), 256, 0, stream>>>(a, n_link);
  MEGA_CUDA_CHECK(cudaGetLastError());
  const int items = num_videos * num_classes;
  seq_iterate_kernel<<<(items + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, stream>>>(a, items);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
