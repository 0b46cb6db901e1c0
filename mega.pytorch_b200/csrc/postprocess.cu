// Box-head post-processing on the device (one launch pair instead of ~60 host syncs per frame).
//
// Reference: PostProcessor.forward / filter_results
// (mega_core/modeling/roi_heads/box_head/inference.py:45-149): softmax over classes; decode with
// weights (10,10,5,5) (box_coder.py:52-95); clip; for every foreground class j: score > thresh ->
// NMS(0.5) (the reference loops over 30 classes calling _C.nms and nonzero(), each a host sync);
// concatenate class by class; if more than `detections_per_img` survive, keep those whose score is
// >= the (n - D + 1)-th smallest (torch.kthvalue on the CPU, inference.py:141-148).
#include "common.cuh"
#include "box_head.cuh"
#include "iou.cuh"
#include "mega_b200.h"

namespace mega {

constexpr int kMaxRois = 512;      // proposals per image handled by one CTA
constexpr int kPostThreads = 512;

__device__ __forceinline__ uint32_t pf2ord(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

struct PostParams {
  const float* logits;   // [R, ld_logits], num_classes valid columns
  int ld_logits;
  const float* deltas;   // [R, ld_deltas], 4*num_classes valid columns
  int ld_deltas;
  const float* proposals;  // [R,4]
  const int* count_ptr;    // device scalar: valid proposals (<= R)
  int r_max;
  int num_classes;
  float im_w, im_h, score_thresh, nms_thresh;
  float wx, wy, ww, wh;
  // per (class, proposal) staging
  float4* cls_boxes;     // [num_classes][r_max]
  float* cls_scores;     // [num_classes][r_max]
  unsigned char* cls_keep;  // [num_classes][r_max]
};

// grid = num_classes - 1 (class j = blockIdx.x + 1)
__global__ void __launch_bounds__(kPostThreads, 1) box_class_nms_kernel(const PostParams p) {
  __shared__ uint64_t skeys[kMaxRois];
  __shared__ float4 sbox[kMaxRois];
  __shared__ float sarea[kMaxRois];
  __shared__ unsigned long long smask[kMaxRois][kMaxRois / 64];
  __shared__ int s_n;
  const int j = blockIdx.x + 1;
  const int tid = threadIdx.x;
  const int R = min(*p.count_ptr, p.r_max);
  float4* ob = p.cls_boxes + static_cast<long long>(j) * p.r_max;
  float* os = p.cls_scores + static_cast<long long>(j) * p.r_max;
  unsigned char* ok = p.cls_keep + static_cast<long long>(j) * p.r_max;
  for (int r = tid; r < kMaxRois; r += blockDim.x) skeys[r] = ~0ULL;
  __syncthreads();

  // softmax probability of class j, decode, clip
  for (int r = tid; r < p.r_max; r += blockDim.x) {
    unsigned char cand = 0;
    if (r < R) {
      const float prob = class_softmax_prob(p.logits + static_cast<long long>(r) * p.ld_logits, p.num_classes, j);
      const float4 box = *reinterpret_cast<const float4*>(p.proposals + static_cast<long long>(r) * 4);
      const float4 o = decode_clip_box(p.deltas + static_cast<long long>(r) * p.ld_deltas + j * 4, box,
                                       BoxCoderW{p.wx, p.wy, p.ww, p.wh}, p.im_w, p.im_h);
      ob[r] = o;
      os[r] = prob;
      cand = prob > p.score_thresh;
      if (cand) skeys[r] = (static_cast<uint64_t>(~pf2ord(prob)) << 32) | static_cast<uint32_t>(r);
    }
    ok[r] = 0;
  }
  __syncthreads();
  // sort candidates: score descending, proposal index ascending
  for (int k = 2; k <= kMaxRois; k <<= 1) {
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int t = tid; t < kMaxRois / 2; t += blockDim.x) {
        const int i = ((t & ~(jj - 1)) << 1) | (t & (jj - 1));
        const int l = i | jj;
        const bool up = ((i & k) == 0);
        const uint64_t a = skeys[i], b = skeys[l];
        if ((a > b) == up) {
          skeys[i] = b;
          skeys[l] = a;
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    int n = 0;
    while (n < kMaxRois && skeys[n] != ~0ULL) ++n;
    s_n = n;
  }
  __syncthreads();
  const int n = s_n;
  for (int i = tid; i < n; i += blockDim.x) {
    const float4 b = ob[static_cast<int>(skeys[i] & 0xffffffffu)];
    sbox[i] = b;
    sarea[i] = box_area_plus1(b);
  }
  __syncthreads();
  const int cb = (n + 63) / 64;
  // same keep / suppress outcome as dividing (iou.cuh): the division only runs within 2^-20 of the threshold
  const float t_lo = __fmul_rn(p.nms_thresh, 1.f - 9.5367431640625e-07f), t_hi = __fmul_rn(p.nms_thresh, 1.f + 9.5367431640625e-07f);
  for (int t = tid; t < n * cb; t += blockDim.x) {
    const int i = t / cb, c = t - i * cb;
    unsigned long long bits = 0;
    const int jend = min(64, n - c * 64);
    const float4 bi = sbox[i];
    const float ai = sarea[i];
    for (int q = max(0, i + 1 - c * 64); q < jend; ++q) {
      const int o = c * 64 + q;
      if (iou_plus1_gt(bi, ai, sbox[o], sarea[o], p.nms_thresh, t_lo, t_hi)) bits |= 1ULL << q;
    }
    smask[i][c] = bits;
  }
  __syncthreads();
  if (tid == 0) {
    unsigned long long remv[kMaxRois / 64];
    for (int c = 0; c < kMaxRois / 64; ++c) remv[c] = 0;
    for (int i = 0; i < n; ++i) {
      if (!((remv[i >> 6] >> (i & 63)) & 1ULL)) {
        ok[static_cast<int>(skeys[i] & 0xffffffffu)] = 1;
        for (int c = i >> 6; c < cb; ++c) remv[c] |= smask[i][c];
      }
    }
  }
}

__global__ void __launch_bounds__(1024, 1) box_final_kernel(const FinalParams p) {
  __shared__ int hist[256];
  __shared__ int warp_sums[32];
  __shared__ int s_total, s_running, s_remaining;
  __shared__ uint32_t s_prefix;
  const int tid = threadIdx.x;
  const int total_slots = (p.num_classes - 1) * p.r_max;  // classes 1..C-1, class-major
  const unsigned char* keep = p.cls_keep + p.r_max;
  const float* scores = p.cls_scores + p.r_max;
  const float4* boxes = p.cls_boxes + p.r_max;
  if (tid == 0) {
    s_total = 0;
    s_running = 0;
  }
  __syncthreads();
  int local = 0;
  for (int i = tid; i < total_slots; i += blockDim.x) local += keep[i];
  for (int off = 16; off > 0; off >>= 1) local += __shfl_xor_sync(0xffffffffu, local, off);
  if ((tid & 31) == 0) atomicAdd(&s_total, local);
  __syncthreads();
  const int total = s_total;
  uint32_t thr_key = 0;  // keep everything with ord(score) >= thr_key
  if (total > p.max_det && p.max_det > 0) {
    // value of the max_det-th largest kept score == kthvalue(n - D + 1)
    if (tid == 0) {
      s_prefix = 0;
      s_remaining = p.max_det;
    }
    __syncthreads();
    uint32_t sel_mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix;
      for (int i = tid; i < total_slots; i += blockDim.x) {
        if (keep[i]) {
          const uint32_t key = ~pf2ord(scores[i]);  // ascending key == descending score
          if ((key & sel_mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1);
        }
      }
      __syncthreads();
      if (tid == 0) {
        int cum = 0, rem = s_remaining, b = 0;
        for (b = 0; b < 256; ++b) {
          if (cum + hist[b] >= rem) break;
          cum += hist[b];
        }
        if (b > 255) b = 255;
        s_prefix = prefix | (static_cast<uint32_t>(b) << shift);
        s_remaining = rem - cum;
      }
      sel_mask |= 0xffu << shift;
      __syncthreads();
    }
    thr_key = ~s_prefix;  // back to ascending-score order value
  }
  // ordered compaction: class-major, proposal index ascending inside a class. The reference's filter_results concatenates each
  // class's boxlist_nms output, i.e. score-descending inside a class (box_head/inference.py:111-136): the SAME detections in a
  // different order within a class (INTEGRATION.md; evaluation sorts by score itself)
  for (int base = 0; base < total_slots; base += blockDim.x) {
    const int i = base + tid;
    const int f = (i < total_slots) && keep[i] && (pf2ord(scores[i]) >= thr_key);
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    const int lane = tid & 31, warp = tid >> 5;
    const int within = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_sums[warp] = __popc(bal);
    __syncthreads();
    int before = s_running;
    for (int w = 0; w < warp; ++w) before += warp_sums[w];
    const int pos = before + within;
    if (f && pos < p.out_cap) {
      const float4 b = boxes[i];
      p.out_boxes[pos * 4 + 0] = b.x;
      p.out_boxes[pos * 4 + 1] = b.y;
      p.out_boxes[pos * 4 + 2] = b.z;
      p.out_boxes[pos * 4 + 3] = b.w;
      p.out_scores[pos] = scores[i];
      p.out_labels[pos] = static_cast<long long>(i / p.r_max + 1);
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < (blockDim.x >> 5); ++w) tot += warp_sums[w];
      s_running += tot;
    }
    __syncthreads();
  }
  if (tid == 0) p.out_count[0] = min(s_running, p.out_cap);
}

void launch_box_final(const FinalParams& f, cudaStream_t stream) { box_final_kernel<<<1, 1024, 0, stream>>>(f); }

static size_t align_up_pp(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace mega

using namespace mega;

extern "C" long long mega_box_postprocess_workspace_bytes(int r_max, int num_classes) {
  if (r_max < 1 || r_max > kMaxRois || num_classes < 2) return -1;
  size_t b = 0;
  b += align_up_pp(sizeof(float4) * r_max * num_classes, 256);
  b += align_up_pp(sizeof(float) * r_max * num_classes, 256);
  b += align_up_pp(static_cast<size_t>(r_max) * num_classes, 256);
  return static_cast<long long>(b);
}

extern "C" int mega_box_postprocess(const float* logits, int ld_logits, const float* deltas, int ld_deltas,
                                    const float* proposals, const int* count_ptr, int r_max, int num_classes,
                                    float im_w, float im_h, float score_thresh, float nms_thresh, int max_det,
                                    float wx, float wy, float ww, float wh, void* workspace,
                                    long long workspace_bytes, float* out_boxes, float* out_scores,
                                    long long* out_labels, int out_cap, int* out_count, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(r_max >= 1 && r_max <= kMaxRois, "box_postprocess: r_max must be in [1, %d]", kMaxRois);
  MEGA_ARG_CHECK(num_classes >= 2, "box_postprocess: need at least one foreground class");
  MEGA_ARG_CHECK(count_ptr != nullptr, "box_postprocess: count_ptr is null");
  MEGA_ARG_CHECK(reinterpret_cast<uintptr_t>(proposals) % 16 == 0, "box_postprocess: proposals must be 16-byte aligned");
  MEGA_ARG_CHECK(ld_logits >= num_classes && ld_deltas >= 4 * num_classes, "box_postprocess: row pitches %d / %d below "
                 "%d logits / %d deltas", ld_logits, ld_deltas, num_classes, 4 * num_classes);
  const long long need = mega_box_postprocess_workspace_bytes(r_max, num_classes);
  MEGA_ARG_CHECK(workspace && workspace_bytes >= need, "box_postprocess: workspace too small (%lld < %lld)",
                 workspace_bytes, need);
  char* w = static_cast<char*>(workspace);
  PostParams p;
  p.logits = logits;
  p.ld_logits = ld_logits;
  p.deltas = deltas;
  p.ld_deltas = ld_deltas;
  p.proposals = proposals;
  p.count_ptr = count_ptr;
  p.r_max = r_max;
  p.num_classes = num_classes;
  p.im_w = im_w;
  p.im_h = im_h;
  p.score_thresh = score_thresh;
  p.nms_thresh = nms_thresh;
  p.wx = wx; p.wy = wy; p.ww = ww; p.wh = wh;
  p.cls_boxes = reinterpret_cast<float4*>(w);
  w += align_up_pp(sizeof(float4) * r_max * num_classes, 256);
  p.cls_scores = reinterpret_cast<float*>(w);
  w += align_up_pp(sizeof(float) * r_max * num_classes, 256);
  p.cls_keep = reinterpret_cast<unsigned char*>(w);
  box_class_nms_kernel<<<num_classes - 1, kPostThreads, 0, stream>>>(p);
  FinalParams f;
  f.cls_boxes = p.cls_boxes;
  f.cls_scores = p.cls_scores;
  f.cls_keep = p.cls_keep;
  f.r_max = r_max;
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
