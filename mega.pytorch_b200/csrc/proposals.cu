// Greedy NMS and RPN proposal selection, entirely on the device (no host round trips).
//
// Reference behaviour restated here:
//   * nms_cuda (mega_core/csrc/cuda/nms.cu:70-131): sort by score, 64x64 IoU bitmask with the
//     "+1" pixel convention and the strict `>` rule (nms.cu:13-21, :60), greedy sweep -- which the
//     reference runs on the HOST after a 4.5 MB device->host copy (nms.cu:99-123); here the sweep
//     is a single-CTA kernel and nothing leaves the device;
//   * RPNPostProcessor.forward_for_single_feature_map (modeling/rpn/inference.py:76-123):
//     sigmoid -> top-k sorted -> BoxCoder.decode (modeling/box_coder.py:52-95) -> clip_to_image
//     (structures/bounding_box.py:214-224) -> remove_small_boxes (structures/boxlist_ops.py:34-48)
//     -> NMS -> first post_nms_top_n.
// Tie rule for equal scores: ascending original index (a stable sort; the reference's GPU sort
// leaves it unspecified, nms.cu:74).
#include "common.cuh"
#include "iou.cuh"
#include "mega_b200.h"

namespace mega {

constexpr int kNmsMaxBoxes = 8192;  // single-CTA bitonic sort capacity
constexpr int kSortThreads = 1024;

__device__ __forceinline__ uint32_t f2ord(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t o) {
  uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(b);
}

// ascending bitonic sort of n (power of two) 64-bit keys held in shared memory
__device__ void bitonic_sort_u64(uint64_t* keys, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int l = i | j;
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
}

__device__ __forceinline__ int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// IoU with the "+1" convention; explicit _rn ops so that no FMA contraction changes a
// comparison against the threshold (bit-exact with the C oracle / the reference kernel).
__device__ __forceinline__ float iou_plus1(const float4 a, const float4 b) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float width = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
  const float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
  const float inter = __fmul_rn(width, height);
  const float sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.f), __fadd_rn(__fsub_rn(a.w, a.y), 1.f));
  const float sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter));
}

// mask[img][i][cb]: bit j of word c set <=> IoU(box i, box c*64+j) > thresh (only c >= i/64)
__global__ void nms_mask_kernel(const float4* __restrict__ boxes, long long boxes_img_stride,
                                const int* __restrict__ n_ptr, int n_host, float thresh,
                                unsigned long long* __restrict__ mask, long long mask_img_stride,
                                int col_blocks) {
  const int img = blockIdx.z;
  const int n = n_ptr ? n_ptr[img] : n_host;
  const int row_start = blockIdx.y, col_start = blockIdx.x;
  if (col_start < row_start) return;
  if (row_start * 64 >= n || col_start * 64 >= n) return;
  const float4* b = boxes + img * boxes_img_stride;
  const int row_size = min(n - row_start * 64, 64);
  const int col_size = min(n - col_start * 64, 64);
  __shared__ float4 blk[64];
  if (threadIdx.x < col_size) blk[threadIdx.x] = b[col_start * 64 + threadIdx.x];
  __syncthreads();
  if (threadIdx.x < row_size) {
    const int cur = row_start * 64 + threadIdx.x;
    const float4 cb = b[cur];
    unsigned long long t = 0;
    const int start = (row_start == col_start) ? threadIdx.x + 1 : 0;
    for (int i = start; i < col_size; ++i) {
      if (iou_plus1(cb, blk[i]) > thresh) t |= 1ULL << i;
    }
    mask[img * mask_img_stride + static_cast<long long>(cur) * col_blocks + col_start] = t;
  }
}

// greedy sweep over the bitmask: one CTA (128 threads) per image; keeps at most max_keep boxes.
// kept_pos[img][0..count) = positions (in sorted order) of the kept boxes, ascending.
__global__ void nms_sweep_kernel(const unsigned long long* __restrict__ mask, long long mask_img_stride,
                                 const unsigned char* __restrict__ valid, long long valid_img_stride,
                                 const int* __restrict__ n_ptr, int n_host, int col_blocks, int max_keep,
                                 int* __restrict__ kept_pos, long long kept_img_stride, int* __restrict__ kept_count) {
  const int img = blockIdx.x;
  const int n = n_ptr ? n_ptr[img] : n_host;
  const unsigned long long* m = mask + img * mask_img_stride;
  const unsigned char* v = valid ? valid + img * valid_img_stride : nullptr;
  int* kp = kept_pos + img * kept_img_stride;
  __shared__ unsigned long long remv[kNmsMaxBoxes / 64];
  __shared__ unsigned long long diag[64];
  __shared__ unsigned long long kept_bits_s;
  __shared__ int kept_cnt;
  const int tid = threadIdx.x;
  const int cb_used = (n + 63) / 64;
  for (int j = tid; j < kNmsMaxBoxes / 64; j += blockDim.x) {
    unsigned long long r = 0;
    if (v && j < cb_used) {
      for (int i = 0; i < 64; ++i) {
        const int p = j * 64 + i;
        if (p < n && !v[p]) r |= 1ULL << i;
      }
    }
    remv[j] = r;
  }
  if (tid == 0) kept_cnt = 0;
  __syncthreads();
  for (int c = 0; c < cb_used; ++c) {
    if (tid < 64) {
      const int i = c * 64 + tid;
      diag[tid] = (i < n) ? m[static_cast<long long>(i) * col_blocks + c] : 0ULL;
    }
    __syncthreads();
    if (tid == 0) {
      unsigned long long r = remv[c], kb = 0;
      int cnt = kept_cnt;
      const int lim = min(64, n - c * 64);
      for (int i = 0; i < lim && cnt < max_keep; ++i) {
        if (!((r >> i) & 1ULL)) {
          kb |= 1ULL << i;
          r |= diag[i];
          kp[cnt++] = c * 64 + i;
        }
      }
      kept_bits_s = kb;
      kept_cnt = cnt;
    }
    __syncthreads();
    if (kept_cnt >= max_keep) break;
    unsigned long long kb = kept_bits_s;
    for (int j = c + 1 + tid; j < cb_used; j += blockDim.x) {
      unsigned long long acc = 0, bits = kb;
      while (bits) {
        const int i = __ffsll(static_cast<long long>(bits)) - 1;
        bits &= bits - 1;
        acc |= m[static_cast<long long>(c * 64 + i) * col_blocks + j];
      }
      remv[j] |= acc;
    }
    __syncthreads();
  }
  if (tid == 0) kept_count[img] = kept_cnt;
}

// ---------------------------------------------------------------- generic NMS op (mega_core._C.nms)
// sort by (score desc, index asc); writes sorted boxes and the permutation
__global__ void __launch_bounds__(kSortThreads, 1)
nms_sort_kernel(const float* __restrict__ boxes, const float* __restrict__ scores, int n,
                float4* __restrict__ sorted_boxes, int* __restrict__ order) {
  extern __shared__ uint64_t skeys[];
  const int np2 = next_pow2(max(n, 2));
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    skeys[i] = (i < n) ? ((static_cast<uint64_t>(~f2ord(scores[i])) << 32) | static_cast<uint32_t>(i))
                       : ~0ULL;
  }
  __syncthreads();
  bitonic_sort_u64(skeys, np2);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int idx = static_cast<int>(skeys[i] & 0xffffffffu);
    order[i] = idx;
    sorted_boxes[i] = make_float4(boxes[idx * 4 + 0], boxes[idx * 4 + 1], boxes[idx * 4 + 2], boxes[idx * 4 + 3]);
  }
}

// kept sorted positions -> original indices, ascending (nms.cu:127-130): flag + ordered compaction
__global__ void __launch_bounds__(kSortThreads, 1)
nms_finalize_kernel(const int* __restrict__ kept_pos, const int* __restrict__ kept_count,
                    const int* __restrict__ order, int n, long long* __restrict__ keep_out,
                    int* __restrict__ count_out) {
  __shared__ unsigned char flag[kNmsMaxBoxes];
  __shared__ int warp_sums[kSortThreads / 32];
  __shared__ int running;
  const int cnt = kept_count[0];
  for (int i = threadIdx.x; i < n; i += blockDim.x) flag[i] = 0;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) flag[order[kept_pos[i]]] = 1;
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int f = (i < n) ? flag[i] : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int within = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_sums[warp] = __popc(bal);
    __syncthreads();
    int before = running;
    for (int w = 0; w < warp; ++w) before += warp_sums[w];
    if (f) keep_out[before + within] = i;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < (blockDim.x >> 5); ++w) tot += warp_sums[w];
      running += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) count_out[0] = running;
}

// ---------------------------------------------------------------- box decode (box_coder.py:52-95)
struct DecodeW {
  float wx, wy, ww, wh, clip;
};
__device__ __forceinline__ float4 decode_box(float d0, float d1, float d2, float d3, float4 box, DecodeW w) {
  const float widths = __fadd_rn(__fsub_rn(box.z, box.x), 1.f);
  const float heights = __fadd_rn(__fsub_rn(box.w, box.y), 1.f);
  const float ctr_x = __fadd_rn(box.x, __fmul_rn(0.5f, widths));
  const float ctr_y = __fadd_rn(box.y, __fmul_rn(0.5f, heights));
  const float dx = __fdiv_rn(d0, w.wx), dy = __fdiv_rn(d1, w.wy);
  const float dw = fminf(__fdiv_rn(d2, w.ww), w.clip), dh = fminf(__fdiv_rn(d3, w.wh), w.clip);
  const float pcx = __fadd_rn(__fmul_rn(dx, widths), ctr_x);
  const float pcy = __fadd_rn(__fmul_rn(dy, heights), ctr_y);
  const float pw = __fmul_rn(expf(dw), widths);
  const float ph = __fmul_rn(expf(dh), heights);
  float4 o;
  o.x = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
  o.y = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
  o.z = __fsub_rn(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), 1.f);
  o.w = __fsub_rn(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), 1.f);
  return o;
}
__device__ __forceinline__ float4 clip_box(float4 b, float im_w, float im_h) {
  b.x = fminf(fmaxf(b.x, 0.f), im_w - 1.f);
  b.y = fminf(fmaxf(b.y, 0.f), im_h - 1.f);
  b.z = fminf(fmaxf(b.z, 0.f), im_w - 1.f);
  b.w = fminf(fmaxf(b.w, 0.f), im_h - 1.f);
  return b;
}

// ---------------------------------------------------------------- RPN: sigmoid + top-k + decode
struct RpnParams {
  const float* head;       // [n_img][H*W][ld]: channels [0,A) logits, [A, 5A) deltas (a*4+c)
  long long head_img_stride;
  int ld, A, H, W, stride;
  const float* base_anchors;  // [A,4]
  float im_w, im_h;
  int pre_nms;     // <= 8192
  float min_size;
  uint32_t* keys;  // workspace [n_img][H*W*A]
  float4* sorted_boxes;  // [n_img][8192]
  float* sorted_scores;  // [n_img][8192]
  int* sorted_anchor;    // [n_img][8192]
  unsigned char* valid;  // [n_img][8192]
  int* n_sorted;         // [n_img]
};

__global__ void __launch_bounds__(kSortThreads, 1) rpn_topk_decode_kernel(const RpnParams p) {
  extern __shared__ uint64_t skeys[];  // 8192 entries
  __shared__ int hist[256];
  __shared__ int warp_sums[kSortThreads / 32];
  __shared__ uint32_t s_prefix;
  __shared__ int s_remaining, s_cnt, s_running;
  const int img = blockIdx.x;
  const int tid = threadIdx.x;
  const int n = p.H * p.W * p.A;
  const float* head = p.head + img * p.head_img_stride;
  uint32_t* keys = p.keys + static_cast<long long>(img) * n;
  const int k = min(p.pre_nms, n);

  // 1. scores -> descending-order keys
  for (int i = tid; i < n; i += blockDim.x) {
    const int cell = i / p.A, a = i - cell * p.A;
    const float logit = head[static_cast<long long>(cell) * p.ld + a];
    const float s = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-logit)));
    keys[i] = ~f2ord(s);
  }
  if (tid == 0) {
    s_prefix = 0;
    s_remaining = k;
  }
  __syncthreads();

  // 2. radix select: value T of the k-th smallest key
  uint32_t sel_mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    // detection scores cluster (most anchors are background): whole warps fall into one bin, and 28 k same-address
    // shared-memory atomics would serialise -> one atomic per warp when its live lanes agree on the bin
    for (int base = 0; base < n; base += blockDim.x) {
      const int i = base + tid;
      const uint32_t key = i < n ? keys[i] : 0u;
      const bool live = i < n && (key & sel_mask) == prefix;
      const uint32_t bin = (key >> shift) & 255u;
      const unsigned m = __ballot_sync(0xffffffffu, live);
      if (m != 0u) {
        const int leader = __ffs(m) - 1;
        const uint32_t lb = __shfl_sync(0xffffffffu, bin, leader);
        const unsigned same = __ballot_sync(0xffffffffu, live && bin == lb);
        if (same == m) {
          if ((tid & 31) == leader) atomicAdd(&hist[lb], __popc(m));
        } else if (live) {
          atomicAdd(&hist[bin], 1);
        }
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
  const uint32_t T = s_prefix;
  const int quota_eq = s_remaining;      // how many keys == T are taken (lowest indices first)
  const int count_lt = k - quota_eq;

  // 3. compaction into the sort buffer
  const int np2 = next_pow2(max(k, 2));
  for (int i = tid; i < np2; i += blockDim.x) skeys[i] = ~0ULL;
  if (tid == 0) {
    s_cnt = 0;
    s_running = 0;
  }
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {       // order inside the sort buffer is irrelevant: one atomic per warp
    const int i = base + tid;
    const uint32_t key = i < n ? keys[i] : 0xffffffffu;
    const bool lt = i < n && key < T;
    const unsigned m = __ballot_sync(0xffffffffu, lt);
    int pos0 = 0;
    if ((tid & 31) == 0 && m != 0u) pos0 = atomicAdd(&s_cnt, __popc(m));
    pos0 = __shfl_sync(0xffffffffu, pos0, 0);
    if (lt) skeys[pos0 + __popc(m & ((1u << (tid & 31)) - 1u))] = (static_cast<uint64_t>(key) << 32) | static_cast<uint32_t>(i);
  }
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + tid;
    const int f = (i < n) && (keys[i] == T);
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    const int lane = tid & 31, warp = tid >> 5;
    const int within = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_sums[warp] = __popc(bal);
    __syncthreads();
    int before = s_running;
    for (int w = 0; w < warp; ++w) before += warp_sums[w];
    const int rank = before + within;
    if (f && rank < quota_eq) skeys[count_lt + rank] = (static_cast<uint64_t>(T) << 32) | static_cast<uint32_t>(i);
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < (blockDim.x >> 5); ++w) tot += warp_sums[w];
      s_running += tot;
    }
    __syncthreads();
    if (s_running >= quota_eq) break;
  }
  __syncthreads();

  // 4. sort (score desc, anchor index asc)
  bitonic_sort_u64(skeys, np2);

  // 5. decode + clip (+ remove_small flag)
  float4* sb = p.sorted_boxes + static_cast<long long>(img) * kNmsMaxBoxes;
  float* ss = p.sorted_scores + static_cast<long long>(img) * kNmsMaxBoxes;
  int* sa = p.sorted_anchor + static_cast<long long>(img) * kNmsMaxBoxes;
  unsigned char* sv = p.valid + static_cast<long long>(img) * kNmsMaxBoxes;
  const DecodeW dwt = {1.f, 1.f, 1.f, 1.f, 4.135166556742356f};  // log(1000/16)
  for (int q = tid; q < k; q += blockDim.x) {
    const uint64_t key = skeys[q];
    const int idx = static_cast<int>(key & 0xffffffffu);
    const float score = ord2f(~static_cast<uint32_t>(key >> 32));
    const int cell = idx / p.A, a = idx - cell * p.A;
    const int wq = cell % p.W, hq = cell / p.W;
    const float sx = static_cast<float>(wq * p.stride), sy = static_cast<float>(hq * p.stride);
    float4 anc;
    anc.x = __fadd_rn(sx, p.base_anchors[a * 4 + 0]);
    anc.y = __fadd_rn(sy, p.base_anchors[a * 4 + 1]);
    anc.z = __fadd_rn(sx, p.base_anchors[a * 4 + 2]);
    anc.w = __fadd_rn(sy, p.base_anchors[a * 4 + 3]);
    const float* d = head + static_cast<long long>(cell) * p.ld + p.A + a * 4;
    float4 box = decode_box(d[0], d[1], d[2], d[3], anc, dwt);
    box = clip_box(box, p.im_w, p.im_h);
    const float ws = __fadd_rn(__fsub_rn(box.z, box.x), 1.f), hs = __fadd_rn(__fsub_rn(box.w, box.y), 1.f);
    sb[q] = box;
    ss[q] = score;
    sa[q] = idx;
    sv[q] = (ws >= p.min_size && hs >= p.min_size) ? 1 : 0;
  }
  if (tid == 0) p.n_sorted[img] = k;
}

// writes the first `post` kept boxes (zero-filled beyond the count)
__global__ void rpn_write_kernel(const float4* __restrict__ sorted_boxes, const float* __restrict__ sorted_scores,
                                 const int* __restrict__ sorted_anchor, const int* __restrict__ kept_pos,
                                 long long kept_img_stride, const int* __restrict__ kept_count, int post,
                                 float4* __restrict__ out_boxes, float* __restrict__ out_scores,
                                 int* __restrict__ out_anchor, int* __restrict__ out_count) {
  const int img = blockIdx.x;
  const int cnt = min(kept_count[img], post);
  for (int i = threadIdx.x; i < post; i += blockDim.x) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    float s = 0.f;
    int a = -1;
    if (i < cnt) {
      const int pos = kept_pos[img * kept_img_stride + i];
      b = sorted_boxes[static_cast<long long>(img) * kNmsMaxBoxes + pos];
      s = sorted_scores[static_cast<long long>(img) * kNmsMaxBoxes + pos];
      a = sorted_anchor[static_cast<long long>(img) * kNmsMaxBoxes + pos];
    }
    out_boxes[static_cast<long long>(img) * post + i] = b;
    out_scores[static_cast<long long>(img) * post + i] = s;
    if (out_anchor) out_anchor[static_cast<long long>(img) * post + i] = a;
  }
  if (threadIdx.x == 0) out_count[img] = cnt;
}

// Greedy NMS of ONE image in ONE CTA without the n x n bitmask: candidates are taken in chunks of 64 (score order); a
// chunk is first tested against the boxes kept so far (all warps, kept list in shared memory), then resolved against
// itself with a 64 x 64 mask, and the survivors join the kept list. Only ~(#candidates x #kept) IoUs are evaluated
// (1.2 M for 6000 candidates / 300 kept, against 18 M for the full mask), the sweep stops at max_keep, and -- what
// matters on the hot path -- the kernel needs one SM, so it overlaps the persistent res5 chain that owns the others
// (nms_mask_kernel's 17 k blocks starve there). Same decisions as mask + sweep: box o goes iff a kept box i < o has
// IoU(i, o) > thresh. Also writes the padded outputs (rpn_write_kernel's job).
constexpr int kGreedyThreads = 512;
constexpr int kGreedyMaxKeep = 1024;

__global__ void __launch_bounds__(kGreedyThreads)
rpn_nms_greedy_kernel(const float4* __restrict__ sorted_boxes, const float* __restrict__ sorted_scores,
                      const int* __restrict__ sorted_anchor, const unsigned char* __restrict__ valid,
                      const int* __restrict__ n_ptr, int n_host, float thresh, int post, float4* __restrict__ out_boxes,
                      float* __restrict__ out_scores, int* __restrict__ out_anchor, int* __restrict__ out_count) {
  __shared__ float4 kept_b[kGreedyMaxKeep];
  __shared__ float kept_a[kGreedyMaxKeep];
  __shared__ int kept_p[kGreedyMaxKeep];
  __shared__ float4 cand[64];
  __shared__ float cand_a[64];
  __shared__ unsigned long long diag[64];
  __shared__ unsigned long long sup_s;
  __shared__ int nk_s;
  const int img = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = n_ptr ? n_ptr[img] : n_host;
  const float4* boxes = sorted_boxes + static_cast<long long>(img) * kNmsMaxBoxes;
  const unsigned char* v = valid ? valid + static_cast<long long>(img) * kNmsMaxBoxes : nullptr;
  const float t_lo = __fmul_rn(thresh, 1.f - 9.5367431640625e-07f), t_hi = __fmul_rn(thresh, 1.f + 9.5367431640625e-07f);
  if (tid == 0) nk_s = 0;
  __syncthreads();
  const int chunks = (n + 63) / 64;
  for (int c = 0; c < chunks; ++c) {
    const int base = c * 64;
    const int csz = min(64, n - base);
    if (tid < 64) {
      const float4 b = tid < csz ? boxes[base + tid] : make_float4(0.f, 0.f, 0.f, 0.f);
      cand[tid] = b;
      cand_a[tid] = box_area_plus1(b);
      diag[tid] = 0ULL;
    }
    if (tid == 0) {
      sup_s = csz < 64 ? (~0ULL << csz) : 0ULL;     // positions past the end count as suppressed
    }
    __syncthreads();
    if (tid < 64 && tid < csz && v && !v[base + tid]) atomicOr(&sup_s, 1ULL << tid);   // remove_small_boxes
    const int nk = nk_s;
    // ---- 1. against the kept list: warp w owns candidates 4w .. 4w+3, lanes stride over the kept boxes
#pragma unroll
    for (int qq = 0; qq < 64 / (kGreedyThreads / 32); ++qq) {
      const int q = warp * (64 / (kGreedyThreads / 32)) + qq;
      const float4 cq = cand[q];
      const float aq = cand_a[q];
      bool hit = false;
      for (int k = lane; k < nk; k += 32) hit |= iou_plus1_gt(kept_b[k], kept_a[k], cq, aq, thresh, t_lo, t_hi);
      if (__any_sync(0xffffffffu, hit) && lane == 0) atomicOr(&sup_s, 1ULL << q);
    }
    // ---- 2. the chunk against itself: thread (q, part) evaluates 8 later candidates
    {
      const int q = tid >> 3, part = tid & 7;
      const float4 cq = cand[q];
      const float aq = cand_a[q];
      unsigned long long bits = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int o = part * 8 + j;
        if (o > q && o < csz && iou_plus1_gt(cq, aq, cand[o], cand_a[o], thresh, t_lo, t_hi)) bits |= 1ULL << o;
      }
      if (bits) atomicOr(&diag[q], bits);
    }
    __syncthreads();
    // ---- 3. warp 0 resolves the chunk in order: every lane tracks the same removed-set `r` and jumps from one
    //         surviving candidate to the next (a kept candidate removes itself and the later ones it overlaps)
    if (warp == 0) {
      const unsigned long long d0 = diag[lane], d1 = diag[lane + 32];
      unsigned long long r = sup_s;
      int cnt = nk;
      while (cnt < post && r != ~0ULL) {
        const int i = __ffsll(static_cast<long long>(~r)) - 1;
        const unsigned long long di_lo = __shfl_sync(0xffffffffu, d0, i & 31);
        const unsigned long long di_hi = __shfl_sync(0xffffffffu, d1, i & 31);
        r |= ((i < 32) ? di_lo : di_hi) | (1ULL << i);
        if (lane == 0) {
          kept_b[cnt] = cand[i];
          kept_a[cnt] = cand_a[i];
          kept_p[cnt] = base + i;
        }
        ++cnt;
      }
      if (lane == 0) nk_s = cnt;
    }
    __syncthreads();
    if (nk_s >= post) break;
  }
  const int cnt = min(nk_s, post);
  for (int i = tid; i < post; i += kGreedyThreads) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    float s = 0.f;
    int a = -1;
    if (i < cnt) {
      const int pos = kept_p[i];
      b = kept_b[i];
      s = sorted_scores[static_cast<long long>(img) * kNmsMaxBoxes + pos];
      a = sorted_anchor[static_cast<long long>(img) * kNmsMaxBoxes + pos];
    }
    out_boxes[static_cast<long long>(img) * post + i] = b;
    out_scores[static_cast<long long>(img) * post + i] = s;
    if (out_anchor) out_anchor[static_cast<long long>(img) * post + i] = a;
  }
  if (tid == 0) out_count[img] = cnt;
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace mega

using namespace mega;

// workspace layout helpers -----------------------------------------------------------------
extern "C" long long mega_nms_workspace_bytes(int n) {
  if (n < 0 || n > kNmsMaxBoxes) return -1;
  const size_t cb = (static_cast<size_t>(n) + 63) / 64;
  size_t b = 0;
  b += align_up(sizeof(float4) * kNmsMaxBoxes, 256);             // sorted boxes
  b += align_up(sizeof(int) * kNmsMaxBoxes, 256);                // order
  b += align_up(sizeof(unsigned long long) * n * (cb ? cb : 1), 256);  // mask
  b += align_up(sizeof(int) * kNmsMaxBoxes, 256);                // kept positions
  b += 256;                                                      // kept count
  return static_cast<long long>(b);
}

extern "C" int mega_nms(const float* boxes, const float* scores, int n, float thresh, void* workspace,
                        long long workspace_bytes, long long* keep_out, int* count_out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(n >= 0, "nms: negative n");
  MEGA_ARG_CHECK(n <= kNmsMaxBoxes, "nms: n=%d exceeds the single-pass capacity %d", n, kNmsMaxBoxes);
  MEGA_ARG_CHECK(count_out != nullptr, "nms: count_out is null");
  if (n == 0) {
    MEGA_CUDA_CHECK(cudaMemsetAsync(count_out, 0, sizeof(int), stream));
    return MEGA_OK;
  }
  MEGA_ARG_CHECK(workspace != nullptr && workspace_bytes >= mega_nms_workspace_bytes(n),
                 "nms: workspace too small (%lld < %lld)", workspace_bytes, mega_nms_workspace_bytes(n));
  const int cb = (n + 63) / 64;
  char* w = static_cast<char*>(workspace);
  float4* sorted_boxes = reinterpret_cast<float4*>(w);
  w += align_up(sizeof(float4) * kNmsMaxBoxes, 256);
  int* order = reinterpret_cast<int*>(w);
  w += align_up(sizeof(int) * kNmsMaxBoxes, 256);
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(w);
  w += align_up(sizeof(unsigned long long) * n * cb, 256);
  int* kept_pos = reinterpret_cast<int*>(w);
  w += align_up(sizeof(int) * kNmsMaxBoxes, 256);
  int* kept_count = reinterpret_cast<int*>(w);

  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(nms_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kNmsMaxBoxes * 8));
    configured = true;
  }
  int np2 = 2;
  while (np2 < n) np2 <<= 1;
  nms_sort_kernel<<<1, kSortThreads, np2 * 8, stream>>>(boxes, scores, n, sorted_boxes, order);
  dim3 grid(cb, cb, 1);
  nms_mask_kernel<<<grid, 64, 0, stream>>>(sorted_boxes, 0, nullptr, n, thresh, mask, 0, cb);
  nms_sweep_kernel<<<1, 128, 0, stream>>>(mask, 0, nullptr, 0, nullptr, n, cb, n, kept_pos, 0, kept_count);
  nms_finalize_kernel<<<1, kSortThreads, 0, stream>>>(kept_pos, kept_count, order, n, keep_out, count_out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" long long mega_rpn_select_workspace_bytes(int n_img, int h, int w, int num_anchors, int pre_nms) {
  if (pre_nms > kNmsMaxBoxes || n_img < 1 || h < 0 || w < 0 || num_anchors < 1) return -1;
  const size_t n = static_cast<size_t>(h) * w * num_anchors;
  const size_t k = pre_nms < static_cast<int>(n) ? pre_nms : n;
  const size_t cb = (k + 63) / 64;
  size_t b = 0;
  b += align_up(sizeof(uint32_t) * n * n_img, 256);
  b += align_up(sizeof(float4) * kNmsMaxBoxes * n_img, 256);
  b += align_up(sizeof(float) * kNmsMaxBoxes * n_img, 256);
  b += align_up(sizeof(int) * kNmsMaxBoxes * n_img, 256);
  b += align_up(static_cast<size_t>(kNmsMaxBoxes) * n_img, 256);
  b += align_up(sizeof(int) * n_img, 256);
  b += align_up(sizeof(unsigned long long) * k * cb * n_img, 256);
  b += align_up(sizeof(int) * kNmsMaxBoxes * n_img, 256);
  b += align_up(sizeof(int) * n_img, 256);
  return static_cast<long long>(b);
}

extern "C" int mega_rpn_select(const float* head, long long head_img_stride, int ld, int n_img, int h, int w,
                               int num_anchors, int stride, const float* base_anchors, float im_w, float im_h,
                               int pre_nms, int post_nms, float nms_thresh, float min_size, void* workspace,
                               long long workspace_bytes, float* out_boxes, float* out_scores, int* out_anchor,
                               int* out_count, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(pre_nms > 0 && pre_nms <= kNmsMaxBoxes, "rpn_select: pre_nms_top_n must be in (0, %d]", kNmsMaxBoxes);
  MEGA_ARG_CHECK(post_nms > 0, "rpn_select: post_nms_top_n must be positive");
  MEGA_ARG_CHECK(n_img >= 1, "rpn_select: n_img=%d, need at least one image", n_img);
  MEGA_ARG_CHECK(h >= 0 && w >= 0 && num_anchors >= 1, "rpn_select: %d x %d cells x %d anchors", h, w, num_anchors);
  MEGA_ARG_CHECK(ld >= 5 * num_anchors, "rpn_select: head row must hold A logits + 4A deltas");
  MEGA_ARG_CHECK(out_boxes != nullptr && out_scores != nullptr && out_count != nullptr, "rpn_select: null output");
  MEGA_ARG_CHECK(reinterpret_cast<uintptr_t>(out_boxes) % 16 == 0, "rpn_select: out_boxes must be 16-byte aligned");
  const long long need = mega_rpn_select_workspace_bytes(n_img, h, w, num_anchors, pre_nms);
  MEGA_ARG_CHECK(workspace != nullptr && workspace_bytes >= need, "rpn_select: workspace too small (%lld < %lld)",
                 workspace_bytes, need);
  const size_t n = static_cast<size_t>(h) * w * num_anchors;
  const int k = pre_nms < static_cast<int>(n) ? pre_nms : static_cast<int>(n);
  const int cb = (k + 63) / 64;
  char* wp = static_cast<char*>(workspace);
  RpnParams p;
  p.head = head;
  p.head_img_stride = head_img_stride;
  p.ld = ld;
  p.A = num_anchors;
  p.H = h;
  p.W = w;
  p.stride = stride;
  p.base_anchors = base_anchors;
  p.im_w = im_w;
  p.im_h = im_h;
  p.pre_nms = pre_nms;
  p.min_size = min_size;
  p.keys = reinterpret_cast<uint32_t*>(wp);
  wp += align_up(sizeof(uint32_t) * n * n_img, 256);
  p.sorted_boxes = reinterpret_cast<float4*>(wp);
  wp += align_up(sizeof(float4) * kNmsMaxBoxes * n_img, 256);
  p.sorted_scores = reinterpret_cast<float*>(wp);
  wp += align_up(sizeof(float) * kNmsMaxBoxes * n_img, 256);
  p.sorted_anchor = reinterpret_cast<int*>(wp);
  wp += align_up(sizeof(int) * kNmsMaxBoxes * n_img, 256);
  p.valid = reinterpret_cast<unsigned char*>(wp);
  wp += align_up(static_cast<size_t>(kNmsMaxBoxes) * n_img, 256);
  p.n_sorted = reinterpret_cast<int*>(wp);
  wp += align_up(sizeof(int) * n_img, 256);
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(wp);
  wp += align_up(sizeof(unsigned long long) * k * cb * n_img, 256);
  int* kept_pos = reinterpret_cast<int*>(wp);
  wp += align_up(sizeof(int) * kNmsMaxBoxes * n_img, 256);
  int* kept_count = reinterpret_cast<int*>(wp);

  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(rpn_topk_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kNmsMaxBoxes * 8));
    configured = true;
  }
  int np2 = 2;
  while (np2 < k) np2 <<= 1;
  rpn_topk_decode_kernel<<<n_img, kSortThreads, np2 * 8, stream>>>(p);
  if (post_nms <= kGreedyMaxKeep) {
    // one-SM greedy NMS (+ output write): overlaps the persistent GEMM chains that own the other SMs
    rpn_nms_greedy_kernel<<<n_img, kGreedyThreads, 0, stream>>>(p.sorted_boxes, p.sorted_scores, p.sorted_anchor, p.valid,
                                                               nullptr, k, nms_thresh, post_nms,
                                                               reinterpret_cast<float4*>(out_boxes), out_scores,
                                                               out_anchor, out_count);
  } else {
    if (k > 0) {
      dim3 grid(cb, cb, n_img);
      nms_mask_kernel<<<grid, 64, 0, stream>>>(p.sorted_boxes, kNmsMaxBoxes, nullptr, k, nms_thresh, mask,
                                               static_cast<long long>(k) * cb, cb);
      nms_sweep_kernel<<<n_img, 128, 0, stream>>>(mask, static_cast<long long>(k) * cb, p.valid, kNmsMaxBoxes, nullptr,
                                                  k, cb, post_nms, kept_pos, kNmsMaxBoxes, kept_count);
    } else {   // an empty map: nothing kept, rpn_write_kernel zero-fills the outputs as the greedy kernel does
      MEGA_CUDA_CHECK(cudaMemsetAsync(kept_count, 0, sizeof(int) * n_img, stream));
    }
    rpn_write_kernel<<<n_img, 256, 0, stream>>>(p.sorted_boxes, p.sorted_scores, p.sorted_anchor, kept_pos, kNmsMaxBoxes,
                                                kept_count, post_nms, reinterpret_cast<float4*>(out_boxes), out_scores,
                                                out_anchor, out_count);
  }
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
