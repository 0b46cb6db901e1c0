// Proposal recall of a whole dataset (mega_proposal_recall, include/mega_b200.h): the per-image body of the reference's
// eval_proposals_vid (data/datasets/evaluation/vid/vid_eval.py:72-119).
//
// Per image, in one CTA:
//   1. sort the proposals by objectness, descending, in shared memory, with the algorithm torch's CPU
//      sort(descending=True) runs (libstdc++'s std::sort, not stable: equal scores end in its order, which the
//      proposals' order among tied entries and so the greedy rounds' tie rules depend on), keep the first `limit`;
//   2. the P' x G IoU matrix with boxlist_iou's "+1" arithmetic in its operation order (structures/boxlist_ops.py:53-90),
//      every fp32 operation separately rounded; column-major (element g * P' + r), in shared memory when it fits, else
//      in the CTA's slot of the global workspace;
//   3. min(P', G) greedy rounds: the largest entry (ties: lowest GT index, then lowest proposal index -- the order of
//      torch's overlaps.max(dim=0) followed by max_overlaps.max(dim=0)) is the round's overlap; its row and column
//      become -1. Entries past min(P', G) are 0;
//   4. hits (overlaps >= iou_thresh) and num_pos (sum of G) as integers, so the result does not depend on scheduling.
// Images without GT or without proposals add their GT to num_pos and nothing else, as in the reference.
//
// Same __host__ __device__ arrangement as seq_nms.cuh: the body is written against a `Lanes` policy (on the device the
// CTA's threads with __syncthreads and a block arg-max, on the host a single lane whose reductions are no-ops), and g++
// compiles it for the CPU suite (tests/native/proposal_recall_host.cpp). Loop bounds and branches depend only on values
// every lane holds, so no lane skips a barrier.
#pragma once
#include <stdint.h>
#include <string.h>

#include "iou.cuh"

#if defined(__CUDACC__)
#define MEGA_PR_HD __host__ __device__ __forceinline__
#else
#define MEGA_PR_HD static inline
#endif

namespace mega_pr {

constexpr int kMaxProps = 8192;             // proposals per image: capacity of the shared-memory sort (64 KB)
constexpr int kSmemMatrixBytes = 32768;     // IoU matrices up to this size stay in shared memory
constexpr int kThreads = 256;
constexpr int kMaxCtas = 1024;              // CTAs of a launch; each walks images blockIdx.x, + gridDim.x, ...

struct PrArgs {
  const float4* prop_boxes;       // [sum P] xyxy
  const float* prop_scores;       // [sum P] objectness
  const long long* prop_off;      // [N + 1]
  const float4* gt_boxes;         // [sum G] xyxy
  const long long* gt_off;        // [N + 1]
  int num_images, max_props, max_gt, limit;
  float thresh;
  int smem_matrix_floats;         // capacity of the shared-memory matrix
  float* gmatrix;                 // [grid][slot_floats] or null
  long long slot_floats;
  float* gt_overlaps;             // [sum G]
};

struct PrCounts {
  unsigned long long hits, num_pos, rejected;
};

struct PrLayout {
  long long keys_bytes, smem_matrix_bytes, slot_bytes, workspace_bytes;
  int grid;
};

MEGA_PR_HD long long pr_align(long long x) { return (x + 255) & ~255LL; }

// launch geometry and memory of one call; false for arguments out of range
MEGA_PR_HD bool pr_layout(int num_images, int max_props, int max_gt, int limit, PrLayout* out) {
  if (num_images < 0 || max_props < 0 || max_props > kMaxProps || max_gt < 0 || limit < 0) return false;
  const long long pk = max_props < limit ? max_props : limit;
  if (pk * max_gt > 0x7fffffffLL) return false;
  const long long matrix = pk * max_gt * 4;
  out->keys_bytes = 8LL * (max_props > 1 ? max_props : 1);
  out->grid = num_images < kMaxCtas ? num_images : kMaxCtas;
  if (matrix <= kSmemMatrixBytes) {
    out->smem_matrix_bytes = matrix;
    out->slot_bytes = 0;
    out->workspace_bytes = 0;
  } else {
    out->smem_matrix_bytes = kSmemMatrixBytes;
    out->slot_bytes = pr_align(matrix);
    out->workspace_bytes = out->slot_bytes * out->grid;
  }
  return true;
}

// One proposal in the sort: objectness and input index.
struct PrItem {
  float s;
  int i;
};

// the comparator torch's CPU sort(descending=True) hands to std::sort: larger first, NaN largest
MEGA_PR_HD bool pr_before(const PrItem& l, const PrItem& r) { return (!(l.s != l.s) && r.s != r.s) || l.s > r.s; }

MEGA_PR_HD void pr_swap(PrItem* a, PrItem* b) {
  const PrItem t = *a;
  *a = *b;
  *b = t;
}

MEGA_PR_HD void pr_unguarded_linear_insert(PrItem* last) {
  const PrItem val = *last;
  PrItem* next = last - 1;
  while (pr_before(val, *next)) {
    *last = *next;
    last = next;
    --next;
  }
  *last = val;
}

MEGA_PR_HD void pr_insertion_sort(PrItem* first, PrItem* last) {
  if (first == last) return;
  for (PrItem* i = first + 1; i != last; ++i) {
    if (pr_before(*i, *first)) {
      const PrItem val = *i;
      for (PrItem* j = i; j != first; --j) *j = *(j - 1);
      *first = val;
    } else {
      pr_unguarded_linear_insert(i);
    }
  }
}

MEGA_PR_HD void pr_adjust_heap(PrItem* first, long long hole, long long len, PrItem value) {
  const long long top = hole;
  long long child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (pr_before(first[child], first[child - 1])) child--;
    first[hole] = first[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    first[hole] = first[child - 1];
    hole = child - 1;
  }
  long long parent = (hole - 1) / 2;
  while (hole > top && pr_before(first[parent], value)) {
    first[hole] = first[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  first[hole] = value;
}

// std::partial_sort(first, last, last): make_heap, then sort_heap (the introsort's fallback past its depth limit)
MEGA_PR_HD void pr_heap_sort(PrItem* first, PrItem* last) {
  const long long len = last - first;
  if (len >= 2) {
    for (long long parent = (len - 2) / 2;; --parent) {
      pr_adjust_heap(first, parent, len, first[parent]);
      if (parent == 0) break;
    }
  }
  while (last - first > 1) {
    --last;
    const PrItem value = *last;
    *last = *first;
    pr_adjust_heap(first, 0, last - first, value);
  }
}

// libstdc++'s std::sort (introsort: median-of-three quicksort down to runs of 16, heap sort past 2 * floor(log2 n)
// levels, then a final insertion sort), step for step, so that equal objectness values end in the order torch's CPU
// sort gives them -- which is not the input order. The recursion on the right part runs from an explicit stack;
// the parts are disjoint, so the processing order does not change the result. Serial: one lane runs it.
MEGA_PR_HD void pr_torch_sort(PrItem* first, int n) {
  if (n <= 1) return;
  int lg = 0;
  while ((2LL << lg) <= n) ++lg;
  struct Part {
    int lo, hi, depth;
  } stack[64];
  int top = 0;
  stack[top++] = {0, n, 2 * lg};
  while (top > 0) {
    const Part part = stack[--top];
    int lo = part.lo, hi = part.hi, depth = part.depth;
    while (hi - lo > 16) {
      if (depth == 0) {
        pr_heap_sort(first + lo, first + hi);
        break;
      }
      --depth;
      // __move_median_to_first(first, first + 1, mid, last - 1)
      PrItem *f = first + lo, *a = f + 1, *b = f + (hi - lo) / 2, *c = first + hi - 1;
      if (pr_before(*a, *b)) {
        if (pr_before(*b, *c)) pr_swap(f, b);
        else if (pr_before(*a, *c)) pr_swap(f, c);
        else pr_swap(f, a);
      } else if (pr_before(*a, *c)) {
        pr_swap(f, a);
      } else if (pr_before(*b, *c)) {
        pr_swap(f, c);
      } else {
        pr_swap(f, b);
      }
      // __unguarded_partition(first + 1, last, first)
      PrItem *l = f + 1, *r = first + hi;
      while (true) {
        while (pr_before(*l, *f)) ++l;
        --r;
        while (pr_before(*f, *r)) --r;
        if (!(l < r)) break;
        pr_swap(l, r);
        ++l;
      }
      const int cut = static_cast<int>(l - first);
      stack[top++] = {cut, hi, depth};
      hi = cut;
    }
  }
  if (n > 16) {
    pr_insertion_sort(first, first + 16);
    for (PrItem* i = first + 16; i != first + n; ++i) pr_unguarded_linear_insert(i);
  } else {
    pr_insertion_sort(first, first + n);
  }
}

// boxlist_iou(proposal, gt): inter / (area_p + area_g - inter), "+1" widths clamped at 0
MEGA_PR_HD float pr_iou(const float4 p, const float4 g) {
  const float ap = mega::box_area_plus1(p), ag = mega::box_area_plus1(g);
  const float left = fmaxf(p.x, g.x), top = fmaxf(p.y, g.y);
  const float right = fminf(p.z, g.z), bottom = fminf(p.w, g.w);
  const float w = fmaxf(MEGA_IOU_ADD(MEGA_IOU_SUB(right, left), 1.f), 0.f);
  const float h = fmaxf(MEGA_IOU_ADD(MEGA_IOU_SUB(bottom, top), 1.f), 0.f);
  const float inter = MEGA_IOU_MUL(w, h);
  return MEGA_IOU_DIV(inter, MEGA_IOU_SUB(MEGA_IOU_ADD(ap, ag), inter));
}

// (v, key) beats (bv, bkey): larger value, ties to the smaller key (= g * P' + r: lower GT, then lower proposal)
MEGA_PR_HD bool pr_better(float v, unsigned key, float bv, unsigned bkey) {
  return v > bv || (v == bv && key < bkey);
}

// one image; `keys` holds max_props entries, `smat` smem_matrix_floats, `gslot` slot_floats (or null).
// Only lane 0 updates `c`.
template <class Lanes>
MEGA_PR_HD void pr_image(const PrArgs& a, const Lanes& L, int img, PrItem* keys, float* smat, float* gslot,
                         PrCounts& c) {
  const long long p0 = a.prop_off[img], g0 = a.gt_off[img];
  const long long np = a.prop_off[img + 1] - p0, ng = a.gt_off[img + 1] - g0;
  const int lane = L.lane(), nl = L.count();
  if (lane == 0) c.num_pos += static_cast<unsigned long long>(ng);
  const bool rejected = np < 0 || np > a.max_props || ng < 0 || ng > a.max_gt;
  const int P = static_cast<int>(np), G = static_cast<int>(ng);
  const int pk = P < a.limit ? P : a.limit;
  if (rejected || pk == 0 || G == 0) {
    for (int j = lane; j < G; j += nl) a.gt_overlaps[g0 + j] = 0.f;
    if (lane == 0 && rejected) c.rejected += 1;
    return;
  }
  // 1. order
  L.sync();                      // the previous image of this CTA is done with the shared memory
  for (int i = lane; i < P; i += nl) keys[i] = {a.prop_scores[p0 + i], i};
  L.sync();
  if (lane == 0) pr_torch_sort(keys, P);
  L.sync();
  // 2. IoU matrix, column-major
  const int cells = pk * G;
  float* m = cells <= a.smem_matrix_floats ? smat : gslot;
  for (int i = lane; i < cells; i += nl) {
    const int g = i / pk, r = i - g * pk;
    m[i] = pr_iou(a.prop_boxes[p0 + keys[r].i], a.gt_boxes[g0 + g]);
  }
  L.sync();
  // 3. greedy rounds
  const int rounds = pk < G ? pk : G;
  unsigned long long hits = 0;
  for (int round = 0; round < rounds; ++round) {
    float bv = -2.f;
    unsigned bk = 0xffffffffu;
    for (int i = lane; i < cells; i += nl) {
      const float v = m[i];
      if (pr_better(v, static_cast<unsigned>(i), bv, bk)) {
        bv = v;
        bk = static_cast<unsigned>(i);
      }
    }
    L.argmax(bv, bk);
    const int g = static_cast<int>(bk / static_cast<unsigned>(pk)), r = static_cast<int>(bk % static_cast<unsigned>(pk));
    if (lane == 0) {
      a.gt_overlaps[g0 + round] = bv;
      hits += bv >= a.thresh ? 1 : 0;
    }
    for (int j = lane; j < G; j += nl) m[j * pk + r] = -1.f;
    for (int j = lane; j < pk; j += nl) m[g * pk + j] = -1.f;
    L.sync();
  }
  for (int j = rounds + lane; j < G; j += nl) a.gt_overlaps[g0 + j] = 0.f;
  if (lane == 0) c.hits += hits + (0.f >= a.thresh ? static_cast<unsigned long long>(G - rounds) : 0ULL);
}

}  // namespace mega_pr
