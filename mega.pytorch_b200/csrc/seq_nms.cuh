// Seq-NMS over whole videos (Han et al., "Seq-NMS for Video Object Detection", arXiv:1602.08465): per (video, class),
// repeatedly pick the highest-scoring chain of linked boxes through consecutive frames, rescore it, suppress what
// overlaps it frame by frame, until no box of the class is left. The contract (include/mega_b200.h, mega_seq_nms) is
// restated in NumPy by tests/seq_nms_oracle.py; the result is deterministic, so kernels and oracle agree bit for bit.
//
// Same __host__ __device__ arrangement as train_ops.cuh: seq_nms.cu runs these bodies in three kernels, and g++ compiles
// the very same code (tests/native/seq_nms_host.cpp) for the CPU suite. The per-(video, class) loop is written
// against a `Lanes` policy: on the device a warp (32 lanes, shuffles, __syncwarp), on the host a single lane whose
// reductions are no-ops. Loop bounds and branches depend only on values every lane holds, so a warp never diverges
// around a reduction.
//
// Storage is indexed by the detection's slot (frame f, position k in the frame's padded row), so nothing is packed:
//   ranges [F, C]     : [lo, hi) of class c in frame f (labels of a frame are ascending: class-major order)
//   links  [F, D, W]  : bit j of word w set iff slot 64w+j of frame f+1 has the same class and IoU > link threshold
//   best   [F, D]     : fp64 DP value of an alive box; -inf once the box is selected or suppressed
//   succ   [F, D]     : slot of the successor in frame f+1 on the best chain, -1 for none
//   fmax   [F, C]     : per (frame, class) the largest best and its slot (ties: smallest slot)
//   bmax   [F, C]     : per (video, class) and block of 32 frames, stored at the block's first frame: the largest fmax
//                       and its frame (ties: smallest frame) -- the root search reads T / 32 values, not T
#pragma once
#include <math.h>
#include <stdint.h>

#include "iou.cuh"

#if defined(__CUDACC__)
#define MEGA_SEQ_HD __host__ __device__ __forceinline__
#else
#define MEGA_SEQ_HD static inline
#endif
#if defined(__CUDA_ARCH__)
#define MEGA_SEQ_CTZ(x) (__ffsll(static_cast<long long>(x)) - 1)
#define MEGA_SEQ_D2F(x) __double2float_rn(x)
#else
#define MEGA_SEQ_CTZ(x) __builtin_ctzll(x)
#define MEGA_SEQ_D2F(x) static_cast<float>(x)
#endif

namespace mega_seq {

constexpr int kMaxDet = 512;        // detections per frame (the engines return at most 300)
constexpr int kFrameBlock = 32;     // frames per root-search block

struct Range {
  int lo, hi;
};

struct SeqArgs {
  const float4* boxes;           // [F, D] xyxy
  const float* scores;           // [F, D]
  const int* labels;             // [F, D], ascending inside a frame's first counts[f] slots
  const int* counts;             // [F]
  const int* video_offsets;      // [V + 1]
  int num_frames, max_det, words, num_classes;
  float link_thresh, link_lo, link_hi, nms_thresh, nms_lo, nms_hi;
  int rescore_max;               // 0: average of the chain, 1: its maximum
  Range* ranges;
  unsigned long long* links;
  double* best;
  int* succ;
  double* fmax_val;
  int* fmax_idx;
  double* bmax_val;
  int* bmax_frame;
  float* out_scores;             // [F, D]
  unsigned char* keep;           // [F, D]
};

MEGA_SEQ_HD long long seq_align(long long x) { return (x + 255) & ~255LL; }

// Workspace layout; with base != nullptr it also points a's scratch arrays into it. Returns the byte count.
MEGA_SEQ_HD long long seq_workspace_layout(int num_frames, int max_det, int num_classes, char* base, SeqArgs* a) {
  const long long f = num_frames, d = max_det, c = num_classes, w = (max_det + 63) / 64;
  long long off = 0;
  const long long o_ranges = off;
  off += seq_align(f * c * static_cast<long long>(sizeof(Range)));
  const long long o_links = off;
  off += seq_align(f * d * w * 8);
  const long long o_best = off;
  off += seq_align(f * d * 8);
  const long long o_succ = off;
  off += seq_align(f * d * 4);
  const long long o_fv = off;
  off += seq_align(f * c * 8);
  const long long o_fi = off;
  off += seq_align(f * c * 4);
  const long long o_bv = off;
  off += seq_align(f * c * 8);
  const long long o_bf = off;
  off += seq_align(f * c * 4);
  if (base != nullptr) {
    a->words = static_cast<int>(w);
    a->ranges = reinterpret_cast<Range*>(base + o_ranges);
    a->links = reinterpret_cast<unsigned long long*>(base + o_links);
    a->best = reinterpret_cast<double*>(base + o_best);
    a->succ = reinterpret_cast<int*>(base + o_succ);
    a->fmax_val = reinterpret_cast<double*>(base + o_fv);
    a->fmax_idx = reinterpret_cast<int*>(base + o_fi);
    a->bmax_val = reinterpret_cast<double*>(base + o_bv);
    a->bmax_frame = reinterpret_cast<int*>(base + o_bf);
  }
  return off;
}

// the division-free band of iou_plus1_gt (iou.cuh), as postprocess.cu computes it
MEGA_SEQ_HD void seq_band(float t, float* lo, float* hi) {
  *lo = MEGA_IOU_MUL(t, 1.f - 9.5367431640625e-07f);
  *hi = MEGA_IOU_MUL(t, 1.f + 9.5367431640625e-07f);
}

// the arguments of mega_seq_nms as the bodies below read them (host code)
inline SeqArgs seq_make_args(const float* boxes, const float* scores, const int* labels, const int* counts,
                             int num_frames, int max_det, const int* video_offsets, int num_classes, float link_iou,
                             float nms_iou, int rescore, void* workspace, float* out_scores, unsigned char* keep) {
  SeqArgs a;
  a.boxes = reinterpret_cast<const float4*>(boxes);
  a.scores = scores;
  a.labels = labels;
  a.counts = counts;
  a.video_offsets = video_offsets;
  a.num_frames = num_frames;
  a.max_det = max_det;
  a.num_classes = num_classes;
  a.link_thresh = link_iou;
  a.nms_thresh = nms_iou;
  seq_band(link_iou, &a.link_lo, &a.link_hi);
  seq_band(nms_iou, &a.nms_lo, &a.nms_hi);
  a.rescore_max = rescore;
  a.out_scores = out_scores;
  a.keep = keep;
  seq_workspace_layout(num_frames, max_det, num_classes, static_cast<char*>(workspace), &a);
  return a;
}

MEGA_SEQ_HD int seq_lower_bound(const int* v, int n, int x) {
  int lo = 0;
  while (n > 0) {
    const int h = n >> 1;
    if (v[lo + h] < x) {
      lo += h + 1;
      n -= h + 1;
    } else {
      n = h;
    }
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------------- bucket
// item = f * C + c: the slot range of class c in frame f
MEGA_SEQ_HD void seq_bucket_item(const SeqArgs& a, long long item) {
  const long long f = item / a.num_classes;
  const int c = static_cast<int>(item - f * a.num_classes);
  const int* lab = a.labels + f * a.max_det;
  const int n = a.counts[f];
  const int lo = seq_lower_bound(lab, n, c);
  Range r;
  r.lo = lo;
  r.hi = lo + seq_lower_bound(lab + lo, n - lo, c + 1);
  a.ranges[item] = r;
}

// -------------------------------------------------------------------------------------------------------- links
// item = (f * D + k) * W + w: word w of the link mask of slot k of frame f over frame f + 1. Also resets the slot's
// state (word 0). The links of a video's last frame point into the next video and are never read.
MEGA_SEQ_HD void seq_link_item(const SeqArgs& a, long long item) {
  const long long slot = item / a.words;
  const int w = static_cast<int>(item - slot * a.words);
  const long long f = slot / a.max_det;
  const int k = static_cast<int>(slot - f * a.max_det);
  if (w == 0) {
    a.best[slot] = 0.0;
    a.keep[slot] = 0;
    a.out_scores[slot] = 0.f;
  }
  unsigned long long bits = 0;
  const int c = a.labels[slot];
  if (k < a.counts[f] && f + 1 < a.num_frames && c >= 0 && c < a.num_classes) {
    const Range r = a.ranges[(f + 1) * a.num_classes + c];
    const int j0 = r.lo > 64 * w ? r.lo : 64 * w;
    const int j1 = r.hi < 64 * w + 64 ? r.hi : 64 * w + 64;
    const float4 bi = a.boxes[slot];
    const float si = mega::box_area_plus1(bi);
    const float4* next = a.boxes + (f + 1) * a.max_det;
    for (int j = j0; j < j1; ++j) {
      const float4 bj = next[j];
      if (mega::iou_plus1_gt(bi, si, bj, mega::box_area_plus1(bj), a.link_thresh, a.link_lo, a.link_hi))
        bits |= 1ULL << (j - 64 * w);
    }
  }
  a.links[item] = bits;
}

// ------------------------------------------------------------------------------------------- per (video, class)
// (v, key) beats (v2, key2): larger value, ties to the smaller key
MEGA_SEQ_HD bool seq_better(double v, int key, double v2, int key2) { return v > v2 || (v == v2 && key < key2); }

// DP step of frame f: best / succ of every alive class-c box from the values of frame f + 1 (has_next), and fmax of
// frame f. Returns (on every lane) whether an alive box's value changed.
template <class Lanes>
MEGA_SEQ_HD bool seq_frame_dp(const SeqArgs& a, const Lanes& L, long long f, int c, bool has_next) {
  const long long C = a.num_classes, D = a.max_det;
  const Range r = a.ranges[f * C + c];
  Range rn;
  rn.lo = rn.hi = 0;
  if (has_next) rn = a.ranges[(f + 1) * C + c];
  const double* best_next = a.best + (f + 1) * D;
  double mv = -INFINITY;
  int mi = 0x7fffffff;
  bool changed = false;
  for (int k = r.lo + L.lane(); k < r.hi; k += L.count()) {
    const long long slot = f * D + k;
    const double old = a.best[slot];
    if (old == -INFINITY) continue;
    double m = -INFINITY;
    int arg = -1;
    for (int w = rn.lo >> 6; rn.hi > rn.lo && w <= (rn.hi - 1) >> 6; ++w) {
      unsigned long long bits = a.links[slot * a.words + w];
      while (bits) {
        const int j = 64 * w + MEGA_SEQ_CTZ(bits);
        bits &= bits - 1;
        const double v = best_next[j];
        if (v > m) {   // ascending j: ties keep the smallest; dead successors (-inf) never win
          m = v;
          arg = j;
        }
      }
    }
    const double nb = static_cast<double>(a.scores[slot]) + (arg < 0 ? 0.0 : m);
    a.succ[slot] = arg;
    changed |= nb != old;
    a.best[slot] = nb;
    if (nb > mv) {
      mv = nb;
      mi = k;
    }
  }
  L.argmax(mv, mi);
  if (L.lane() == 0) {
    a.fmax_val[f * C + c] = mv;
    a.fmax_idx[f * C + c] = mi;
  }
  return L.any(changed);
}

template <class Lanes>
MEGA_SEQ_HD void seq_block_max(const SeqArgs& a, const Lanes& L, int f0, int f1, int blk, int c) {
  const long long C = a.num_classes;
  const int t0 = f0 + kFrameBlock * blk;
  const int t1 = t0 + kFrameBlock < f1 ? t0 + kFrameBlock : f1;
  double v = -INFINITY;
  int fr = 0x7fffffff;
  for (int t = t0 + L.lane(); t < t1; t += L.count()) {
    const double x = a.fmax_val[t * C + c];
    if (x > v) {
      v = x;
      fr = t;
    }
  }
  L.argmax(v, fr);
  if (L.lane() == 0) {
    a.bmax_val[t0 * C + c] = v;
    a.bmax_frame[t0 * C + c] = fr;
  }
}

// Seq-NMS of class c in video v (frames [f0, f1)): initial backward DP, then per iteration
//   root = alive box with the largest best (ties: smallest frame, then smallest slot), chain = root + successors;
//   rescore the chain, mark it selected, suppress the alive boxes overlapping it frame by frame;
//   recompute the DP from the chain's last frame b downward: frames >= a unconditionally (boxes died there), below a
//   only while the frame above changed -- best[t] depends on frames >= t only, so the first unchanged frame below a
//   ends the update.
template <class Lanes>
MEGA_SEQ_HD void seq_video_class(const SeqArgs& a, const Lanes& L, int v, int c) {
  const long long C = a.num_classes, D = a.max_det;
  const int f0 = a.video_offsets[v], f1 = a.video_offsets[v + 1];
  if (f1 <= f0) return;
  const int nblk = (f1 - f0 + kFrameBlock - 1) / kFrameBlock;
  for (int t = f1 - 1; t >= f0; --t) {
    seq_frame_dp(a, L, t, c, t + 1 < f1);
    L.sync();
  }
  for (int blk = 0; blk < nblk; ++blk) seq_block_max(a, L, f0, f1, blk, c);
  L.sync();
  for (;;) {
    double rv = -INFINITY;
    int rf = 0x7fffffff;
    for (int blk = L.lane(); blk < nblk; blk += L.count()) {
      const long long at = static_cast<long long>(f0 + kFrameBlock * blk) * C + c;
      const double x = a.bmax_val[at];
      if (x > rv) {
        rv = x;
        rf = a.bmax_frame[at];
      }
    }
    L.argmax(rv, rf);
    if (rv == -INFINITY) break;
    const int ta = rf;
    const int ka = a.fmax_idx[ta * C + c];
    // every iteration removes the alive root, so the loop ends; should stale maxima ever name a removed box, stop
    // (a wrong result the tests see) instead of selecting it forever
    if (a.best[ta * D + ka] == -INFINITY) break;
    // chain length and maximum score
    int len = 0, tb = ta;
    float smax = -INFINITY;
    for (int t = ta, k = ka;; ++t) {
      const long long slot = t * D + k;
      const float s = a.scores[slot];
      smax = s > smax ? s : smax;
      ++len;
      tb = t;
      k = a.succ[slot];
      if (k < 0) break;
    }
    const float score = a.rescore_max ? smax : MEGA_SEQ_D2F(rv / static_cast<double>(len));
    // select and suppress, frame by frame (a frame's suppression only involves that frame's chain box)
    for (int t = ta, k = ka;; ++t) {
      const long long slot = t * D + k;
      const Range r = a.ranges[t * C + c];
      const float4 bs = a.boxes[slot];
      const float ss = mega::box_area_plus1(bs);
      for (int j = r.lo + L.lane(); j < r.hi; j += L.count()) {
        const long long sj = t * D + j;
        if (j == k || a.best[sj] == -INFINITY) continue;
        const float4 bj = a.boxes[sj];
        if (mega::iou_plus1_gt(bj, mega::box_area_plus1(bj), bs, ss, a.nms_thresh, a.nms_lo, a.nms_hi))
          a.best[sj] = -INFINITY;
      }
      const int next = a.succ[slot];
      if (L.lane() == 0) {
        a.best[slot] = -INFINITY;
        a.keep[slot] = 1;
        a.out_scores[slot] = score;
      }
      if (next < 0) break;
      k = next;
    }
    L.sync();
    int lo = tb;
    for (int t = tb; t >= f0; --t) {
      const bool changed = seq_frame_dp(a, L, t, c, t + 1 < f1);
      L.sync();
      lo = t;
      if (t < ta && !changed) break;
    }
    for (int blk = (lo - f0) / kFrameBlock; blk <= (tb - f0) / kFrameBlock; ++blk) seq_block_max(a, L, f0, f1, blk, c);
    L.sync();
  }
}

}  // namespace mega_seq
