// Detection AP of ImageNet VID (mega_vid_eval / mega_vid_match_host, include/mega_b200.h): the bodies of the reference's
// calc_detection_vid_prec_rec and calc_detection_vid_ap (data/datasets/evaluation/vid/vid_eval.py:156-343).
//
//   ve_match      greedy matching of one (image, class): detections in score order against the class's GT boxes,
//                 fp32 "+1" IoUs computed once and shared by all motion ranges; per range a match flag and the
//                 detection's ignore weight (0, 1, empty_weight or n_ignored / num_gt in fp64);
//   ve_fp_weight  the weight a detection adds to the false-positive sum (`fps` of vid_eval.py:271-276);
//   ve_cumsum     the cumulative tp (integer) and fp (fp64, strictly left to right: np.cumsum is sequential) of one
//                 (class, range) list in its global score order;
//   ve_prec_rec   prec = tp / (fp + tp + eps), rec = tp / n_pos, evaluated left to right as numpy does;
//   ve_steps      the right-to-left precision envelope and the points where recall changes, compacted to
//                 (mrec[i+1] - mrec[i], mpre[i+1], mrec[i+1]); the caller's np.sum of the products is the AP.
//
// Same __host__ __device__ arrangement as seq_nms.cuh and proposal_recall.cuh: g++ compiles these bodies for the CPU
// suite (tests/native/vid_eval_host.cpp) and for mega_vid_match_host, nvcc for the kernels of vid_eval.cu. Every fp
// operation is a separately rounded IEEE operation on both (explicit _rn intrinsics on the device, -ffp-contract=off
// on the host).
#pragma once
#include <stdint.h>
#include <string.h>

#include "iou.cuh"

#if defined(__CUDACC__)
#define MEGA_VE_HD __host__ __device__ __forceinline__
#else
#define MEGA_VE_HD static inline
#endif
#if defined(__CUDA_ARCH__)
#define MEGA_VE_DADD(a, b) __dadd_rn((a), (b))
#define MEGA_VE_DSUB(a, b) __dsub_rn((a), (b))
#define MEGA_VE_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define MEGA_VE_DADD(a, b) ((a) + (b))
#define MEGA_VE_DSUB(a, b) ((a) - (b))
#define MEGA_VE_DDIV(a, b) ((a) / (b))
#endif

namespace mega_ve {

constexpr int kMaxRanges = 8;         // motion ranges of one call
constexpr double kEps = 2.220446049250313e-16;   // np.spacing(1)

// One range: GT with motion IoU m is ignored iff m < lo or m > hi (a NaN motion -- the GT has no motion entry, or the
// evaluation has no motion list -- is never ignored); empty_weight is the ignore weight of detections of a class
// without GT in the image (already 0 where the reference's fraction is 1).
struct VeRange {
  double lo, hi, empty_weight;
};

MEGA_VE_HD bool ve_ignored(double m, const VeRange& r) { return m < r.lo || m > r.hi; }

// Ordering key of a score: descending score <=> ascending key; NaN first (numpy's argsort puts NaN last, [::-1] first),
// -0 and +0 equal.
MEGA_VE_HD uint32_t ve_desc_key(float s) {
  if (s != s) return 0u;                       // NaN: ahead of +inf, whose key is 0x007fffff
  uint32_t b;
  memcpy(&b, &s, 4);
  if (s == 0.f) b = 0u;                        // -0 -> +0
  const uint32_t asc = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return ~asc;
}

// Greedy matching of one image's detections of one class (vid_eval.py:201-262, integer-typed "+1" boxes).
// `S` provides
//   int n_pred() / n_gt_all()         detections of the class in match order, GT boxes of the image (any class);
//   float4 pred(j) / float4 gt(k)     xyxy boxes;
//   bool in_class(k)                  GT k belongs to the class (GT keep their order: gb[gsel]);
//   bool ignored(k, r)                GT k is ignored under range r;
//   double empty_weight(r);
//   unsigned char* selec(r)           n_gt_all() bytes of scratch per range (only the class's entries are used);
//   void put(j, r, signed char match, double weight).
#if defined(__CUDACC__)
#pragma nv_exec_check_disable   // S is host-only for mega_vid_match_host, device-only in the kernel
#endif
template <class S>
MEGA_VE_HD void ve_match(const S& s, int nr, float iou_thresh) {
  const int np = s.n_pred(), ng = s.n_gt_all();
  if (np == 0) return;
  int num_gt = 0, n_ignored[kMaxRanges];
  for (int r = 0; r < nr; ++r) n_ignored[r] = 0;
  for (int k = 0; k < ng; ++k) {
    if (!s.in_class(k)) continue;
    ++num_gt;
    for (int r = 0; r < nr; ++r) n_ignored[r] += s.ignored(k, r) ? 1 : 0;
  }
  if (num_gt == 0) {                                   // vid_eval.py:207-210
    for (int j = 0; j < np; ++j)
      for (int r = 0; r < nr; ++r) s.put(j, r, 0, s.empty_weight(r));
    return;
  }
  for (int r = 0; r < nr; ++r) {   // only the class's own entries: other classes of the image may be matching meanwhile
    unsigned char* sel = s.selec(r);
    for (int k = 0; k < ng; ++k)
      if (s.in_class(k)) sel[k] = 0;
  }
  for (int j = 0; j < np; ++j) {
    const float4 p = s.pred(j);
    const float px1 = p.x, py1 = p.y;
    const float px2 = MEGA_IOU_ADD(p.z, 1.0f), py2 = MEGA_IOU_ADD(p.w, 1.0f);
    const float parea = MEGA_IOU_MUL(MEGA_IOU_ADD(MEGA_IOU_SUB(px2, px1), 1.0f),
                                     MEGA_IOU_ADD(MEGA_IOU_SUB(py2, py1), 1.0f));
    double iou_match[kMaxRanges], iou_ig[kMaxRanges], iou_nig[kMaxRanges];
    int arg[kMaxRanges];
    for (int r = 0; r < nr; ++r) iou_match[r] = iou_thresh, iou_ig[r] = -1.0, iou_nig[r] = -1.0, arg[r] = -1;
    for (int k = 0; k < ng; ++k) {
      if (!s.in_class(k)) continue;
      const float4 g = s.gt(k);
      const float gx1 = g.x, gy1 = g.y, gx2 = MEGA_IOU_ADD(g.z, 1.0f), gy2 = MEGA_IOU_ADD(g.w, 1.0f);
      const float garea = MEGA_IOU_MUL(MEGA_IOU_ADD(MEGA_IOU_SUB(gx2, gx1), 1.0f),
                                       MEGA_IOU_ADD(MEGA_IOU_SUB(gy2, gy1), 1.0f));
      const float ltx = px1 > gx1 ? px1 : gx1, lty = py1 > gy1 ? py1 : gy1;
      const float rbx = px2 < gx2 ? px2 : gx2, rby = py2 < gy2 ? py2 : gy2;
      float w = MEGA_IOU_ADD(MEGA_IOU_SUB(rbx, ltx), 1.0f), h = MEGA_IOU_ADD(MEGA_IOU_SUB(rby, lty), 1.0f);
      w = w < 0.f ? 0.f : w;
      h = h < 0.f ? 0.f : h;
      const float inter = MEGA_IOU_MUL(w, h);
      const double v = MEGA_IOU_DIV(inter, MEGA_IOU_SUB(MEGA_IOU_ADD(parea, garea), inter));
      for (int r = 0; r < nr; ++r) {
        const bool ig = s.ignored(k, r);
        if (ig && v > iou_ig[r]) iou_ig[r] = v;
        if (!ig && v > iou_nig[r]) iou_nig[r] = v;
        if (s.selec(r)[k] || v < iou_match[r]) continue;
        if (v == iou_match[r]) {
          if (arg[r] < 0 || s.ignored(arg[r], r)) arg[r] = k;
        } else {
          arg[r] = k;
        }
        iou_match[r] = v;
      }
    }
    for (int r = 0; r < nr; ++r) {
      if (arg[r] >= 0) {
        s.put(j, r, 1, s.ignored(arg[r], r) ? 1.0 : 0.0);
        s.selec(r)[arg[r]] = 1;
      } else if (iou_nig[r] > iou_ig[r]) {
        s.put(j, r, 0, 0.0);
      } else if (iou_ig[r] > iou_nig[r]) {
        s.put(j, r, 0, 1.0);
      } else {
        s.put(j, r, 0, MEGA_VE_DDIV(static_cast<double>(n_ignored[r]), static_cast<double>(num_gt)));
      }
    }
  }
}

// fps of one detection: ((match == 0) & (ign != 1)) * where(ign == 0, 1, ign); tps = (match == 1) & (ign != 1)
MEGA_VE_HD double ve_fp_weight(signed char match, double ign) {
  return (match == 0 && ign != 1.0) ? (ign == 0.0 ? 1.0 : ign) : 0.0;
}
MEGA_VE_HD double ve_tp_flag(signed char match, double ign) { return (match == 1 && ign != 1.0) ? 1.0 : 0.0; }

// In place over n entries of one (class, range) list in global order: fp[i] (the fps weight) becomes the cumulative
// fp sum, tp[i] (the tps flag, 0 or 1) the cumulative tp count, exactly representable in fp64.
MEGA_VE_HD void ve_cumsum(double* fp, double* tp, long long n) {
  double f = 0.0;
  long long t = 0;
  for (long long i = 0; i < n; ++i) {
    f = MEGA_VE_DADD(f, fp[i]);
    t += tp[i] != 0.0 ? 1 : 0;
    fp[i] = f;
    tp[i] = static_cast<double>(t);
  }
}

// prec = tp / (fp + tp + eps) (the int64 tp converted to fp64 by numpy's promotion), rec = tp / n_pos
MEGA_VE_HD double ve_prec(double fp_cum, double tp_cum) {
  return MEGA_VE_DDIV(tp_cum, MEGA_VE_DADD(MEGA_VE_DADD(fp_cum, tp_cum), kEps));
}
MEGA_VE_HD double ve_rec(double tp_cum, long long n_pos) { return MEGA_VE_DDIV(tp_cum, static_cast<double>(n_pos)); }

// calc_detection_vid_ap over one (class, range) with n_pos > 0: mpre = [0, prec, 0], mrec = [0, rec, 1], mpre made
// non-increasing from the right, one output per i with mrec[i+1] != mrec[i]: dr = mrec[i+1] - mrec[i], mp = mpre[i+1],
// rr = mrec[i+1], in increasing i. Returns the number of points, or -1 (nothing written) when it exceeds `cap`.
// prec holds no NaN (its denominator is >= eps), so np.nan_to_num is the identity here.
MEGA_VE_HD long long ve_steps(const double* prec, const double* rec, long long n, long long cap, double* dr, double* mp,
                              double* rr) {
  long long cnt = 0;
  double prev = 0.0;
  for (long long i = 0; i <= n; ++i) {
    const double cur = i < n ? rec[i] : 1.0;
    cnt += cur != prev ? 1 : 0;
    prev = cur;
  }
  if (cnt > cap) return -1;
  long long k = cnt;
  double m = 0.0;
  for (long long i = n; i >= 0; --i) {
    if (i < n) m = prec[i] > m ? prec[i] : m;       // np.maximum: prec >= 0, no NaN
    const double cur = i < n ? rec[i] : 1.0, before = i > 0 ? rec[i - 1] : 0.0;
    if (cur != before) {
      --k;
      dr[k] = MEGA_VE_DSUB(cur, before);
      mp[k] = m;
      rr[k] = cur;
    }
  }
  return cnt;
}

}  // namespace mega_ve
