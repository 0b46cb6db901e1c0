// IoU threshold decisions shared by the proposal (proposals.cu), detection (postprocess.cu) and Seq-NMS (seq_nms.cu)
// kernels. Reference arithmetic: nms.cu:16-19 / nms_cpu.cpp:6-75 ("+1" pixel convention, fp32, division then compare).
// The functions are __host__ __device__: g++ compiles them for the host builds under tests/native, where every fp32
// operation is a separately rounded IEEE operation as well (x86-64 SSE without -mfma, -ffp-contract=off).
#pragma once

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#define MEGA_IOU_HD __host__ __device__ __forceinline__
#else
#include <math.h>
#define MEGA_IOU_HD static inline
struct float4 {   // host-only builds: the layout of CUDA's vector type
  float x, y, z, w;
};
#endif
#if defined(__CUDA_ARCH__)
#define MEGA_IOU_ADD(a, b) __fadd_rn((a), (b))
#define MEGA_IOU_SUB(a, b) __fsub_rn((a), (b))
#define MEGA_IOU_MUL(a, b) __fmul_rn((a), (b))
#define MEGA_IOU_DIV(a, b) __fdiv_rn((a), (b))
#else
#define MEGA_IOU_ADD(a, b) ((a) + (b))
#define MEGA_IOU_SUB(a, b) ((a) - (b))
#define MEGA_IOU_MUL(a, b) ((a) * (b))
#define MEGA_IOU_DIV(a, b) ((a) / (b))
#endif

namespace mega {

MEGA_IOU_HD float box_area_plus1(const float4 a) {
  return MEGA_IOU_MUL(MEGA_IOU_ADD(MEGA_IOU_SUB(a.z, a.x), 1.f), MEGA_IOU_ADD(MEGA_IOU_SUB(a.w, a.y), 1.f));
}

// iou_plus1(a, b) > thresh with the SAME outcome for every input, but without the division unless the quotient is
// within 2^-20 (relative) of the threshold: RN(inter / u) > t is decided by inter vs t*u whenever the true quotient is
// more than a few ulps away from t (t_lo = t*(1-2^-20), t_hi = t*(1+2^-20); the two products carry 2^-24 relative
// error each, far inside the band). sa / sb: box_area_plus1 of a / b.
MEGA_IOU_HD bool iou_plus1_gt(const float4 a, const float sa, const float4 b, const float sb, const float thresh,
                              const float t_lo, const float t_hi) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float width = fmaxf(MEGA_IOU_ADD(MEGA_IOU_SUB(right, left), 1.f), 0.f);
  const float height = fmaxf(MEGA_IOU_ADD(MEGA_IOU_SUB(bottom, top), 1.f), 0.f);
  const float inter = MEGA_IOU_MUL(width, height);
  const float u = MEGA_IOU_SUB(MEGA_IOU_ADD(sa, sb), inter);
  if (u > 0.f) {
    if (inter > MEGA_IOU_MUL(t_hi, u)) return true;
    if (inter < MEGA_IOU_MUL(t_lo, u)) return false;
  }
  return MEGA_IOU_DIV(inter, u) > thresh;
}

}  // namespace mega
