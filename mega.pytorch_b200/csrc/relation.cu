// Relation-module softmax with the geometric position bias generated on the fly.
//
// Reference (mega_core/modeling/roi_heads/box_head/roi_box_feature_extractors.py):
//   extract_position_matrix :146-176, extract_position_embedding :125-144 (materialises a
//   [1,64,N,M] fp32 tensor -- 648 MB at N=675, M=3750), Wg 1x1 conv + ReLU :593-597,
//   weighted_aff = log(aff_weight + 1e-6) + aff/sqrt(64) :624-632, softmax over M :633.
// Here nothing of that is materialised: for every (query n, key m) pair the four log-ratios,
// the 64 sin/cos features, the 64->16 projection, ReLU, log and the scaled logit are computed in
// registers and the soft-max is taken in place over the [G,N,M] logits produced by the
// wgmma Q.K^T GEMM. One CTA per query row; two passes over its [16,M] slice (L2-resident):
// logits + online (max, sum), then normalise.
#include <stdlib.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "mega_b200.h"

namespace mega {

constexpr int kGroups = 16;
constexpr int kEmb = 64;
constexpr int kRelThreads = 256;

struct RelParams {
  float* s;                 // [G][N][ldm] logits in, probabilities out
  __half* p16;              // optional: probabilities are written here as fp16 [G][N][ldm] (A operand of the fp16
                            // P.V' GEMM) instead of in place
  int p_split;              // p16 != NULL: 0 = plain fp16 probabilities, 1 = the split-fp16 format (include/mega_b200.h): p16 then
                            // addresses a tensor of the logits' shape and byte size, value e of it = halves 2e - (e & 31) (hi)
                            // and 2e - (e & 31) + 32 (lo)  (ldm % 32 == 0)
  long long head_stride;    // N * ldm
  int ldm;
  const float* boxes_q;     // [N,4] or NULL (no position term)
  const float* boxes_k;     // [M,4]
  const float* wg;          // [16,64] (Wgs[i].weight) or NULL
  const float* bg;          // [16]
  const float* inv_dim;     // [8]: 1 / 1000^(k/8)  (divisors, passed as the reference's dim_mat)
  const int* m_valid_ptr;   // device scalar: number of valid keys (<= ldm), or NULL -> m_host
  int m_host;
  const int* n_valid_ptr;   // rows >= *n_valid_ptr are skipped (padding rows of the key frame), or NULL
  int n_valid_off;          // rows in [n_valid, n_valid_off) are padding; rows >= n_valid_off are live
  float scale;
};

// (SPLIT is a compile-time tag: a run-time test inside the 16-fold unrolled loops of the callers cost the fp16 engine 17-28 %
//  of its soft-max kernels)
template <bool SPLIT>
__device__ __forceinline__ void store_prob16(__half* p16, long long e, float pr) {
  if (SPLIT) {
    const __half hi = __float2half_rn(pr);
    __half* b = p16 + 2 * e - (e & 31);
    b[0] = hi;
    b[32] = __float2half_rn(pr - __half2float(hi));
  } else {
    p16[e] = __float2half_rn(pr);
  }
}

// SMEM_STAGE: the row's [16, ldm] logits live in shared memory between the passes (ldm <= 1024), so the
// global logits are read once and the probabilities written once.
template <bool SMEM_STAGE>
__global__ void __launch_bounds__(kRelThreads)
relation_softmax_kernel(const RelParams p) {
  extern __shared__ float stage_s[];   // [16][ldm] when SMEM_STAGE
  __shared__ float wg_s[kEmb][kGroups];  // e-major so the 16 group weights of one feature are contiguous
  __shared__ float bg_s[kGroups];
  __shared__ float dim_s[8];
  __shared__ float red_max[kRelThreads / 32][kGroups];
  __shared__ float red_sum[kRelThreads / 32][kGroups];
  __shared__ float fin_max[kGroups], fin_inv[kGroups];

  const int n = blockIdx.x;
  const int tid = threadIdx.x;
  const int m_valid = p.m_valid_ptr ? min(*p.m_valid_ptr, p.ldm) : p.m_host;
  if (p.n_valid_ptr) {
    const int nv = *p.n_valid_ptr;
    if (n >= nv && n < p.n_valid_off) return;  // padding query row: nothing downstream reads it
  }
  const bool has_pe = (p.boxes_q != nullptr);
  if (has_pe) {
    for (int i = tid; i < kEmb * kGroups; i += blockDim.x) {
      const int g = i / kEmb, e = i - g * kEmb;
      wg_s[e][g] = p.wg[i];
    }
    if (tid < kGroups) bg_s[tid] = p.bg[tid];
    if (tid < 8) dim_s[tid] = p.inv_dim[tid];
  }
  __syncthreads();

  float qw = 1.f, qh = 1.f, qcx = 0.f, qcy = 0.f;
  if (has_pe) {
    const float4 q = *reinterpret_cast<const float4*>(p.boxes_q + static_cast<long long>(n) * 4);
    qw = __fadd_rn(__fsub_rn(q.z, q.x), 1.f);
    qh = __fadd_rn(__fsub_rn(q.w, q.y), 1.f);
    qcx = __fmul_rn(0.5f, __fadd_rn(q.x, q.z));
    qcy = __fmul_rn(0.5f, __fadd_rn(q.y, q.w));
  }
  float* srow = p.s + static_cast<long long>(n) * p.ldm;

  // running (max, sum) per head: one read+write pass produces the logits and the statistics,
  // a second read+write pass normalises (online soft-max; same value as exp(l - max) / sum)
  float mx[kGroups], sm[kGroups];
#pragma unroll
  for (int g = 0; g < kGroups; ++g) {
    mx[g] = -INFINITY;
    sm[g] = 0.f;
  }

  for (int m = tid; m < m_valid; m += blockDim.x) {
    float bias[kGroups];
    if (has_pe) {
      const float4 k = *reinterpret_cast<const float4*>(p.boxes_k + static_cast<long long>(m) * 4);
      const float kw = __fadd_rn(__fsub_rn(k.z, k.x), 1.f);
      const float kh = __fadd_rn(__fsub_rn(k.w, k.y), 1.f);
      const float kcx = __fmul_rn(0.5f, __fadd_rn(k.x, k.z));
      const float kcy = __fmul_rn(0.5f, __fadd_rn(k.y, k.w));
      float delta[4];
      delta[0] = logf(__fadd_rn(fabsf(__fdiv_rn(__fsub_rn(qcx, kcx), qw)), 1e-3f));
      delta[1] = logf(__fadd_rn(fabsf(__fdiv_rn(__fsub_rn(qcy, kcy), qh)), 1e-3f));
      delta[2] = logf(__fdiv_rn(qw, kw));
      delta[3] = logf(__fdiv_rn(qh, kh));
#pragma unroll
      for (int g = 0; g < kGroups; ++g) bias[g] = bg_s[g];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float d100 = __fmul_rn(delta[c], 100.0f);
#pragma unroll 1
        for (int kf = 0; kf < 8; ++kf) {
          const float arg = __fdiv_rn(d100, dim_s[kf]);
          // Cody-Waite reduction to [-pi, pi] (|arg| < ~1e3 here), then the SFU sin/cos
          // (abs error ~5e-7, far below the 1e-5 tolerance on the soft-max output)
          const float kq = rintf(arg * 0.15915494309189535f);
          float r = fmaf(-kq, 6.28125f, arg);
          r = fmaf(-kq, 1.9353071795864769e-3f, r);
          const float sv = __sinf(r), cv = __cosf(r);
          const float4* ws = reinterpret_cast<const float4*>(&wg_s[c * 16 + kf][0]);
          const float4* wc = reinterpret_cast<const float4*>(&wg_s[c * 16 + 8 + kf][0]);
#pragma unroll
          for (int g4 = 0; g4 < 4; ++g4) {
            const float4 a = ws[g4], b = wc[g4];
            bias[g4 * 4 + 0] = fmaf(a.x, sv, fmaf(b.x, cv, bias[g4 * 4 + 0]));
            bias[g4 * 4 + 1] = fmaf(a.y, sv, fmaf(b.y, cv, bias[g4 * 4 + 1]));
            bias[g4 * 4 + 2] = fmaf(a.z, sv, fmaf(b.z, cv, bias[g4 * 4 + 2]));
            bias[g4 * 4 + 3] = fmaf(a.w, sv, fmaf(b.w, cv, bias[g4 * 4 + 3]));
          }
        }
      }
#pragma unroll
      for (int g = 0; g < kGroups; ++g) bias[g] = __logf(__fadd_rn(fmaxf(bias[g], 0.f), 1e-6f));
    } else {
#pragma unroll
      for (int g = 0; g < kGroups; ++g) bias[g] = 0.f;
    }
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      float* sp = srow + g * p.head_stride + m;
      const float l = __fadd_rn(bias[g], __fmul_rn(p.scale, *sp));
      if (SMEM_STAGE) stage_s[g * p.ldm + m] = l; else *sp = l;
      const float nm = fmaxf(mx[g], l);
      sm[g] = sm[g] * __expf(mx[g] - nm) + __expf(l - nm);
      mx[g] = nm;
    }
  }

  // ---- block reduction of (max, sum) per head
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int g = 0; g < kGroups; ++g) {
    float m_ = mx[g], s_ = sm[g];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m_, off);
      const float os = __shfl_xor_sync(0xffffffffu, s_, off);
      const float nm = fmaxf(m_, om);
      const float a = (m_ == -INFINITY) ? 0.f : s_ * __expf(m_ - nm);
      const float b = (om == -INFINITY) ? 0.f : os * __expf(om - nm);
      s_ = a + b;
      m_ = nm;
    }
    if (lane == 0) {
      red_max[warp][g] = m_;
      red_sum[warp][g] = s_;
    }
  }
  __syncthreads();
  if (tid < kGroups) {
    float m_ = -INFINITY;
    for (int w = 0; w < kRelThreads / 32; ++w) m_ = fmaxf(m_, red_max[w][tid]);
    float s_ = 0.f;
    for (int w = 0; w < kRelThreads / 32; ++w)
      if (red_max[w][tid] != -INFINITY) s_ += red_sum[w][tid] * __expf(red_max[w][tid] - m_);
    fin_max[tid] = m_;
    fin_inv[tid] = 1.0f / s_;
  }
  __syncthreads();

  // ---- pass 2: normalise in place; padded key columns get probability 0
  for (int m = tid; m < p.ldm; m += blockDim.x) {
    if (p.p16 && p.p_split) {
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const float l = SMEM_STAGE ? stage_s[g * p.ldm + (m < m_valid ? m : 0)] : srow[g * p.head_stride + m];
        const float pr = (m < m_valid) ? __expf(l - fin_max[g]) * fin_inv[g] : 0.f;
        store_prob16<true>(p.p16, static_cast<long long>(n) * p.ldm + g * p.head_stride + m, pr);
      }
    } else {
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        float* sp = srow + g * p.head_stride + m;
        const float l = SMEM_STAGE ? stage_s[g * p.ldm + (m < m_valid ? m : 0)] : *sp;
        const float pr = (m < m_valid) ? __expf(l - fin_max[g]) * fin_inv[g] : 0.f;
        if (p.p16) p.p16[static_cast<long long>(n) * p.ldm + g * p.head_stride + m] = __float2half_rn(pr);
        else *sp = pr;
      }
    }
  }
}

// ---- the same soft-max with the 64 x 16 position weights passed BY VALUE in the kernel parameters: every weight is a
// constant-bank operand of its FFMA (no shared-memory loads at all: the smem variant above spends 256 LDS.128 per
// (query, key) pair next to its 1024 FFMAs), the k loop is fully unrolled so independent sin/cos chains overlap, the
// division by 1000^(k/8) is a reciprocal multiply + one Newton correction (same rounding as __fdiv_rn), and the online
// soft-max needs one exp per logit instead of two.
struct RelParamsW {
  RelParams b;
  float wg[kEmb * kGroups];   // [e][g]
  float bg[kGroups];
  float dim[8];
  float inv_dim[8];
};

template <bool SMEM_STAGE>
__global__ void __launch_bounds__(kRelThreads)
relation_softmax_pe_kernel(const __grid_constant__ RelParamsW pw) {
  const RelParams& p = pw.b;
  extern __shared__ float stage_s[];   // [16][ldm] when SMEM_STAGE
  __shared__ float red_max[kRelThreads / 32][kGroups];
  __shared__ float red_sum[kRelThreads / 32][kGroups];
  __shared__ float fin_max[kGroups], fin_inv[kGroups];

  const int n = blockIdx.x;
  const int tid = threadIdx.x;
  const int m_valid = p.m_valid_ptr ? min(*p.m_valid_ptr, p.ldm) : p.m_host;
  if (p.n_valid_ptr) {
    const int nv = *p.n_valid_ptr;
    if (n >= nv && n < p.n_valid_off) return;
  }
  const float4 q = *reinterpret_cast<const float4*>(p.boxes_q + static_cast<long long>(n) * 4);
  const float qw = __fadd_rn(__fsub_rn(q.z, q.x), 1.f);
  const float qh = __fadd_rn(__fsub_rn(q.w, q.y), 1.f);
  const float qcx = __fmul_rn(0.5f, __fadd_rn(q.x, q.z));
  const float qcy = __fmul_rn(0.5f, __fadd_rn(q.y, q.w));
  float* srow = p.s + static_cast<long long>(n) * p.ldm;

  float mx[kGroups], sm[kGroups];
#pragma unroll
  for (int g = 0; g < kGroups; ++g) {
    mx[g] = -INFINITY;
    sm[g] = 0.f;
  }
  for (int m = tid; m < m_valid; m += kRelThreads) {
    float lg[kGroups];
#pragma unroll
    for (int g = 0; g < kGroups; ++g) lg[g] = srow[g * p.head_stride + m];   // issued early: overlaps the arithmetic
    const float4 k = *reinterpret_cast<const float4*>(p.boxes_k + static_cast<long long>(m) * 4);
    const float kw = __fadd_rn(__fsub_rn(k.z, k.x), 1.f);
    const float kh = __fadd_rn(__fsub_rn(k.w, k.y), 1.f);
    const float kcx = __fmul_rn(0.5f, __fadd_rn(k.x, k.z));
    const float kcy = __fmul_rn(0.5f, __fadd_rn(k.y, k.w));
    float delta[4];
    delta[0] = logf(__fadd_rn(fabsf(__fdiv_rn(__fsub_rn(qcx, kcx), qw)), 1e-3f));
    delta[1] = logf(__fadd_rn(fabsf(__fdiv_rn(__fsub_rn(qcy, kcy), qh)), 1e-3f));
    delta[2] = logf(__fdiv_rn(qw, kw));
    delta[3] = logf(__fdiv_rn(qh, kh));
    float bias[kGroups];
#pragma unroll
    for (int g = 0; g < kGroups; ++g) bias[g] = pw.bg[g];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float d100 = __fmul_rn(delta[c], 100.0f);
#pragma unroll
      for (int kf = 0; kf < 8; ++kf) {
        // arg = d100 / dim[kf], correctly rounded: q0 = a * (1/b); r = a - q0 * b (exact in an fma); q = q0 + r * (1/b)
        const float q0 = __fmul_rn(d100, pw.inv_dim[kf]);
        const float rem = __fmaf_rn(-q0, pw.dim[kf], d100);
        const float arg = __fmaf_rn(rem, pw.inv_dim[kf], q0);
        const float kq = rintf(arg * 0.15915494309189535f);
        float r = fmaf(-kq, 6.28125f, arg);
        r = fmaf(-kq, 1.9353071795864769e-3f, r);
        const float sv = __sinf(r), cv = __cosf(r);
#pragma unroll
        for (int g = 0; g < kGroups; ++g) {
          bias[g] = fmaf(pw.wg[(c * 16 + kf) * kGroups + g], sv, fmaf(pw.wg[(c * 16 + 8 + kf) * kGroups + g], cv, bias[g]));
        }
      }
    }
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      const float b = __logf(__fadd_rn(fmaxf(bias[g], 0.f), 1e-6f));
      const float l = __fadd_rn(b, __fmul_rn(p.scale, lg[g]));
      if (SMEM_STAGE) stage_s[g * p.ldm + m] = l; else srow[g * p.head_stride + m] = l;
      // online (max, sum) with one exp: e = exp(-|l - mx|)
      const float d = l - mx[g];
      const float e = __expf(-fabsf(d));
      sm[g] = (d > 0.f) ? fmaf(sm[g], e, 1.f) : (sm[g] + e);
      mx[g] = fmaxf(mx[g], l);
    }
  }

  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int g = 0; g < kGroups; ++g) {
    float m_ = mx[g], s_ = sm[g];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m_, off);
      const float os = __shfl_xor_sync(0xffffffffu, s_, off);
      const float nm = fmaxf(m_, om);
      const float a = (m_ == -INFINITY) ? 0.f : s_ * __expf(m_ - nm);
      const float b = (om == -INFINITY) ? 0.f : os * __expf(om - nm);
      s_ = a + b;
      m_ = nm;
    }
    if (lane == 0) {
      red_max[warp][g] = m_;
      red_sum[warp][g] = s_;
    }
  }
  __syncthreads();
  if (tid < kGroups) {
    float m_ = -INFINITY;
    for (int w = 0; w < kRelThreads / 32; ++w) m_ = fmaxf(m_, red_max[w][tid]);
    float s_ = 0.f;
    for (int w = 0; w < kRelThreads / 32; ++w)
      if (red_max[w][tid] != -INFINITY) s_ += red_sum[w][tid] * __expf(red_max[w][tid] - m_);
    fin_max[tid] = m_;
    fin_inv[tid] = 1.0f / s_;
  }
  __syncthreads();
  for (int m = tid; m < p.ldm; m += kRelThreads) {
    if (p.p16 && p.p_split) {
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const float l = SMEM_STAGE ? stage_s[g * p.ldm + (m < m_valid ? m : 0)] : srow[g * p.head_stride + m];
        const float pr = (m < m_valid) ? __expf(l - fin_max[g]) * fin_inv[g] : 0.f;
        store_prob16<true>(p.p16, static_cast<long long>(n) * p.ldm + g * p.head_stride + m, pr);
      }
    } else {
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        float* sp = srow + g * p.head_stride + m;
        const float l = SMEM_STAGE ? stage_s[g * p.ldm + (m < m_valid ? m : 0)] : *sp;
        const float pr = (m < m_valid) ? __expf(l - fin_max[g]) * fin_inv[g] : 0.f;
        if (p.p16) p.p16[static_cast<long long>(n) * p.ldm + g * p.head_stride + m] = __float2half_rn(pr);
        else *sp = pr;
      }
    }
  }
}

// ---- the position bias as a tensor-core product. bias[m, g] = sum_e emb[m, e] * Wg[g, e] is a [keys x 64] x [64 x 16]
// GEMM per query row: 1024 FFMAs per (query, key) pair on the SIMT pipe, but 3 x 32 warp-level m16n8k8 MMAs per 32 pairs
// on the tensor cores. To keep fp32-level accuracy (the bias feeds log(relu(.) + 1e-6)) both operands are split
// x = hi + lo with hi = x truncated to TF32 (exactly representable) and the product is hi*hi + hi*lo + lo*hi with fp32
// accumulation ("3xTF32", relative error ~1e-6). Each thread computes exactly the sin / cos values of its own A
// fragment slots (pairs g, g+8 x frequencies t, t+4 of the lane = 4g + t), so nothing is transposed through memory.
__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

constexpr int kWgPitch = 24;   // floats per feature row of the smem weight tables (conflict-free B-fragment reads)

template <bool SMEM_STAGE>
__global__ void __launch_bounds__(kRelThreads)
relation_softmax_mma_kernel(const __grid_constant__ RelParamsW pw) {
  const RelParams& p = pw.b;
  extern __shared__ float stage_s[];   // [16][ldm] when SMEM_STAGE
  __shared__ uint32_t wg_hi[kEmb * kWgPitch], wg_lo[kEmb * kWgPitch];
  __shared__ float red_max[kRelThreads / 32][kGroups];
  __shared__ float red_sum[kRelThreads / 32][kGroups];
  __shared__ float fin_max[kGroups], fin_inv[kGroups];

  const int n = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int m_valid = p.m_valid_ptr ? min(*p.m_valid_ptr, p.ldm) : p.m_host;
  if (p.n_valid_ptr) {
    const int nv = *p.n_valid_ptr;
    if (n >= nv && n < p.n_valid_off) return;
  }
  for (int i = tid; i < kEmb * kGroups; i += kRelThreads) {
    const int e = i / kGroups, h = i - e * kGroups;
    uint32_t hi, lo;
    split_tf32(pw.wg[e * kGroups + h], hi, lo);
    wg_hi[e * kWgPitch + h] = hi;
    wg_lo[e * kWgPitch + h] = lo;
  }
  __syncthreads();
  const float4 q = *reinterpret_cast<const float4*>(p.boxes_q + static_cast<long long>(n) * 4);
  const float qw = __fadd_rn(__fsub_rn(q.z, q.x), 1.f);
  const float qh = __fadd_rn(__fsub_rn(q.w, q.y), 1.f);
  const float qcx = __fmul_rn(0.5f, __fadd_rn(q.x, q.z));
  const float qcy = __fmul_rn(0.5f, __fadd_rn(q.y, q.w));
  float* srow = p.s + static_cast<long long>(n) * p.ldm;
  // this lane's two frequencies (k columns t and t + 4 of every 8-wide k-step)
  const float dimA = pw.dim[t], invA = pw.inv_dim[t], dimB = pw.dim[t + 4], invB = pw.inv_dim[t + 4];
  // this lane's four heads: columns 2t, 2t+1 of the two n-tiles
  const int hd[4] = {2 * t, 2 * t + 1, 8 + 2 * t, 9 + 2 * t};
  float bgv[4], mx[4], sm[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    bgv[j] = pw.bg[hd[j]];
    mx[j] = -INFINITY;
    sm[j] = 0.f;
  }

  for (int m0 = warp * 32; m0 < m_valid; m0 += (kRelThreads / 32) * 32) {
    // ---- lane L: the four 100 x log-ratios of key m0 + L
    const int mk = min(m0 + lane, m_valid - 1);
    const float4 k = *reinterpret_cast<const float4*>(p.boxes_k + static_cast<long long>(mk) * 4);
    const float kw = __fadd_rn(__fsub_rn(k.z, k.x), 1.f);
    const float kh = __fadd_rn(__fsub_rn(k.w, k.y), 1.f);
    const float kcx = __fmul_rn(0.5f, __fadd_rn(k.x, k.z));
    const float kcy = __fmul_rn(0.5f, __fadd_rn(k.y, k.w));
    float d100[4];
    d100[0] = __fmul_rn(logf(__fadd_rn(fabsf(__fdiv_rn(__fsub_rn(qcx, kcx), qw)), 1e-3f)), 100.0f);
    d100[1] = __fmul_rn(logf(__fadd_rn(fabsf(__fdiv_rn(__fsub_rn(qcy, kcy), qh)), 1e-3f)), 100.0f);
    d100[2] = __fmul_rn(logf(__fdiv_rn(qw, kw)), 100.0f);
    d100[3] = __fmul_rn(logf(__fdiv_rn(qh, kh)), 100.0f);
    // the 16 logits of this lane's C-fragment slots, issued before the arithmetic so their latency is covered
    float lg[2][2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int m = min(m0 + mt * 16 + g + half * 8, m_valid - 1);
#pragma unroll
        for (int j = 0; j < 4; ++j) lg[mt][half][j] = srow[hd[j] * p.head_stride + m];
      }
    float acc[2][2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[mt][nt][j] = 0.f;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        // A-fragment slots of this lane: rows (pairs) g, g + 8 of the m-tile; k columns (frequencies) t, t + 4
        const float dlo = __shfl_sync(0xffffffffu, d100[c], mt * 16 + g);
        const float dhi = __shfl_sync(0xffffffffu, d100[c], mt * 16 + g + 8);
        float sv[4], cv[4];
#pragma unroll
        for (int slot = 0; slot < 4; ++slot) {
          const float d = (slot & 1) ? dhi : dlo;                 // a0/a2: row g, a1/a3: row g + 8
          const float dm = (slot & 2) ? dimB : dimA, iv = (slot & 2) ? invB : invA;   // a0/a1: col t, a2/a3: col t + 4
          const float q0 = __fmul_rn(d, iv);
          const float rem = __fmaf_rn(-q0, dm, d);
          const float arg = __fmaf_rn(rem, iv, q0);
          const float kq = rintf(arg * 0.15915494309189535f);
          float r = fmaf(-kq, 6.28125f, arg);
          r = fmaf(-kq, 1.9353071795864769e-3f, r);
          sv[slot] = __sinf(r);
          cv[slot] = __cosf(r);
        }
#pragma unroll
        for (int sc = 0; sc < 2; ++sc) {            // k-step 2c: the sin block of coordinate c, 2c + 1: the cos block
          uint32_t ahi[4], alo[4];
#pragma unroll
          for (int slot = 0; slot < 4; ++slot) split_tf32(sc ? cv[slot] : sv[slot], ahi[slot], alo[slot]);
          const int e0 = (2 * c + sc) * 8;          // first feature of this k-step
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) {
            const int o0 = (e0 + t) * kWgPitch + nt * 8 + g, o1 = (e0 + t + 4) * kWgPitch + nt * 8 + g;
            const uint32_t bh0 = wg_hi[o0], bh1 = wg_hi[o1], bl0 = wg_lo[o0], bl1 = wg_lo[o1];
            mma_tf32_16x8x8(acc[mt][nt], alo, bh0, bh1);
            mma_tf32_16x8x8(acc[mt][nt], ahi, bl0, bl1);
            mma_tf32_16x8x8(acc[mt][nt], ahi, bh0, bh1);
          }
        }
      }
    }
    // ---- C fragments: (pair g | g + 8 of m-tile mt) x (heads 2t, 2t+1 of n-tile nt)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int m = m0 + mt * 16 + g + half * 8;
        if (m < m_valid) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float bsum = acc[mt][j >> 1][half * 2 + (j & 1)] + bgv[j];
            const float b = __logf(__fadd_rn(fmaxf(bsum, 0.f), 1e-6f));
            const float l = __fadd_rn(b, __fmul_rn(p.scale, lg[mt][half][j]));
            if (SMEM_STAGE) stage_s[hd[j] * p.ldm + m] = l; else srow[hd[j] * p.head_stride + m] = l;
            const float d = l - mx[j];
            const float e = __expf(-fabsf(d));
            sm[j] = (d > 0.f) ? fmaf(sm[j], e, 1.f) : (sm[j] + e);
            mx[j] = fmaxf(mx[j], l);
          }
        }
      }
    }
  }

  // ---- (max, sum) per head: lanes with the same t (8 lanes: xor 4, 8, 16), then across warps
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float m_ = mx[j], s_ = sm[j];
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m_, off);
      const float os = __shfl_xor_sync(0xffffffffu, s_, off);
      const float nm = fmaxf(m_, om);
      const float a = (m_ == -INFINITY) ? 0.f : s_ * __expf(m_ - nm);
      const float b = (om == -INFINITY) ? 0.f : os * __expf(om - nm);
      s_ = a + b;
      m_ = nm;
    }
    if (g == 0) {
      red_max[warp][hd[j]] = m_;
      red_sum[warp][hd[j]] = s_;
    }
  }
  __syncthreads();
  if (tid < kGroups) {
    float m_ = -INFINITY;
    for (int w = 0; w < kRelThreads / 32; ++w) m_ = fmaxf(m_, red_max[w][tid]);
    float s_ = 0.f;
    for (int w = 0; w < kRelThreads / 32; ++w)
      if (red_max[w][tid] != -INFINITY) s_ += red_sum[w][tid] * __expf(red_max[w][tid] - m_);
    fin_max[tid] = m_;
    fin_inv[tid] = 1.0f / s_;
  }
  __syncthreads();
  for (int m = tid; m < p.ldm; m += kRelThreads) {
    if (p.p16 && p.p_split) {
#pragma unroll
      for (int h = 0; h < kGroups; ++h) {
        const float l = SMEM_STAGE ? stage_s[h * p.ldm + (m < m_valid ? m : 0)] : srow[h * p.head_stride + m];
        const float pr = (m < m_valid) ? __expf(l - fin_max[h]) * fin_inv[h] : 0.f;
        store_prob16<true>(p.p16, static_cast<long long>(n) * p.ldm + h * p.head_stride + m, pr);
      }
    } else {
#pragma unroll
      for (int h = 0; h < kGroups; ++h) {
        float* sp = srow + h * p.head_stride + m;
        const float l = SMEM_STAGE ? stage_s[h * p.ldm + (m < m_valid ? m : 0)] : *sp;
        const float pr = (m < m_valid) ? __expf(l - fin_max[h]) * fin_inv[h] : 0.f;
        if (p.p16) p.p16[static_cast<long long>(n) * p.ldm + h * p.head_stride + m] = __float2half_rn(pr);
        else *sp = pr;
      }
    }
  }
}

// No position term: one warp per (head, query row); the row (<= 1024 keys) stays in registers, so the
// logits are read once and the probabilities written once.
__global__ void __launch_bounds__(256)
plain_softmax_kernel(float* __restrict__ s, __half* __restrict__ p16, int p_split, int n_rows, int ldm, long long head_stride,
                     const int* m_valid_ptr, int m_host, const int* n_valid_ptr, int n_valid_off, float scale) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= n_rows * kGroups) return;
  const int g = wid / n_rows, n = wid - g * n_rows;
  if (n_valid_ptr) {
    const int nv = *n_valid_ptr;
    if (n >= nv && n < n_valid_off) return;
  }
  const int m_valid = m_valid_ptr ? min(*m_valid_ptr, ldm) : m_host;
  float* row = s + g * head_stride + static_cast<long long>(n) * ldm;
  float v[32];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int m = j * 32 + lane;
    v[j] = (m < m_valid) ? scale * row[m] : -INFINITY;
    mx = fmaxf(mx, v[j]);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    v[j] = (j * 32 + lane < m_valid) ? expf(v[j] - mx) : 0.f;
    sum += v[j];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  const float inv = sum > 0.f ? 1.0f / sum : 0.f;   // no valid key (m_valid == 0): every probability 0, not 0 * inf
  if (p16 && p_split) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int m = j * 32 + lane;
      if (m < ldm) store_prob16<true>(p16, g * head_stride + static_cast<long long>(n) * ldm + m, v[j] * inv);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int m = j * 32 + lane;
      if (m < ldm) {
        if (p16) p16[g * head_stride + static_cast<long long>(n) * ldm + m] = __float2half_rn(v[j] * inv);
        else row[m] = v[j] * inv;
      }
    }
  }
}

}  // namespace mega

using namespace mega;

static int relation_softmax_impl(float* logits, void* probs_f16, int p_split, int n_rows, int ldm, const float* boxes_q,
                                 const float* boxes_k, const float* wg, const float* bg, const float* dim_mat,
                                 const int* m_valid_ptr, int m_host, const int* n_valid_ptr, int n_valid_off,
                                 float scale, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(logits != nullptr && n_rows >= 0 && ldm > 0, "relation_softmax: bad arguments");
  MEGA_ARG_CHECK((boxes_q == nullptr) || (boxes_k && wg && bg && dim_mat),
                 "relation_softmax: position term needs boxes_k, wg, bg and dim_mat");
  MEGA_ARG_CHECK(m_valid_ptr != nullptr || (m_host >= 0 && m_host <= ldm), "relation_softmax: m out of range");
  if (n_rows == 0) return MEGA_OK;
  RelParams p;
  p.s = logits;
  MEGA_ARG_CHECK(!p_split || (ldm % 32 == 0 && (reinterpret_cast<uintptr_t>(probs_f16) & 127) == 0),
                 "relation_softmax: split-fp16 probabilities need ldm %% 32 == 0 and a 128-byte aligned tensor");
  p.p16 = static_cast<__half*>(probs_f16);
  p.p_split = p_split;
  p.head_stride = static_cast<long long>(n_rows) * ldm;
  p.ldm = ldm;
  p.boxes_q = boxes_q;
  p.boxes_k = boxes_k;
  p.wg = wg;
  p.bg = bg;
  p.inv_dim = dim_mat;
  p.m_valid_ptr = m_valid_ptr;
  p.m_host = m_host;
  p.n_valid_ptr = n_valid_ptr;
  p.n_valid_off = n_valid_off;
  p.scale = scale;
  if (boxes_q == nullptr && ldm <= 1024) {
    const long long warps = static_cast<long long>(n_rows) * kGroups;
    plain_softmax_kernel<<<static_cast<int>((warps * 32 + 255) / 256), 256, 0, stream>>>(
        logits, p.p16, p_split, n_rows, ldm, p.head_stride, m_valid_ptr, m_host, n_valid_ptr, n_valid_off, scale);
  } else if (ldm <= 1024) {
    const int smem = kGroups * ldm * static_cast<int>(sizeof(float));
    static bool configured = false;
    if (!configured) {
      MEGA_CUDA_CHECK(cudaFuncSetAttribute(relation_softmax_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           kGroups * 1024 * static_cast<int>(sizeof(float))));
      configured = true;
    }
    relation_softmax_kernel<true><<<n_rows, kRelThreads, smem, stream>>>(p);
  } else {
    relation_softmax_kernel<false><<<n_rows, kRelThreads, 0, stream>>>(p);
  }
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_relation_softmax(float* logits, int n_rows, int ldm, const float* boxes_q, const float* boxes_k,
                                     const float* wg, const float* bg, const float* dim_mat, const int* m_valid_ptr,
                                     int m_host, const int* n_valid_ptr, int n_valid_off, float scale,
                                     void* stream_v) {
  return relation_softmax_impl(logits, nullptr, 0, n_rows, ldm, boxes_q, boxes_k, wg, bg, dim_mat, m_valid_ptr, m_host,
                               n_valid_ptr, n_valid_off, scale, stream_v);
}

extern "C" int mega_relation_softmax_f16(float* logits, void* probs_f16, int n_rows, int ldm, const float* boxes_q,
                                         const float* boxes_k, const float* wg, const float* bg, const float* dim_mat,
                                         const int* m_valid_ptr, int m_host, const int* n_valid_ptr, int n_valid_off,
                                         float scale, void* stream_v) {
  MEGA_ARG_CHECK(probs_f16 != nullptr, "relation_softmax_f16: probs_f16 is NULL");
  return relation_softmax_impl(logits, probs_f16, 0, n_rows, ldm, boxes_q, boxes_k, wg, bg, dim_mat, m_valid_ptr, m_host,
                               n_valid_ptr, n_valid_off, scale, stream_v);
}

/* same, the probabilities written in the split-fp16 format (a tensor of the logits' shape and byte size) */
extern "C" int mega_relation_softmax_split16(float* logits, void* probs, int n_rows, int ldm, const float* boxes_q,
                                             const float* boxes_k, const float* wg, const float* bg, const float* dim_mat,
                                             const int* m_valid_ptr, int m_host, const int* n_valid_ptr, int n_valid_off,
                                             float scale, void* stream_v) {
  MEGA_ARG_CHECK(probs != nullptr, "relation_softmax_split16: probs is NULL");
  return relation_softmax_impl(logits, probs, 1, n_rows, ldm, boxes_q, boxes_k, wg, bg, dim_mat, m_valid_ptr, m_host,
                               n_valid_ptr, n_valid_off, scale, stream_v);
}

static int relation_softmax_pe_impl(float* logits, void* probs_f16, int p_split, int n_rows, int ldm, const float* boxes_q,
                                    const float* boxes_k, const float* wg_host, const float* bg_host,
                                    const float* dim_mat_host, const int* m_valid_ptr, int m_host,
                                    const int* n_valid_ptr, int n_valid_off, float scale, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(!p_split || (probs_f16 != nullptr && ldm % 32 == 0 && (reinterpret_cast<uintptr_t>(probs_f16) & 127) == 0),
                 "relation_softmax_pe: split-fp16 probabilities need ldm %% 32 == 0 and a 128-byte aligned tensor");
  MEGA_ARG_CHECK(logits != nullptr && n_rows >= 0 && ldm > 0 && boxes_q && boxes_k && wg_host && bg_host && dim_mat_host,
                 "relation_softmax_pe: bad arguments");
  MEGA_ARG_CHECK(m_valid_ptr != nullptr || (m_host >= 0 && m_host <= ldm), "relation_softmax_pe: m out of range");
  if (n_rows == 0) return MEGA_OK;
  RelParamsW pw;
  RelParams& p = pw.b;
  p.s = logits;
  p.p16 = static_cast<__half*>(probs_f16);
  p.p_split = p_split;
  p.head_stride = static_cast<long long>(n_rows) * ldm;
  p.ldm = ldm;
  p.boxes_q = boxes_q;
  p.boxes_k = boxes_k;
  p.wg = nullptr;
  p.bg = nullptr;
  p.inv_dim = nullptr;
  p.m_valid_ptr = m_valid_ptr;
  p.m_host = m_host;
  p.n_valid_ptr = n_valid_ptr;
  p.n_valid_off = n_valid_off;
  p.scale = scale;
  for (int g = 0; g < kGroups; ++g) {
    pw.bg[g] = bg_host[g];
    for (int e = 0; e < kEmb; ++e) pw.wg[e * kGroups + g] = wg_host[g * kEmb + e];
  }
  for (int k = 0; k < 8; ++k) {
    pw.dim[k] = dim_mat_host[k];
    pw.inv_dim[k] = 1.0f / dim_mat_host[k];
  }
  static int use_mma = -1;
  if (use_mma < 0) {
    const char* e = getenv("MEGA_B200_SOFTMAX_SIMT");
    use_mma = (e && e[0] == '1') ? 0 : 1;
  }
  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(relation_softmax_pe_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kGroups * 1024 * static_cast<int>(sizeof(float))));
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(relation_softmax_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kGroups * 1024 * static_cast<int>(sizeof(float))));
    configured = true;
  }
  const int smem = kGroups * ldm * static_cast<int>(sizeof(float));
  // measured (B200, 675 query rows): keys <= 1024 (logits staged in smem) 60 us with the tensor-core bias vs 70 us
  // with FFMAs; 3750 keys (two passes over 163 MB of fp32 logits in global memory: bandwidth-bound) 250 vs 242 us
  if (use_mma && ldm <= 1024) {
    relation_softmax_mma_kernel<true><<<n_rows, kRelThreads, smem, stream>>>(pw);
  } else if (ldm <= 1024) {
    relation_softmax_pe_kernel<true><<<n_rows, kRelThreads, smem, stream>>>(pw);
  } else {
    relation_softmax_pe_kernel<false><<<n_rows, kRelThreads, 0, stream>>>(pw);
  }
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_relation_softmax_pe(float* logits, void* probs_f16, int n_rows, int ldm, const float* boxes_q,
                                        const float* boxes_k, const float* wg_host, const float* bg_host,
                                        const float* dim_mat_host, const int* m_valid_ptr, int m_host,
                                        const int* n_valid_ptr, int n_valid_off, float scale, void* stream_v) {
  return relation_softmax_pe_impl(logits, probs_f16, 0, n_rows, ldm, boxes_q, boxes_k, wg_host, bg_host, dim_mat_host,
                                  m_valid_ptr, m_host, n_valid_ptr, n_valid_off, scale, stream_v);
}

/* same, the probabilities written in the split-fp16 format (a tensor of the logits' shape and byte size) */
extern "C" int mega_relation_softmax_pe_split16(float* logits, void* probs, int n_rows, int ldm, const float* boxes_q,
                                                const float* boxes_k, const float* wg_host, const float* bg_host,
                                                const float* dim_mat_host, const int* m_valid_ptr, int m_host,
                                                const int* n_valid_ptr, int n_valid_off, float scale, void* stream_v) {
  return relation_softmax_pe_impl(logits, probs, 1, n_rows, ldm, boxes_q, boxes_k, wg_host, bg_host, dim_mat_host,
                                  m_valid_ptr, m_host, n_valid_ptr, n_valid_off, scale, stream_v);
}
