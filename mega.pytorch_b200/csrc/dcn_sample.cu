// Deformable-convolution sampling over NHWC activations into the column operand of a 1x1 GEMM: the middle launch of a
// deformable bottleneck conv2 (MODEL.RESNETS.STAGE_WITH_DCN). The offset conv before it and the contraction after it
// (K = 9 C, tap-major) are conv_gemm launches. One output row per pixel:
//     cols[pixel][tap * C + c] = mask(pixel, tap) * bilinear(input, position(pixel, tap, g))[c],   g = c / (C / dg)
// with position = (h * stride - dil + i * dil + dh, w * stride - dil + j * dil + dw) for tap = 3 i + j (the DFConv2d
// padding: dil), (dh, dw) = offset[pixel][18 g + 2 tap], offset[pixel][18 g + 2 tap + 1] -- deformable group g of dg
// samples its C / dg consecutive channels at its own 9 positions -- and mask = sigmoid(offset[pixel][18 + tap]) for
// DCN v2 (one group), 1 for v1. The geometry and the interpolation are dcn_sample.cuh, shared with deform.cu's tile
// kernel.
//
// A CTA owns kSampPix / dg consecutive pixels (at least one): the 9 dg (tap, group) samples of each get their geometry
// (floor, weights, corner indices) once, into dynamic shared memory -- at most 16 x 9 samples for dg <= 16, 9 dg above;
// then every thread takes (pixel, tap, 8-channel chunk) items, chunk fastest, and reads the geometry of the chunk's
// group. The four corners of a sample are contiguous C-vectors in NHWC, so a warp reads whole corner rows with 128-bit
// loads and writes the column row contiguously. Values are interpolated in fp32 in every storage format.
#include "common.cuh"
#include "dcn_sample.cuh"
#include "mega_b200.h"

namespace mega {

constexpr int kSampPix = 16;
constexpr int kSampThreads = 256;
constexpr int kSampMaxGroups = 128;     // 9 x 128 samples of one pixel: 41.5 KB of geometry, under the 48 KB default

struct Vec8 {
  float v[8];
};

// 8 consecutive channels starting at element `e` (a multiple of 8) of an NHWC tensor in the storage format FMT
template <int FMT>
__device__ __forceinline__ Vec8 load8(const void* base, long long e) {
  Vec8 r;
  if (FMT == MEGA_DCN_FP32) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(base) + e));
    const float4 b = __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(base) + e + 4));
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  } else if (FMT == MEGA_DCN_FP16) {
    const uint4 h = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(base) + e));
    const uint32_t w[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = h2_to_f2(w[k]);
      r.v[2 * k] = f.x; r.v[2 * k + 1] = f.y;
    }
  } else {      // split-fp16: group e / 32 is 128 bytes [32 hi halves | 32 lo halves]; value = hi + lo
    const char* g = static_cast<const char*>(base) + (e >> 5) * 128 + (e & 31) * 2;
    const uint4 hi = __ldg(reinterpret_cast<const uint4*>(g));
    const uint4 lo = __ldg(reinterpret_cast<const uint4*>(g + 64));
    const uint32_t wh[4] = {hi.x, hi.y, hi.z, hi.w}, wl[4] = {lo.x, lo.y, lo.z, lo.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = h2_to_f2(wh[k]), b = h2_to_f2(wl[k]);
      r.v[2 * k] = a.x + b.x; r.v[2 * k + 1] = a.y + b.y;
    }
  }
  return r;
}

template <int FMT>
__device__ __forceinline__ void store8(void* base, long long e, const float (&x)[8]) {
  if (FMT == MEGA_DCN_FP32) {
    float* p = static_cast<float*>(base) + e;
    *reinterpret_cast<float4*>(p) = make_float4(x[0], x[1], x[2], x[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(x[4], x[5], x[6], x[7]);
  } else if (FMT == MEGA_DCN_FP16) {
    *reinterpret_cast<uint4*>(static_cast<uint16_t*>(base) + e) =
        make_uint4(f2_to_h2(x[0], x[1]), f2_to_h2(x[2], x[3]), f2_to_h2(x[4], x[5]), f2_to_h2(x[6], x[7]));
  } else {      // the split of ops.pack_split16: hi = fp16(x), lo = fp16(x - hi), both saturating
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      hi[k] = f2_to_h2_sat(x[2 * k], x[2 * k + 1]);
      const float2 b = h2_to_f2(hi[k]);
      lo[k] = f2_to_h2_sat(x[2 * k] - b.x, x[2 * k + 1] - b.y);
    }
    char* g = static_cast<char*>(base) + (e >> 5) * 128 + (e & 31) * 2;
    *reinterpret_cast<uint4*>(g) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(g + 64) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

template <int FMT>
__global__ void __launch_bounds__(kSampThreads)
dcn_sample_nhwc_kernel(const void* __restrict__ input, int height, int width, int channels, int groups,
                       int cta_pix, const float* __restrict__ offset, int offset_ld, int modulated, int stride,
                       int dil, int ho, int wo, long long pixels, void* __restrict__ cols) {
  extern __shared__ float4 smem[];
  DcnTap* geo = reinterpret_cast<DcnTap*>(smem);                       // [cta_pix][9][groups]
  float* mval = reinterpret_cast<float*>(geo + cta_pix * 9 * groups);   // likewise
  const long long p0 = static_cast<long long>(blockIdx.x) * cta_pix;
  const int npix = static_cast<int>(min(static_cast<long long>(cta_pix), pixels - p0));
  const int per_pix = 9 * groups;
  for (int t = threadIdx.x; t < npix * per_pix; t += kSampThreads) {
    const int lp = t / per_pix, r = t - lp * per_pix, tap = r / groups, grp = r - tap * groups;
    const long long pix = p0 + lp;
    const int i = tap / 3, j = tap - 3 * i;
    const int w_col = static_cast<int>(pix % wo), h_col = static_cast<int>((pix / wo) % ho);
    const float* o = offset + pix * offset_ld;
    const float h_im = h_col * stride - dil + i * dil + __ldg(o + 18 * grp + 2 * tap);
    const float w_im = w_col * stride - dil + j * dil + __ldg(o + 18 * grp + 2 * tap + 1);
    geo[t] = dcn_tap_geometry(h_im, w_im, height, width);
    mval[t] = modulated ? dcn_sigmoid(__ldg(o + 18 + tap)) : 1.f;
  }
  __syncthreads();
  const int chunks = channels >> 3, group_chunks = chunks / groups;
  const long long plane = static_cast<long long>(height) * width;
  for (int it = threadIdx.x; it < npix * 9 * chunks; it += kSampThreads) {
    const int t = it / chunks, q = it - t * chunks;
    const long long pix = p0 + t / 9;
    const int tap = t % 9;
    const int s = t * groups + q / group_chunks;
    const DcnTap g = geo[s];
    const long long img = pix / (static_cast<long long>(ho) * wo) * plane;      // first pixel of the image
    const int c = q * 8;
    float x[8];
    if (g.i00 == kDcnOutside) {
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = 0.f;
    } else {
      Vec8 v[4];
      const int idx[4] = {g.i00, g.i01, g.i10, g.i11};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (idx[r] >= 0) {
          v[r] = load8<FMT>(input, (img + idx[r]) * channels + c);
        } else {
#pragma unroll
          for (int k = 0; k < 8; ++k) v[r].v[k] = 0.f;
        }
      }
      const float m = mval[s];
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = dcn_blend(g, v[0].v[k], v[1].v[k], v[2].v[k], v[3].v[k]) * m;
    }
    store8<FMT>(cols, pix * 9 * channels + tap * channels + c, x);
  }
}

}  // namespace mega

using namespace mega;

extern "C" int mega_dcn_sample_nhwc_groups(const void* input, int format, int batch, int height, int width,
                                           int channels, int deformable_groups, const float* offset, int offset_ld,
                                           int modulated, int stride, int dil, void* cols, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int dg = deformable_groups;
  MEGA_ARG_CHECK(format == MEGA_DCN_FP32 || format == MEGA_DCN_FP16 || format == MEGA_DCN_SPLIT16,
                 "dcn_sample_nhwc: format must be MEGA_DCN_FP32, _FP16 or _SPLIT16");
  MEGA_ARG_CHECK(batch >= 0 && height > 0 && width > 0 && channels > 0 && channels % 32 == 0,
                 "dcn_sample_nhwc: channels must be a positive multiple of 32");
  MEGA_ARG_CHECK(dg >= 1 && dg <= kSampMaxGroups && channels % dg == 0 && (channels / dg) % 8 == 0,
                 "dcn_sample_nhwc: deformable_groups must be 1..128 and divide channels into multiples of 8");
  MEGA_ARG_CHECK(!modulated || dg == 1, "dcn_sample_nhwc: modulated sampling takes one deformable group");
  MEGA_ARG_CHECK(stride >= 1 && dil >= 1, "dcn_sample_nhwc: stride and dilation must be >= 1");
  MEGA_ARG_CHECK(offset_ld >= (modulated ? 27 : 18 * dg), "dcn_sample_nhwc: offset_ld smaller than the offset channels");
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(input) & 15) == 0 && (reinterpret_cast<uintptr_t>(cols) & 15) == 0,
                 "dcn_sample_nhwc: input and cols must be 16-byte aligned");
  const int ho = (height - 1) / stride + 1, wo = (width - 1) / stride + 1;     // 3x3, padding = dilation
  const long long pixels = static_cast<long long>(batch) * ho * wo;
  if (pixels == 0) return MEGA_OK;
  const int cta_pix = max(1, kSampPix / dg);
  const size_t smem = (sizeof(DcnTap) + sizeof(float)) * 9 * dg * cta_pix;
  const long long blocks = (pixels + cta_pix - 1) / cta_pix;
  MEGA_ARG_CHECK(blocks < (1LL << 31), "dcn_sample_nhwc: grid too large");
  const unsigned grid = static_cast<unsigned>(blocks);
  if (format == MEGA_DCN_FP32)
    dcn_sample_nhwc_kernel<MEGA_DCN_FP32><<<grid, kSampThreads, smem, stream>>>(
        input, height, width, channels, dg, cta_pix, offset, offset_ld, modulated, stride, dil, ho, wo, pixels, cols);
  else if (format == MEGA_DCN_FP16)
    dcn_sample_nhwc_kernel<MEGA_DCN_FP16><<<grid, kSampThreads, smem, stream>>>(
        input, height, width, channels, dg, cta_pix, offset, offset_ld, modulated, stride, dil, ho, wo, pixels, cols);
  else
    dcn_sample_nhwc_kernel<MEGA_DCN_SPLIT16><<<grid, kSampThreads, smem, stream>>>(
        input, height, width, channels, dg, cta_pix, offset, offset_ld, modulated, stride, dil, ho, wo, pixels, cols);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_dcn_sample_nhwc(const void* input, int format, int batch, int height, int width, int channels,
                                    const float* offset, int offset_ld, int modulated, int stride, int dil,
                                    void* cols, void* stream_v) {
  return mega_dcn_sample_nhwc_groups(input, format, batch, height, width, channels, 1, offset, offset_ld, modulated,
                                     stride, dil, cols, stream_v);
}
