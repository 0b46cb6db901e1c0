// Memory-bound helpers of the backbone and the window/memory plumbing:
//   * stem im2col (7x7 / stride 2 / pad 3 over the NCHW input image -> K-major GEMM operand),
//     feeding the wgmma GEMM for BaseStem.conv1 (modeling/backbone/resnet.py:347-366);
//   * 3x3 / stride 2 / pad 1 max-pool in NHWC (resnet.py:365);
//   * row gather (replaces the torch.cat of 25-deep deques every frame,
//     detector/generalized_rcnn_mega.py:213-216 and roi_box_feature_extractors.py:674-688);
//   * NCHW <-> NHWC converters for the module-API boundary.
// All are pure bandwidth kernels: 128-bit accesses, grid-stride, one pass.
#include <cuda_fp16.h>
#include "common.cuh"
#include "mega_b200.h"

namespace mega {

// out[n][oh*Wo+ow][k], k = c*49 + r*7 + s for k < 147 (matches weight.view(64,147)), zero for k >= 147
__global__ void stem_im2col_kernel(const float* __restrict__ in, int n_img, int height, int width, int ho, int wo,
                                   int kpad, float* __restrict__ out) {
  const int groups = kpad / 4;
  const long long total = static_cast<long long>(n_img) * ho * wo * groups;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int grp = static_cast<int>(i % groups);
    const long long pix = i / groups;
    const int ow = static_cast<int>(pix % wo);
    const int oh = static_cast<int>((pix / wo) % ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(wo) * ho));
    float v[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int k = grp * 4 + t;
      float val = 0.f;
      if (k < 147) {
        const int c = k / 49, rs = k - c * 49, r = rs / 7, s = rs - r * 7;
        const int ih = oh * 2 - 3 + r, iw = ow * 2 - 3 + s;
        if (ih >= 0 && ih < height && iw >= 0 && iw < width)
          val = __ldg(in + ((static_cast<long long>(n) * 3 + c) * height + ih) * width + iw);
      }
      v[t] = val;
    }
    *reinterpret_cast<float4*>(out + pix * kpad + grp * 4) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

__global__ void maxpool3x3s2_nhwc_kernel(const float* __restrict__ in, int n_img, int height, int width, int channels,
                                         int ho, int wo, float* __restrict__ out) {
  const int cg = channels / 4;
  const long long total = static_cast<long long>(n_img) * ho * wo * cg;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % cg);
    const long long pix = i / cg;
    const int ow = static_cast<int>(pix % wo);
    const int oh = static_cast<int>((pix / wo) % ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(wo) * ho));
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < 3; ++r) {
      const int ih = oh * 2 - 1 + r;
      if (ih < 0 || ih >= height) continue;
      for (int s = 0; s < 3; ++s) {
        const int iw = ow * 2 - 1 + s;
        if (iw < 0 || iw >= width) continue;
        const float4 v = ldg_f4(in + ((static_cast<long long>(n) * height + ih) * width + iw) * channels + c4 * 4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    *reinterpret_cast<float4*>(out + pix * channels + c4 * 4) = m;
  }
}

// dst[didx ? didx[i] : i, :] = src[idx ? idx[i] : i, :] (source index < 0 -> zeros, destination
// index < 0 -> row skipped); row_len multiple of 4
__global__ void gather_rows_kernel(const float* __restrict__ src, long long src_ld, const int* __restrict__ idx,
                                   int n_rows, int row_len, float* __restrict__ dst, long long dst_ld,
                                   const int* __restrict__ didx) {
  const int vec = row_len / 4;
  const long long total = static_cast<long long>(n_rows) * vec;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / vec), c = static_cast<int>(i - static_cast<long long>(r) * vec);
    const int s = idx ? idx[r] : r;
    const int d = didx ? didx[r] : r;
    if (d < 0) continue;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s >= 0) v = ldg_f4(src + static_cast<long long>(s) * src_ld + c * 4);
    *reinterpret_cast<float4*>(dst + static_cast<long long>(d) * dst_ld + c * 4) = v;
  }
}

// same, element-wise, for rows that are not a multiple of 4 floats (e.g. per-frame counters)
__global__ void gather_rows_scalar_kernel(const float* __restrict__ src, long long src_ld, const int* __restrict__ idx,
                                          int n_rows, int row_len, float* __restrict__ dst, long long dst_ld,
                                          const int* __restrict__ didx) {
  const long long total = static_cast<long long>(n_rows) * row_len;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / row_len), c = static_cast<int>(i - static_cast<long long>(r) * row_len);
    const int s = idx ? idx[r] : r;
    const int d = didx ? didx[r] : r;
    if (d < 0) continue;
    dst[static_cast<long long>(d) * dst_ld + c] = (s >= 0) ? src[static_cast<long long>(s) * src_ld + c] : 0.f;
  }
}

// tiled transpose of a [rows, cols] matrix per image (rows*cols floats per image)
__global__ void transpose_kernel(const float* __restrict__ in, int rows, int cols, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const long long img_off = static_cast<long long>(blockIdx.z) * rows * cols;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[j][threadIdx.x] = in[img_off + static_cast<long long>(r) * cols + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[img_off + static_cast<long long>(c) * rows + r] = tile[threadIdx.x][j];
  }
}

// fp16 variants of the two backbone helpers (the fp16-operand engine keeps activations in fp16)
__global__ void stem_im2col_f16_kernel(const float* __restrict__ in, int n_img, int height, int width, int ho, int wo,
                                       int kpad, __half* __restrict__ out) {
  const int groups = kpad / 8;
  const long long total = static_cast<long long>(n_img) * ho * wo * groups;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int grp = static_cast<int>(i % groups);
    const long long pix = i / groups;
    const int ow = static_cast<int>(pix % wo);
    const int oh = static_cast<int>((pix / wo) % ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(wo) * ho));
    float v[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int k = grp * 8 + t;
      float val = 0.f;
      if (k < 147) {
        const int c = k / 49, rs = k - c * 49, r = rs / 7, s = rs - r * 7;
        const int ih = oh * 2 - 3 + r, iw = ow * 2 - 3 + s;
        if (ih >= 0 && ih < height && iw >= 0 && iw < width)
          val = __ldg(in + ((static_cast<long long>(n) * 3 + c) * height + ih) * width + iw);
      }
      v[t] = val;
    }
    *reinterpret_cast<uint4*>(out + pix * kpad + grp * 8) =
        make_uint4(f2_to_h2(v[0], v[1]), f2_to_h2(v[2], v[3]), f2_to_h2(v[4], v[5]), f2_to_h2(v[6], v[7]));
  }
}

__global__ void maxpool3x3s2_nhwc_f16_kernel(const __half* __restrict__ in, int n_img, int height, int width,
                                             int channels, int ho, int wo, __half* __restrict__ out) {
  const int cg = channels / 8;
  const long long total = static_cast<long long>(n_img) * ho * wo * cg;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % cg);
    const long long pix = i / cg;
    const int ow = static_cast<int>(pix % wo);
    const int oh = static_cast<int>((pix / wo) % ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(wo) * ho));
    const __half2 ninf = __float2half2_rn(-INFINITY);
    __half2 m0 = ninf, m1 = ninf, m2 = ninf, m3 = ninf;
    for (int r = 0; r < 3; ++r) {
      const int ih = oh * 2 - 1 + r;
      if (ih < 0 || ih >= height) continue;
      for (int s = 0; s < 3; ++s) {
        const int iw = ow * 2 - 1 + s;
        if (iw < 0 || iw >= width) continue;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(
            in + ((static_cast<long long>(n) * height + ih) * width + iw) * channels + c8 * 8));
        m0 = __hmax2(m0, *reinterpret_cast<const __half2*>(&v.x));
        m1 = __hmax2(m1, *reinterpret_cast<const __half2*>(&v.y));
        m2 = __hmax2(m2, *reinterpret_cast<const __half2*>(&v.z));
        m3 = __hmax2(m3, *reinterpret_cast<const __half2*>(&v.w));
      }
    }
    uint4 o;
    o.x = *reinterpret_cast<uint32_t*>(&m0); o.y = *reinterpret_cast<uint32_t*>(&m1);
    o.z = *reinterpret_cast<uint32_t*>(&m2); o.w = *reinterpret_cast<uint32_t*>(&m3);
    *reinterpret_cast<uint4*>(out + pix * channels + c8 * 8) = o;
  }
}

// NCHW fp32 image -> zero-bordered NHWC (8 channels per pixel: c0..c2 + 5 zeros) [N][H+6][WP][8], WP >= W+8 even:
// the A operand of BaseStem.conv1 (7x7 / stride 2 / pad 3) as a row-slab implicit GEMM -- the 7 taps of one filter
// row are 56 (+8 zero-weighted) contiguous elements, fetched by TMA through an overlapping strided view (no im2col)
template <typename T>
__global__ void stem_prep_kernel(const float* __restrict__ in, int n_img, int height, int width, int wp, T* __restrict__ out) {
  const int hp = height + 6;
  const long long total = static_cast<long long>(n_img) * hp * wp;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % wp) - 3;
    const int y = static_cast<int>((i / wp) % hp) - 3;
    const int n = static_cast<int>(i / (static_cast<long long>(wp) * hp));
    float v[3] = {0.f, 0.f, 0.f};
    if (y >= 0 && y < height && x >= 0 && x < width) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __ldg(in + ((static_cast<long long>(n) * 3 + c) * height + y) * width + x);
    }
    T* o = out + i * 8;
    if (sizeof(T) == 2) {
      *reinterpret_cast<uint4*>(o) = make_uint4(f2_to_h2(v[0], v[1]), f2_to_h2(v[2], 0.f), 0u, 0u);
    } else {
      reinterpret_cast<float4*>(o)[0] = make_float4(v[0], v[1], v[2], 0.f);
      reinterpret_cast<float4*>(o)[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// several independent row copies in ONE launch (blockIdx.y = job): the window / memory plumbing of a frame is a dozen
// tiny gathers whose launch gaps cost more than the bytes they move
constexpr int kMaxCopyJobs = 16;
struct CopyJobs {
  mega_copy_job j[kMaxCopyJobs];
};

__global__ void copy_rows_batch_kernel(const __grid_constant__ CopyJobs jobs) {
  const mega_copy_job& jb = jobs.j[blockIdx.y];
  const float* src = static_cast<const float*>(jb.src);
  float* dst = static_cast<float*>(jb.dst);
  const bool vec = !((jb.row_len & 3) || (jb.src_ld & 3) || (jb.dst_ld & 3) || (reinterpret_cast<uintptr_t>(src) & 15) ||
                     (reinterpret_cast<uintptr_t>(dst) & 15));
  if (vec) {
    const int nv = jb.row_len / 4;
    const long long total = static_cast<long long>(jb.n_rows) * nv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int r = static_cast<int>(i / nv), c = static_cast<int>(i - static_cast<long long>(r) * nv);
      const int s = jb.src_idx ? jb.src_idx[r] : r;
      const int d = jb.dst_idx ? jb.dst_idx[r] : r;
      if (d < 0) continue;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (s >= 0) v = ldg_f4(src + static_cast<long long>(s) * jb.src_ld + c * 4);
      *reinterpret_cast<float4*>(dst + static_cast<long long>(d) * jb.dst_ld + c * 4) = v;
    }
  } else {
    const long long total = static_cast<long long>(jb.n_rows) * jb.row_len;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int r = static_cast<int>(i / jb.row_len), c = static_cast<int>(i - static_cast<long long>(r) * jb.row_len);
      const int s = jb.src_idx ? jb.src_idx[r] : r;
      const int d = jb.dst_idx ? jb.dst_idx[r] : r;
      if (d < 0) continue;
      dst[static_cast<long long>(d) * jb.dst_ld + c] = (s >= 0) ? src[static_cast<long long>(s) * jb.src_ld + c] : 0.f;
    }
  }
}

static int grid_for(long long total, int block) {
  long long b = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

// ---- split-fp16 format (include/mega_b200.h): every aligned group of 32 fp32 values <-> 128 bytes [32 hi halves | 32 lo
// halves]. A team of 8 lanes owns a group: lane l holds values 4l .. 4l+3 (one 16-byte access); the 16-byte chunks of the
// packed row pair the halves of two neighbouring lanes, exchanged by shuffle. In-place conversion is safe: every load of
// a group precedes its stores (same warp instruction order).
__global__ void split16_pack_kernel(const float* __restrict__ src, uint4* __restrict__ dst, long long n_groups) {
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long w = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5; w * 4 < n_groups; w += warps) {
    const long long g = w * 4 + (lane >> 3);
    const bool ok = g < n_groups;
    const int l = lane & 7;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) x = *reinterpret_cast<const float4*>(src + g * 32 + l * 4);
    const uint32_t h0 = f2_to_h2_sat(x.x, x.y), h1 = f2_to_h2_sat(x.z, x.w);
    const float2 b0 = h2_to_f2(h0), b1 = h2_to_f2(h1);
    const uint32_t l0 = f2_to_h2_sat(x.x - b0.x, x.y - b0.y), l1 = f2_to_h2_sat(x.z - b1.x, x.w - b1.y);
    // even lane: writes the hi chunk l/2 = (own hi, partner hi); odd lane: the lo chunk 4 + l/2 = (partner lo, own lo)
    const bool odd = l & 1;
    const uint32_t s0 = odd ? h0 : l0, s1 = odd ? h1 : l1;          // what the partner needs from this lane
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    if (ok) {
      const uint4 o = odd ? make_uint4(r0, r1, l0, l1) : make_uint4(h0, h1, r0, r1);
      dst[g * 8 + (odd ? 4 : 0) + (l >> 1)] = o;
    }
  }
}

__global__ void split16_unpack_kernel(const uint4* __restrict__ src, float* __restrict__ dst, long long n_groups) {
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long w = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5; w * 4 < n_groups; w += warps) {
    const long long g = w * 4 + (lane >> 3);
    const bool ok = g < n_groups;
    const int l = lane & 7;
    const bool odd = l & 1;
    uint4 c = make_uint4(0u, 0u, 0u, 0u);
    if (ok) c = src[g * 8 + (odd ? 4 : 0) + (l >> 1)];     // even: hi of values 8q .. 8q+7, odd: their lo (q = l / 2)
    // even lane keeps values 8q .. 8q+3 (needs the partner's lo first half), odd lane 8q+4 .. 8q+7 (partner's hi second half)
    const uint32_t s0 = odd ? c.x : c.z, s1 = odd ? c.y : c.w;
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    const uint32_t h0 = odd ? r0 : c.x, h1 = odd ? r1 : c.y, l0 = odd ? c.z : r0, l1 = odd ? c.w : r1;
    if (ok) {
      const float2 a0 = h2_to_f2(h0), a1 = h2_to_f2(h1), b0 = h2_to_f2(l0), b1 = h2_to_f2(l1);
      *reinterpret_cast<float4*>(dst + g * 32 + l * 4) = make_float4(a0.x + b0.x, a0.y + b0.y, a1.x + b1.x, a1.y + b1.y);
    }
  }
}

}  // namespace mega

using namespace mega;

extern "C" int mega_stem_im2col(const float* input, int n_img, int height, int width, int kpad, float* out,
                                void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(kpad >= 148 && (kpad & 3) == 0, "stem_im2col: kpad must be a multiple of 4 >= 148");
  const int ho = (height - 1) / 2 + 1, wo = (width - 1) / 2 + 1;
  const long long total = static_cast<long long>(n_img) * ho * wo * (kpad / 4);
  stem_im2col_kernel<<<grid_for(total, 256), 256, 0, stream>>>(input, n_img, height, width, ho, wo, kpad, out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_stem_im2col_f16(const float* input, int n_img, int height, int width, int kpad, void* out,
                                    void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(kpad >= 152 && (kpad & 7) == 0, "stem_im2col_f16: kpad must be a multiple of 8 >= 152");
  const int ho = (height - 1) / 2 + 1, wo = (width - 1) / 2 + 1;
  const long long total = static_cast<long long>(n_img) * ho * wo * (kpad / 8);
  stem_im2col_f16_kernel<<<grid_for(total, 256), 256, 0, stream>>>(input, n_img, height, width, ho, wo, kpad,
                                                                   static_cast<__half*>(out));
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_stem_prep(const float* input, int n_img, int height, int width, int wp, void* out, int f16,
                              void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(wp >= width + 8 && (wp & 1) == 0, "stem_prep: padded width must be even and >= width + 8");
  const long long total = static_cast<long long>(n_img) * (height + 6) * wp;
  if (f16) stem_prep_kernel<__half><<<grid_for(total, 256), 256, 0, stream>>>(input, n_img, height, width, wp, static_cast<__half*>(out));
  else stem_prep_kernel<float><<<grid_for(total, 256), 256, 0, stream>>>(input, n_img, height, width, wp, static_cast<float*>(out));
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_maxpool3x3s2_nhwc_f16(const void* input, int n_img, int height, int width, int channels, void* out,
                                          void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK((channels & 7) == 0, "maxpool_f16: channels must be a multiple of 8");
  const int ho = (height - 1) / 2 + 1, wo = (width - 1) / 2 + 1;
  const long long total = static_cast<long long>(n_img) * ho * wo * (channels / 8);
  maxpool3x3s2_nhwc_f16_kernel<<<grid_for(total, 256), 256, 0, stream>>>(
      static_cast<const __half*>(input), n_img, height, width, channels, ho, wo, static_cast<__half*>(out));
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_maxpool3x3s2_nhwc(const float* input, int n_img, int height, int width, int channels, float* out,
                                      void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK((channels & 3) == 0, "maxpool: channels must be a multiple of 4");
  const int ho = (height - 1) / 2 + 1, wo = (width - 1) / 2 + 1;
  const long long total = static_cast<long long>(n_img) * ho * wo * (channels / 4);
  maxpool3x3s2_nhwc_kernel<<<grid_for(total, 256), 256, 0, stream>>>(input, n_img, height, width, channels, ho, wo,
                                                                     out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_gather_rows(const float* src, long long src_ld, const int* idx, int n_rows, int row_len,
                                float* dst, long long dst_ld, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_rows == 0) return MEGA_OK;
  if ((row_len & 3) || (src_ld & 3) || (dst_ld & 3) || (reinterpret_cast<uintptr_t>(src) & 15) ||
      (reinterpret_cast<uintptr_t>(dst) & 15)) {
    gather_rows_scalar_kernel<<<grid_for(static_cast<long long>(n_rows) * row_len, 256), 256, 0, stream>>>(
        src, src_ld, idx, n_rows, row_len, dst, dst_ld, nullptr);
    MEGA_CUDA_CHECK(cudaGetLastError());
    return MEGA_OK;
  }
  const long long total = static_cast<long long>(n_rows) * (row_len / 4);
  gather_rows_kernel<<<grid_for(total, 256), 256, 0, stream>>>(src, src_ld, idx, n_rows, row_len, dst, dst_ld,
                                                               nullptr);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_copy_rows(const float* src, long long src_ld, const int* src_idx, float* dst, long long dst_ld,
                              const int* dst_idx, int n_rows, int row_len, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_rows == 0) return MEGA_OK;
  if ((row_len & 3) || (src_ld & 3) || (dst_ld & 3) || (reinterpret_cast<uintptr_t>(src) & 15) ||
      (reinterpret_cast<uintptr_t>(dst) & 15)) {
    gather_rows_scalar_kernel<<<grid_for(static_cast<long long>(n_rows) * row_len, 256), 256, 0, stream>>>(
        src, src_ld, src_idx, n_rows, row_len, dst, dst_ld, dst_idx);
    MEGA_CUDA_CHECK(cudaGetLastError());
    return MEGA_OK;
  }
  const long long total = static_cast<long long>(n_rows) * (row_len / 4);
  gather_rows_kernel<<<grid_for(total, 256), 256, 0, stream>>>(src, src_ld, src_idx, n_rows, row_len, dst, dst_ld,
                                                               dst_idx);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

// per image: in [rows, cols] -> out [cols, rows]; NCHW->NHWC is rows=C, cols=H*W
extern "C" int mega_transpose_2d(const float* input, int n_img, int rows, int cols, float* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_img == 0 || rows == 0 || cols == 0) return MEGA_OK;
  dim3 grid((cols + 31) / 32, (rows + 31) / 32, n_img), block(32, 8);
  transpose_kernel<<<grid, block, 0, stream>>>(input, rows, cols, out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_copy_rows_batch(const mega_copy_job* jobs_host, int n_jobs, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(jobs_host != nullptr && n_jobs >= 0 && n_jobs <= kMaxCopyJobs, "copy_rows_batch: at most %d jobs", kMaxCopyJobs);
  if (n_jobs == 0) return MEGA_OK;
  CopyJobs jobs;
  long long most = 1;
  for (int i = 0; i < n_jobs; ++i) {
    jobs.j[i] = jobs_host[i];
    const long long words = static_cast<long long>(jobs_host[i].n_rows) * jobs_host[i].row_len;
    if (words / 4 > most) most = words / 4;
  }
  for (int i = n_jobs; i < kMaxCopyJobs; ++i) jobs.j[i] = jobs_host[0];
  dim3 grid(grid_for(most, 256) > 132 ? 132 : grid_for(most, 256), n_jobs);
  copy_rows_batch_kernel<<<grid, 256, 0, stream>>>(jobs);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

/* fp32 -> split-fp16 (include/mega_b200.h) over n_values contiguous values (a multiple of 32); dst == src converts in place */
extern "C" int mega_split16_pack(const float* src, void* dst, long long n_values, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(n_values >= 0 && (n_values & 31) == 0, "split16_pack: n_values must be a multiple of 32 (got %lld)", n_values);
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(src) & 127) == 0 && (reinterpret_cast<uintptr_t>(dst) & 127) == 0,
                 "split16_pack: tensors must be 128-byte aligned");
  if (n_values == 0) return MEGA_OK;
  split16_pack_kernel<<<grid_for(n_values / 4, 256), 256, 0, stream>>>(src, static_cast<uint4*>(dst), n_values / 32);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_split16_unpack(const void* src, float* dst, long long n_values, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(n_values >= 0 && (n_values & 31) == 0, "split16_unpack: n_values must be a multiple of 32 (got %lld)", n_values);
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(src) & 127) == 0 && (reinterpret_cast<uintptr_t>(dst) & 127) == 0,
                 "split16_unpack: tensors must be 128-byte aligned");
  if (n_values == 0) return MEGA_OK;
  split16_unpack_kernel<<<grid_for(n_values / 4, 256), 256, 0, stream>>>(static_cast<const uint4*>(src), dst, n_values / 32);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
