// ROIAlign forward (mega_core/csrc/cuda/ROIAlign_cuda.cu:16-122, cpu/ROIAlign_cpu.cpp:17-219).
//
// Two layouts:
//   * mega_roi_align_forward_nchw -- the `_C.roi_align_forward` contract: NCHW fp32 in,
//     [K,C,ph,pw] out, one thread per output element (same mapping as the reference kernel);
//   * mega_roi_align_forward_nhwc -- the engine's layout: NHWC feature map in, [K, ph*pw, C] out
//     (bin-major, channel-minor). One CTA per (roi, bin); threads span channels with 128-bit
//     loads, so every bilinear corner is one fully coalesced row read and the output row feeds
//     the l_fcs[0] GEMM as its K-major A operand without a transpose.
// Arithmetic is written with explicit round-to-nearest ops (no FMA contraction) in the
// reference's association order, so results are bit-identical to the C oracle.
#include <cuda_fp16.h>
#include <cstdlib>
#include "common.cuh"
#include "mega_b200.h"

namespace mega {

struct Bilinear {
  int y_low, y_high, x_low, x_high;
  float w1, w2, w3, w4;
  bool empty;
};

__device__ __forceinline__ Bilinear bilinear_setup(int height, int width, float y, float x) {
  Bilinear b;
  b.empty = (y < -1.0f || y > static_cast<float>(height) || x < -1.0f || x > static_cast<float>(width));
  if (b.empty) {
    b.y_low = b.y_high = b.x_low = b.x_high = 0;
    b.w1 = b.w2 = b.w3 = b.w4 = 0.f;
    return b;
  }
  if (y <= 0) y = 0;
  if (x <= 0) x = 0;
  int y_low = static_cast<int>(y), x_low = static_cast<int>(x), y_high, x_high;
  if (y_low >= height - 1) {
    y_high = y_low = height - 1;
    y = static_cast<float>(y_low);
  } else {
    y_high = y_low + 1;
  }
  if (x_low >= width - 1) {
    x_high = x_low = width - 1;
    x = static_cast<float>(x_low);
  } else {
    x_high = x_low + 1;
  }
  const float ly = __fsub_rn(y, static_cast<float>(y_low)), lx = __fsub_rn(x, static_cast<float>(x_low));
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  b.y_low = y_low; b.y_high = y_high; b.x_low = x_low; b.x_high = x_high;
  b.w1 = __fmul_rn(hy, hx); b.w2 = __fmul_rn(hy, lx); b.w3 = __fmul_rn(ly, hx); b.w4 = __fmul_rn(ly, lx);
  return b;
}

__device__ __forceinline__ float blend(const Bilinear& b, float v1, float v2, float v3, float v4) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(b.w1, v1), __fmul_rn(b.w2, v2)), __fmul_rn(b.w3, v3)),
                   __fmul_rn(b.w4, v4));
}

struct RoiGeom {
  float start_w, start_h, bin_w, bin_h;
  int grid_w, grid_h, batch;
};

__device__ __forceinline__ RoiGeom roi_geom(const float* roi, float scale, int ph, int pw, int sampling_ratio) {
  RoiGeom g;
  g.batch = static_cast<int>(roi[0]);
  g.start_w = __fmul_rn(roi[1], scale);
  g.start_h = __fmul_rn(roi[2], scale);
  const float end_w = __fmul_rn(roi[3], scale), end_h = __fmul_rn(roi[4], scale);
  const float roi_w = fmaxf(__fsub_rn(end_w, g.start_w), 1.f);
  const float roi_h = fmaxf(__fsub_rn(end_h, g.start_h), 1.f);
  g.bin_h = __fdiv_rn(roi_h, static_cast<float>(ph));
  g.bin_w = __fdiv_rn(roi_w, static_cast<float>(pw));
  g.grid_h = sampling_ratio > 0 ? sampling_ratio : static_cast<int>(ceilf(__fdiv_rn(roi_h, static_cast<float>(ph))));
  g.grid_w = sampling_ratio > 0 ? sampling_ratio : static_cast<int>(ceilf(__fdiv_rn(roi_w, static_cast<float>(pw))));
  return g;
}

__device__ __forceinline__ float sample_coord(float start, int p, float bin, int i, int grid) {
  // start + p*bin + (i + .5f) * bin / grid   (ROIAlign_cuda.cu:106-110)
  return __fadd_rn(__fadd_rn(start, __fmul_rn(static_cast<float>(p), bin)),
                   __fdiv_rn(__fmul_rn(static_cast<float>(i) + .5f, bin), static_cast<float>(grid)));
}

__global__ void roi_align_nchw_kernel(const float* __restrict__ in, int channels, int height, int width,
                                      const float* __restrict__ rois, long long total, float scale, int ph, int pw,
                                      int sampling_ratio, float* __restrict__ out) {
  for (long long index = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; index < total;
       index += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pwi = static_cast<int>(index % pw);
    const int phi = static_cast<int>((index / pw) % ph);
    const int c = static_cast<int>((index / pw / ph) % channels);
    const long long n = index / pw / ph / channels;
    const RoiGeom g = roi_geom(rois + n * 5, scale, ph, pw, sampling_ratio);
    const float* plane = in + (static_cast<long long>(g.batch) * channels + c) * height * width;
    const float count = static_cast<float>(g.grid_h * g.grid_w);
    float acc = 0.f;
    for (int iy = 0; iy < g.grid_h; ++iy) {
      const float y = sample_coord(g.start_h, phi, g.bin_h, iy, g.grid_h);
      for (int ix = 0; ix < g.grid_w; ++ix) {
        const float x = sample_coord(g.start_w, pwi, g.bin_w, ix, g.grid_w);
        const Bilinear b = bilinear_setup(height, width, y, x);
        float val = 0.f;
        if (!b.empty) {
          val = blend(b, plane[b.y_low * width + b.x_low], plane[b.y_low * width + b.x_high],
                      plane[b.y_high * width + b.x_low], plane[b.y_high * width + b.x_high]);
        }
        acc = __fadd_rn(acc, val);
      }
    }
    out[index] = __fdiv_rn(acc, count);
  }
}

// ---- 16-byte channel vectors of the NHWC kernels: 4 floats or 8 halves; arithmetic always in fp32
template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void unpack(const uint4& r, float (&v)[4]) {
    v[0] = __uint_as_float(r.x); v[1] = __uint_as_float(r.y); v[2] = __uint_as_float(r.z); v[3] = __uint_as_float(r.w);
  }
  static __device__ __forceinline__ uint4 pack(const float (&v)[4]) {
    return make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3]));
  }
};
template <> struct Vec16<__half> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack(const uint4& r, float (&v)[8]) {
    const float2 a = h2_to_f2(r.x), b = h2_to_f2(r.y), c = h2_to_f2(r.z), d = h2_to_f2(r.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  }
  static __device__ __forceinline__ uint4 pack(const float (&v)[8]) {
    return make_uint4(f2_to_h2(v[0], v[1]), f2_to_h2(v[2], v[3]), f2_to_h2(v[4], v[5]), f2_to_h2(v[6], v[7]));
  }
};
__device__ __forceinline__ uint4 ldg_u4(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// grid = (ph*pw, K); block = 256 threads, each thread owns 16-byte channel groups.
template <typename T>
__global__ void __launch_bounds__(256)
roi_align_nhwc_kernel(const T* __restrict__ in, int channels, int height, int width, long long in_img_stride,
                      const float* __restrict__ rois, int roi_ld, int roi_box_off, const int* __restrict__ roi_batch,
                      float scale, int ph, int pw, int sampling_ratio, T* __restrict__ out,
                      long long out_roi_stride) {
  constexpr int V = Vec16<T>::N;
  const int bin = blockIdx.x;
  const int n = blockIdx.y;
  const int phi = bin / pw, pwi = bin - phi * pw;
  float roi5[5];
  roi5[0] = roi_batch ? static_cast<float>(roi_batch[n]) : 0.f;
  const float* rb = rois + static_cast<long long>(n) * roi_ld + roi_box_off;
  if (roi_box_off < 0) {  // packed [K,5] (batch, x1, y1, x2, y2)
    rb = rois + static_cast<long long>(n) * roi_ld;
    roi5[0] = rb[0];
    rb += 1;
  }
  roi5[1] = rb[0]; roi5[2] = rb[1]; roi5[3] = rb[2]; roi5[4] = rb[3];
  const RoiGeom g = roi_geom(roi5, scale, ph, pw, sampling_ratio);
  const T* img = in + static_cast<long long>(g.batch) * in_img_stride;
  const float count = static_cast<float>(g.grid_h * g.grid_w);
  T* orow = out + static_cast<long long>(n) * out_roi_stride + static_cast<long long>(bin) * channels;
  for (int c = threadIdx.x * V; c < channels; c += blockDim.x * V) {
    float acc[V];
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = 0.f;
    for (int iy = 0; iy < g.grid_h; ++iy) {
      const float y = sample_coord(g.start_h, phi, g.bin_h, iy, g.grid_h);
      for (int ix = 0; ix < g.grid_w; ++ix) {
        const float x = sample_coord(g.start_w, pwi, g.bin_w, ix, g.grid_w);
        const Bilinear b = bilinear_setup(height, width, y, x);
        if (b.empty) continue;  // adds exactly 0 in the reference
        float v1[V], v2[V], v3[V], v4[V];
        Vec16<T>::unpack(ldg_u4(img + (static_cast<long long>(b.y_low) * width + b.x_low) * channels + c), v1);
        Vec16<T>::unpack(ldg_u4(img + (static_cast<long long>(b.y_low) * width + b.x_high) * channels + c), v2);
        Vec16<T>::unpack(ldg_u4(img + (static_cast<long long>(b.y_high) * width + b.x_low) * channels + c), v3);
        Vec16<T>::unpack(ldg_u4(img + (static_cast<long long>(b.y_high) * width + b.x_high) * channels + c), v4);
#pragma unroll
        for (int e = 0; e < V; ++e) acc[e] = __fadd_rn(acc[e], blend(b, v1[e], v2[e], v3[e], v4[e]));
      }
    }
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = __fdiv_rn(acc[e], count);
    *reinterpret_cast<uint4*>(orow + c) = Vec16<T>::pack(acc);
  }
}

// Same arithmetic, less L2 traffic: one CTA per (roi, 256-byte channel slice) first copies the cells the roi can
// touch (rows r0..r1 x cols c0..c1 of the map, 256 B per cell) into shared memory, then all 49 bins sample from
// there; neighbouring samples share corners, so each cell is fetched once per slice instead of up to ~8 times. ROIs
// whose footprint exceeds the shared-memory budget (whole-image boxes) read global memory directly.
constexpr int kRoiSliceBytes = 256;      // channel bytes per CTA: 64 floats / 128 halves
constexpr int kRoiMaxCells = 192;        // 192 cells x 256 B = 48 KB per CTA (4 CTAs per SM)

template <typename T>
__global__ void __launch_bounds__(256)
roi_align_nhwc_cached_kernel(const T* __restrict__ in, int channels, int height, int width, long long in_img_stride,
                             const float* __restrict__ rois, int roi_ld, int roi_box_off,
                             const int* __restrict__ roi_batch, float scale, int ph, int pw, int sampling_ratio,
                             T* __restrict__ out, long long out_roi_stride) {
  constexpr int V = Vec16<T>::N;
  constexpr int kSlice = kRoiSliceBytes / static_cast<int>(sizeof(T));
  extern __shared__ uint4 cell_s[];   // [cells][16] 16-byte vectors
  const int slice = blockIdx.x;
  const int n = blockIdx.y;
  float roi5[5];
  roi5[0] = roi_batch ? static_cast<float>(roi_batch[n]) : 0.f;
  const float* rb = rois + static_cast<long long>(n) * roi_ld + roi_box_off;
  if (roi_box_off < 0) {
    rb = rois + static_cast<long long>(n) * roi_ld;
    roi5[0] = rb[0];
    rb += 1;
  }
  roi5[1] = rb[0]; roi5[2] = rb[1]; roi5[3] = rb[2]; roi5[4] = rb[3];
  const RoiGeom g = roi_geom(roi5, scale, ph, pw, sampling_ratio);
  const T* img = in + static_cast<long long>(g.batch) * in_img_stride + slice * kSlice;
  // footprint of every sample this roi can take (after the reference's clamping of y, x to the map)
  const float end_h = __fadd_rn(g.start_h, __fmul_rn(g.bin_h, static_cast<float>(ph)));
  const float end_w = __fadd_rn(g.start_w, __fmul_rn(g.bin_w, static_cast<float>(pw)));
  int r0 = static_cast<int>(floorf(fmaxf(g.start_h, 0.f))), r1 = static_cast<int>(floorf(fmaxf(end_h, 0.f))) + 1;
  int c0 = static_cast<int>(floorf(fmaxf(g.start_w, 0.f))), c1 = static_cast<int>(floorf(fmaxf(end_w, 0.f))) + 1;
  r0 = min(max(r0, 0), height - 1); r1 = min(max(r1, 0), height - 1);
  c0 = min(max(c0, 0), width - 1); c1 = min(max(c1, 0), width - 1);
  const int rh = r1 - r0 + 1, rw = c1 - c0 + 1;
  const bool cached = (rh * rw <= kRoiMaxCells);
  if (cached) {
    for (int i = threadIdx.x; i < rh * rw * 16; i += blockDim.x) {
      const int cell = i >> 4, q = i & 15;
      const int rr = cell / rw, cc = cell - rr * rw;
      cell_s[i] = ldg_u4(img + (static_cast<long long>(r0 + rr) * width + (c0 + cc)) * channels + q * V);
    }
  }
  __syncthreads();
  const int q = threadIdx.x & 15;
  const float count = static_cast<float>(g.grid_h * g.grid_w);
  T* obase = out + static_cast<long long>(n) * out_roi_stride + slice * kSlice + q * V;
  for (int bin = threadIdx.x >> 4; bin < ph * pw; bin += blockDim.x >> 4) {
    const int phi = bin / pw, pwi = bin - phi * pw;
    float acc[V];
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = 0.f;
    for (int iy = 0; iy < g.grid_h; ++iy) {
      const float y = sample_coord(g.start_h, phi, g.bin_h, iy, g.grid_h);
      for (int ix = 0; ix < g.grid_w; ++ix) {
        const float x = sample_coord(g.start_w, pwi, g.bin_w, ix, g.grid_w);
        const Bilinear b = bilinear_setup(height, width, y, x);
        if (b.empty) continue;
        uint4 r1v, r2v, r3v, r4v;
        const bool inside = cached && b.y_low >= r0 && b.y_high <= r1 && b.x_low >= c0 && b.x_high <= c1;
        if (inside) {
          r1v = cell_s[((b.y_low - r0) * rw + (b.x_low - c0)) * 16 + q];
          r2v = cell_s[((b.y_low - r0) * rw + (b.x_high - c0)) * 16 + q];
          r3v = cell_s[((b.y_high - r0) * rw + (b.x_low - c0)) * 16 + q];
          r4v = cell_s[((b.y_high - r0) * rw + (b.x_high - c0)) * 16 + q];
        } else {
          r1v = ldg_u4(img + (static_cast<long long>(b.y_low) * width + b.x_low) * channels + q * V);
          r2v = ldg_u4(img + (static_cast<long long>(b.y_low) * width + b.x_high) * channels + q * V);
          r3v = ldg_u4(img + (static_cast<long long>(b.y_high) * width + b.x_low) * channels + q * V);
          r4v = ldg_u4(img + (static_cast<long long>(b.y_high) * width + b.x_high) * channels + q * V);
        }
        float v1[V], v2[V], v3[V], v4[V];
        Vec16<T>::unpack(r1v, v1); Vec16<T>::unpack(r2v, v2); Vec16<T>::unpack(r3v, v3); Vec16<T>::unpack(r4v, v4);
#pragma unroll
        for (int e = 0; e < V; ++e) acc[e] = __fadd_rn(acc[e], blend(b, v1[e], v2[e], v3[e], v4[e]));
      }
    }
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = __fdiv_rn(acc[e], count);
    *reinterpret_cast<uint4*>(obase + static_cast<long long>(bin) * channels) = Vec16<T>::pack(acc);
  }
}

// ---- fp16 fast path (the fp16-operand engine): same sampling geometry, but (i) the bilinear set-up is separable, so the
// CTA computes it ONCE per roi -- 7 x grid_h row entries and 7 x grid_w column entries in shared memory -- instead of once
// per (bin, sample, channel group); (ii) the blend uses fused multiply-adds in fp32 (results are rounded to fp16 at the
// store anyway, so the bit-exact association order of the fp32 kernels buys nothing here).
struct AxisSample {
  int lo, hi;       // clamped cell indices; -1 when the sample lies outside [-1, size] (contributes nothing)
  float wlo, whi;   // weights of the two cells
};
constexpr int kRoiMaxGrid = 8;   // samples per bin and axis handled by the fast path (roi extent up to 8*7 cells)

__device__ __forceinline__ AxisSample axis_sample(float c, int size) {
  AxisSample a;
  if (c < -1.0f || c > static_cast<float>(size)) {   // the reference adds exactly 0 for such samples
    a.lo = a.hi = -1;
    a.wlo = a.whi = 0.f;
    return a;
  }
  if (c <= 0) c = 0;
  int lo = static_cast<int>(c), hi;
  if (lo >= size - 1) {
    hi = lo = size - 1;
    c = static_cast<float>(lo);
  } else {
    hi = lo + 1;
  }
  const float l = c - static_cast<float>(lo);
  a.lo = lo; a.hi = hi; a.wlo = 1.f - l; a.whi = l;
  return a;
}

__global__ void __launch_bounds__(256)
roi_align_nhwc_f16_fast_kernel(const __half* __restrict__ in, int channels, int height, int width, long long in_img_stride,
                               const float* __restrict__ rois, int roi_ld, int roi_box_off,
                               const int* __restrict__ roi_batch, float scale, int ph, int pw, int sampling_ratio,
                               __half* __restrict__ out, long long out_roi_stride) {
  constexpr int kSlice = kRoiSliceBytes / 2;     // 128 channels per CTA
  extern __shared__ uint4 cell_s[];              // [cells][16] 16-byte vectors
  __shared__ AxisSample ys[7 * kRoiMaxGrid], xs[7 * kRoiMaxGrid];
  const int slice = blockIdx.x;
  const int n = blockIdx.y;
  float roi5[5];
  roi5[0] = roi_batch ? static_cast<float>(roi_batch[n]) : 0.f;
  const float* rb = rois + static_cast<long long>(n) * roi_ld + roi_box_off;
  if (roi_box_off < 0) {
    rb = rois + static_cast<long long>(n) * roi_ld;
    roi5[0] = rb[0];
    rb += 1;
  }
  roi5[1] = rb[0]; roi5[2] = rb[1]; roi5[3] = rb[2]; roi5[4] = rb[3];
  const RoiGeom g = roi_geom(roi5, scale, ph, pw, sampling_ratio);
  const __half* img = in + static_cast<long long>(g.batch) * in_img_stride + slice * kSlice;
  const float end_h = __fadd_rn(g.start_h, __fmul_rn(g.bin_h, static_cast<float>(ph)));
  const float end_w = __fadd_rn(g.start_w, __fmul_rn(g.bin_w, static_cast<float>(pw)));
  int r0 = static_cast<int>(floorf(fmaxf(g.start_h, 0.f))), r1 = static_cast<int>(floorf(fmaxf(end_h, 0.f))) + 1;
  int c0 = static_cast<int>(floorf(fmaxf(g.start_w, 0.f))), c1 = static_cast<int>(floorf(fmaxf(end_w, 0.f))) + 1;
  r0 = min(max(r0, 0), height - 1); r1 = min(max(r1, 0), height - 1);
  c0 = min(max(c0, 0), width - 1); c1 = min(max(c1, 0), width - 1);
  const int rh = r1 - r0 + 1, rw = c1 - c0 + 1;
  const bool cached = (rh * rw <= kRoiMaxCells);
  if (cached) {
    for (int i = threadIdx.x; i < rh * rw * 16; i += blockDim.x) {
      const int cell = i >> 4, q = i & 15;
      const int rr = cell / rw, cc = cell - rr * rw;
      cell_s[i] = ldg_u4(img + (static_cast<long long>(r0 + rr) * width + (c0 + cc)) * channels + q * 8);
    }
  }
  // rois with more than kRoiMaxGrid samples per bin and axis (boxes far larger than the map) compute the entries inline
  const bool tabled = g.grid_h <= kRoiMaxGrid && g.grid_w <= kRoiMaxGrid;
  if (tabled) {
    for (int i = threadIdx.x; i < ph * g.grid_h; i += blockDim.x)
      ys[i] = axis_sample(sample_coord(g.start_h, i / g.grid_h, g.bin_h, i % g.grid_h, g.grid_h), height);
    for (int i = threadIdx.x; i < pw * g.grid_w; i += blockDim.x)
      xs[i] = axis_sample(sample_coord(g.start_w, i / g.grid_w, g.bin_w, i % g.grid_w, g.grid_w), width);
  }
  __syncthreads();
  const int q = threadIdx.x & 15;
  const float inv_count = 1.0f / static_cast<float>(g.grid_h * g.grid_w);
  __half* obase = out + static_cast<long long>(n) * out_roi_stride + slice * kSlice + q * 8;
  for (int bin = threadIdx.x >> 4; bin < ph * pw; bin += blockDim.x >> 4) {
    const int phi = bin / pw, pwi = bin - phi * pw;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int iy = 0; iy < g.grid_h; ++iy) {
      const AxisSample ay = tabled ? ys[phi * g.grid_h + iy]
                                   : axis_sample(sample_coord(g.start_h, phi, g.bin_h, iy, g.grid_h), height);
      if (ay.lo < 0) continue;
      for (int ix = 0; ix < g.grid_w; ++ix) {
        const AxisSample ax = tabled ? xs[pwi * g.grid_w + ix]
                                     : axis_sample(sample_coord(g.start_w, pwi, g.bin_w, ix, g.grid_w), width);
        if (ax.lo < 0) continue;
        const float w1 = ay.wlo * ax.wlo, w2 = ay.wlo * ax.whi, w3 = ay.whi * ax.wlo, w4 = ay.whi * ax.whi;
        uint4 v1, v2, v3, v4;
        if (cached) {     // the footprint covers every clamped sample cell by construction
          v1 = cell_s[((ay.lo - r0) * rw + (ax.lo - c0)) * 16 + q];
          v2 = cell_s[((ay.lo - r0) * rw + (ax.hi - c0)) * 16 + q];
          v3 = cell_s[((ay.hi - r0) * rw + (ax.lo - c0)) * 16 + q];
          v4 = cell_s[((ay.hi - r0) * rw + (ax.hi - c0)) * 16 + q];
        } else {
          v1 = ldg_u4(img + (static_cast<long long>(ay.lo) * width + ax.lo) * channels + q * 8);
          v2 = ldg_u4(img + (static_cast<long long>(ay.lo) * width + ax.hi) * channels + q * 8);
          v3 = ldg_u4(img + (static_cast<long long>(ay.hi) * width + ax.lo) * channels + q * 8);
          v4 = ldg_u4(img + (static_cast<long long>(ay.hi) * width + ax.hi) * channels + q * 8);
        }
        const uint32_t* p1 = &v1.x; const uint32_t* p2 = &v2.x; const uint32_t* p3 = &v3.x; const uint32_t* p4 = &v4.x;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 a = h2_to_f2(p1[e]), b = h2_to_f2(p2[e]), c = h2_to_f2(p3[e]), d = h2_to_f2(p4[e]);
          acc[2 * e] = fmaf(w4, d.x, fmaf(w3, c.x, fmaf(w2, b.x, fmaf(w1, a.x, acc[2 * e]))));
          acc[2 * e + 1] = fmaf(w4, d.y, fmaf(w3, c.y, fmaf(w2, b.y, fmaf(w1, a.y, acc[2 * e + 1]))));
        }
      }
    }
    uint4 o;
    o.x = f2_to_h2(acc[0] * inv_count, acc[1] * inv_count); o.y = f2_to_h2(acc[2] * inv_count, acc[3] * inv_count);
    o.z = f2_to_h2(acc[4] * inv_count, acc[5] * inv_count); o.w = f2_to_h2(acc[6] * inv_count, acc[7] * inv_count);
    *reinterpret_cast<uint4*>(obase + static_cast<long long>(bin) * channels) = o;
  }
}

// ---- fp16 separable path (feature maps up to 64 x 64 cells). The samples of a bin form a grid_h x grid_w lattice and a
// sample's four bilinear weights are (row weight) x (column weight), so the sum over the lattice factorises:
//     out[ph, pw] = 1/count * sum_y Wy[ph][y] * ( sum_x Wx[pw][x] * f[y, x] ),
// Wy[ph][y] = total weight the grid_h sample rows of bin-row ph put on map row y (same for columns). Every cell of the
// roi's footprint is then read ~once per bin-row it touches (not 4 times per sample) and costs one FMA per channel in
// the row pass: rois larger than the shared-memory cache of the kernel above - the common case for VID objects - get
// ~4x fewer loads and FMAs. Same skipping (samples outside [-1, size]) and clamping rules, applied per axis.
constexpr int kSepMaxDim = 64;
constexpr int kSepMaxGrid = 16;    // samples per bin and axis kept in the coordinate tables (else computed inline)
// MEGA_B200_ROI_SEPARABLE=0 keeps the per-sample kernel above for every roi
static const bool g_roi_separable = [] {
  const char* e = getenv("MEGA_B200_ROI_SEPARABLE");
  return e != nullptr ? e[0] != '0' : true;     // default ON: 181 -> 130 us (rois of 40-360 px), 583 -> 268 us (200-900 px), tools/roi_probe.py on a B200
}();

// SPLIT: the map and the result are split-fp16 tensors (include/mega_b200.h; the strict engine): a thread's 8 channels are
// one 16-byte chunk of hi halves plus the 16-byte chunk of their lo halves 64 bytes further, in and out.
template <bool SPLIT>
struct SepIo {
  static constexpr int kEB = SPLIT ? 4 : 2;      // bytes per value
  // byte offset of thread q's 8 channels inside the 128-channel slice of a pixel
  static __device__ __forceinline__ int chunk_off(int q) { return SPLIT ? (q >> 2) * 128 + (q & 3) * 16 : q * 16; }
  static __device__ __forceinline__ void load8(const char* p, float (&v)[8]) {
    const uint4 h = ldg_u4(p);
    const uint32_t* ph_ = &h.x;
    if (SPLIT) {
      const uint4 l = ldg_u4(p + 64);
      const uint32_t* pl = &l.x;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = h2_to_f2(ph_[e]), b = h2_to_f2(pl[e]);
        v[2 * e] = a.x + b.x;
        v[2 * e + 1] = a.y + b.y;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = h2_to_f2(ph_[e]);
        v[2 * e] = a.x;
        v[2 * e + 1] = a.y;
      }
    }
  }
  static __device__ __forceinline__ void store8(char* p, const float (&v)[8]) {
    if (SPLIT) {
      uint32_t hh[4], ll[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        hh[e] = f2_to_h2_sat(v[2 * e], v[2 * e + 1]);
        const float2 back = h2_to_f2(hh[e]);
        ll[e] = f2_to_h2_sat(v[2 * e] - back.x, v[2 * e + 1] - back.y);
      }
      *reinterpret_cast<uint4*>(p) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
      *reinterpret_cast<uint4*>(p + 64) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
    } else {
      *reinterpret_cast<uint4*>(p) = make_uint4(f2_to_h2(v[0], v[1]), f2_to_h2(v[2], v[3]), f2_to_h2(v[4], v[5]), f2_to_h2(v[6], v[7]));
    }
  }
};

template <bool SPLIT>
__global__ void __launch_bounds__(256)
roi_align_nhwc_sep_kernel(const void* __restrict__ in_v, int channels, int height, int width, long long in_img_stride,
                          const float* __restrict__ rois, int roi_ld, int roi_box_off,
                          const int* __restrict__ roi_batch, float scale, int ph, int pw, int sampling_ratio,
                          void* __restrict__ out_v, long long out_roi_stride) {
  using Io = SepIo<SPLIT>;
  constexpr int kEB = Io::kEB;
  constexpr int kSlice = 128;                    // channels per CTA
  __shared__ float Wy[7][kSepMaxDim], Wx[7][kSepMaxDim];
  __shared__ AxisSample ys[7 * kSepMaxGrid], xs[7 * kSepMaxGrid];
  __shared__ int ylo[7], yhi[7], xlo[7], xhi[7];
  __shared__ float4 U[kSepMaxDim][kSlice / 4];   // row-weighted partial sums, fp32: [x][128 channels]
  const int slice = blockIdx.x;
  const int n = blockIdx.y;
  const int tid = threadIdx.x;
  float roi5[5];
  roi5[0] = roi_batch ? static_cast<float>(roi_batch[n]) : 0.f;
  const float* rb = rois + static_cast<long long>(n) * roi_ld + roi_box_off;
  if (roi_box_off < 0) {
    rb = rois + static_cast<long long>(n) * roi_ld;
    roi5[0] = rb[0];
    rb += 1;
  }
  roi5[1] = rb[0]; roi5[2] = rb[1]; roi5[3] = rb[2]; roi5[4] = rb[3];
  const RoiGeom g = roi_geom(roi5, scale, ph, pw, sampling_ratio);
  const char* img = static_cast<const char*>(in_v) + (static_cast<long long>(g.batch) * in_img_stride + slice * kSlice) * kEB;
  if (tid < 7) {
    ylo[tid] = kSepMaxDim; yhi[tid] = -1;
    xlo[tid] = kSepMaxDim; xhi[tid] = -1;
  }
  __syncthreads();
  // 1. per-axis weight tables. First every sample coordinate once (7 x grid entries per axis), then one thread per
  //    (bin index, cell) adds up the samples that touch its cell, in sample order (deterministic, no float atomics).
  const bool tabled = g.grid_h <= kSepMaxGrid && g.grid_w <= kSepMaxGrid;
  if (tabled) {
    for (int i = tid; i < ph * g.grid_h; i += blockDim.x)
      ys[i] = axis_sample(sample_coord(g.start_h, i / g.grid_h, g.bin_h, i % g.grid_h, g.grid_h), height);
    for (int i = tid; i < pw * g.grid_w; i += blockDim.x)
      xs[i] = axis_sample(sample_coord(g.start_w, i / g.grid_w, g.bin_w, i % g.grid_w, g.grid_w), width);
    __syncthreads();
  }
  for (int i = tid; i < ph * height; i += blockDim.x) {
    const int p = i / height, r = i - p * height;
    float wsum = 0.f;
    for (int iy = 0; iy < g.grid_h; ++iy) {
      const AxisSample a = tabled ? ys[p * g.grid_h + iy]
                                  : axis_sample(sample_coord(g.start_h, p, g.bin_h, iy, g.grid_h), height);
      if (a.lo == r) wsum += a.wlo;
      if (a.hi == r) wsum += a.whi;
    }
    Wy[p][r] = wsum;
    if (wsum != 0.f) {
      atomicMin(&ylo[p], r);
      atomicMax(&yhi[p], r);
    }
  }
  for (int i = tid; i < pw * width; i += blockDim.x) {
    const int p = i / width, c = i - p * width;
    float wsum = 0.f;
    for (int ix = 0; ix < g.grid_w; ++ix) {
      const AxisSample a = tabled ? xs[p * g.grid_w + ix]
                                  : axis_sample(sample_coord(g.start_w, p, g.bin_w, ix, g.grid_w), width);
      if (a.lo == c) wsum += a.wlo;
      if (a.hi == c) wsum += a.whi;
    }
    Wx[p][c] = wsum;
    if (wsum != 0.f) {
      atomicMin(&xlo[p], c);
      atomicMax(&xhi[p], c);
    }
  }
  __syncthreads();
  int c_first = kSepMaxDim, c_last = -1;          // columns any bin-column needs
  for (int p = 0; p < pw; ++p) {
    c_first = min(c_first, xlo[p]);
    c_last = max(c_last, xhi[p]);
  }
  const int q = tid & 15, worker = tid >> 4;
  const float inv_count = 1.0f / static_cast<float>(g.grid_h * g.grid_w);
  char* obase = static_cast<char*>(out_v) + (static_cast<long long>(n) * out_roi_stride + slice * kSlice) * kEB + Io::chunk_off(q);
  for (int phi = 0; phi < ph; ++phi) {
    // 2. row pass: U[x] = sum_y Wy[phi][y] * f[y, x]   (thread = 8 channels of one column; 16 columns in flight)
    const int y0 = ylo[phi], y1 = yhi[phi];
    for (int x = c_first + worker; x <= c_last; x += 16) {
      float acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
      const char* col = img + static_cast<long long>(x) * channels * kEB + Io::chunk_off(q);
      const long long row_stride = static_cast<long long>(width) * channels * kEB;
      for (int y = y0; y <= y1; y += 4) {          // four rows in flight per thread (L2 latency)
        float v[4][8];
        float w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool live = y + j <= y1;
          w[j] = live ? Wy[phi][y + j] : 0.f;
          Io::load8(col + static_cast<long long>(live ? y + j : y1) * row_stride, v[j]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] = fmaf(w[j], v[j][e], acc[e]);
        }
      }
      U[x][q * 2] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      U[x][q * 2 + 1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    __syncthreads();
    // 3. column pass: one thread per (bin column, 8 channels)
    if (worker < pw) {
      float acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
      for (int x = xlo[worker]; x <= xhi[worker]; ++x) {
        const float w = Wx[worker][x];
        const float4 u0 = U[x][q * 2], u1 = U[x][q * 2 + 1];
        acc[0] = fmaf(w, u0.x, acc[0]); acc[1] = fmaf(w, u0.y, acc[1]);
        acc[2] = fmaf(w, u0.z, acc[2]); acc[3] = fmaf(w, u0.w, acc[3]);
        acc[4] = fmaf(w, u1.x, acc[4]); acc[5] = fmaf(w, u1.y, acc[5]);
        acc[6] = fmaf(w, u1.z, acc[6]); acc[7] = fmaf(w, u1.w, acc[7]);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] *= inv_count;
      Io::store8(obase + static_cast<long long>(phi * pw + worker) * channels * kEB, acc);
    }
    __syncthreads();
  }
}

template <typename T>
static int roi_align_nhwc_launch(const T* input, int channels, int height, int width, long long in_img_stride,
                                 const float* rois, int roi_ld, int roi_box_off, const int* roi_batch, int num_rois,
                                 float spatial_scale, int pooled_h, int pooled_w, int sampling_ratio, T* output,
                                 long long out_roi_stride, cudaStream_t stream) {
  constexpr int V = Vec16<T>::N;
  constexpr int kSlice = kRoiSliceBytes / static_cast<int>(sizeof(T));
  MEGA_ARG_CHECK((channels % V) == 0, "roi_align_nhwc: channels must be a multiple of 16 bytes");
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(input) & 15) == 0 && (reinterpret_cast<uintptr_t>(output) & 15) == 0 &&
                     (out_roi_stride % V) == 0 && (in_img_stride % V) == 0,
                 "roi_align_nhwc: 16-byte alignment required");
  if (num_rois == 0) return MEGA_OK;
  if ((channels % kSlice) == 0) {
    static bool configured = false;
    if (!configured) {
      MEGA_CUDA_CHECK(cudaFuncSetAttribute(roi_align_nhwc_cached_kernel<T>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, kRoiMaxCells * 256));
      configured = true;
    }
    dim3 cgrid(channels / kSlice, num_rois);
    roi_align_nhwc_cached_kernel<T><<<cgrid, 256, kRoiMaxCells * 256, stream>>>(
        input, channels, height, width, in_img_stride, rois, roi_ld, roi_box_off, roi_batch, spatial_scale, pooled_h,
        pooled_w, sampling_ratio, output, out_roi_stride);
    MEGA_CUDA_CHECK(cudaGetLastError());
    return MEGA_OK;
  }
  dim3 grid(pooled_h * pooled_w, num_rois);
  roi_align_nhwc_kernel<T><<<grid, 256, 0, stream>>>(input, channels, height, width, in_img_stride, rois, roi_ld,
                                                     roi_box_off, roi_batch, spatial_scale, pooled_h, pooled_w,
                                                     sampling_ratio, output, out_roi_stride);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

}  // namespace mega

using namespace mega;

extern "C" int mega_roi_align_forward_nchw(const float* input, int batch, int channels, int height, int width,
                                           const float* rois, int num_rois, float spatial_scale, int pooled_h,
                                           int pooled_w, int sampling_ratio, float* output, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  (void)batch;
  MEGA_ARG_CHECK(pooled_h > 0 && pooled_w > 0 && channels > 0, "roi_align: bad pooled size / channels");
  const long long total = static_cast<long long>(num_rois) * channels * pooled_h * pooled_w;
  if (total == 0) return MEGA_OK;  // ROIAlign_cuda.cu:278-281
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  roi_align_nchw_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(input, channels, height, width, rois, total,
                                                                      spatial_scale, pooled_h, pooled_w,
                                                                      sampling_ratio, output);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_roi_align_forward_nhwc(const float* input, int channels, int height, int width,
                                           long long in_img_stride, const float* rois, int roi_ld, int roi_box_off,
                                           const int* roi_batch, int num_rois, float spatial_scale, int pooled_h,
                                           int pooled_w, int sampling_ratio, float* output, long long out_roi_stride,
                                           void* stream_v) {
  return roi_align_nhwc_launch<float>(input, channels, height, width, in_img_stride, rois, roi_ld, roi_box_off,
                                      roi_batch, num_rois, spatial_scale, pooled_h, pooled_w, sampling_ratio, output,
                                      out_roi_stride, static_cast<cudaStream_t>(stream_v));
}

extern "C" int mega_roi_align_forward_nhwc_f16(const void* input, int channels, int height, int width,
                                               long long in_img_stride, const float* rois, int roi_ld, int roi_box_off,
                                               const int* roi_batch, int num_rois, float spatial_scale, int pooled_h,
                                               int pooled_w, int sampling_ratio, void* output,
                                               long long out_roi_stride, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  // fast path: 128-channel slices, up to 7x7 bins
  const bool fast = (channels % 128) == 0 && pooled_h <= 7 && pooled_w <= 7 &&
                    (reinterpret_cast<uintptr_t>(input) & 15) == 0 && (reinterpret_cast<uintptr_t>(output) & 15) == 0 &&
                    (out_roi_stride % 8) == 0 && (in_img_stride % 8) == 0;
  if (fast && height <= kSepMaxDim && width <= kSepMaxDim && g_roi_separable) {
    if (num_rois == 0) return MEGA_OK;
    dim3 grid(channels / 128, num_rois);
    roi_align_nhwc_sep_kernel<false><<<grid, 256, 0, stream>>>(
        input, channels, height, width, in_img_stride, rois, roi_ld, roi_box_off, roi_batch,
        spatial_scale, pooled_h, pooled_w, sampling_ratio, output, out_roi_stride);
    MEGA_CUDA_CHECK(cudaGetLastError());
    return MEGA_OK;
  }
  if (fast) {
    if (num_rois == 0) return MEGA_OK;
    static bool configured = false;
    if (!configured) {
      MEGA_CUDA_CHECK(cudaFuncSetAttribute(roi_align_nhwc_f16_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           kRoiMaxCells * 256));
      configured = true;
    }
    dim3 grid(channels / 128, num_rois);
    roi_align_nhwc_f16_fast_kernel<<<grid, 256, kRoiMaxCells * 256, stream>>>(
        static_cast<const __half*>(input), channels, height, width, in_img_stride, rois, roi_ld, roi_box_off, roi_batch,
        spatial_scale, pooled_h, pooled_w, sampling_ratio, static_cast<__half*>(output), out_roi_stride);
    MEGA_CUDA_CHECK(cudaGetLastError());
    return MEGA_OK;
  }
  return roi_align_nhwc_launch<__half>(static_cast<const __half*>(input), channels, height, width, in_img_stride, rois,
                                       roi_ld, roi_box_off, roi_batch, num_rois, spatial_scale, pooled_h, pooled_w,
                                       sampling_ratio, static_cast<__half*>(output), out_roi_stride, stream);
}

/* ROIAlign over a split-fp16 NHWC map into split-fp16 rows (include/mega_b200.h; the strict engine's format): the separable
 * kernel, maps up to 64 x 64 cells, channels a multiple of 128, bins up to 7 x 7 (MEGA_ERR_ARG otherwise: the caller then
 * unpacks and uses mega_roi_align_forward_nhwc). Blends in fp32 with fused multiply-adds: results agree with the reference's
 * association order to ~1e-6 relative, not bit for bit (layers/roi_align.py:13-36, ROIAlign_cuda.cu:62-115). */
extern "C" int mega_roi_align_forward_nhwc_split16(const void* input, int channels, int height, int width,
                                                   long long in_img_stride, const float* rois, int roi_ld, int roi_box_off,
                                                   const int* roi_batch, int num_rois, float spatial_scale, int pooled_h,
                                                   int pooled_w, int sampling_ratio, void* output,
                                                   long long out_roi_stride, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK((channels % 128) == 0 && pooled_h <= 7 && pooled_w <= 7 && pooled_h > 0 && pooled_w > 0 &&
                     height <= kSepMaxDim && width <= kSepMaxDim,
                 "roi_align_split16: needs channels %% 128 == 0, bins <= 7x7, map <= 64x64 (got C %d, %dx%d bins, map %dx%d)",
                 channels, pooled_h, pooled_w, height, width);
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(input) & 127) == 0 && (reinterpret_cast<uintptr_t>(output) & 127) == 0 &&
                     (out_roi_stride % 32) == 0 && (in_img_stride % 32) == 0,
                 "roi_align_split16: 128-byte alignment required");
  if (num_rois == 0) return MEGA_OK;
  dim3 grid(channels / 128, num_rois);
  roi_align_nhwc_sep_kernel<true><<<grid, 256, 0, stream>>>(input, channels, height, width, in_img_stride, rois, roi_ld,
                                                             roi_box_off, roi_batch, spatial_scale, pooled_h, pooled_w,
                                                             sampling_ratio, output, out_roi_stride);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
