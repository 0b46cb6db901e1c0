// Kernels of the FGFA path (flow-guided feature aggregation) that are not convolutions:
//   * image pairs for FlowNetS: avg-pool(2, ceil) of image / 255 per frame, and the 19 (key, frame) pairs laid out for
//     the 7x7 / stride-2 first convolution as an implicit GEMM (detector/generalized_rcnn_fgfa.py:198-202,
//     backbone/flownet.py:55-57);
//   * NHWC 2x2 average pooling with ceil_mode (flownet.py:113);
//   * warp + adaptive weights + aggregation: bilinear resampling of the cached feature / embedding maps along the flow
//     (get_grid / resample :45-62), cosine similarity of the warped embeddings with the key frame's (:64-76),
//     soft-max over the window and the weighted sum (:206-214) -- in one pass, nothing of the [19, 3072, h, w] warped
//     tensor (559 MB at 600x1000) is materialised.
// Element type T is the engine's activation type (fp32 or fp16); arithmetic is fp32.
#include <cuda_fp16.h>
#include "common.cuh"
#include "mega_b200.h"

namespace mega {

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// img [3,H,W] fp32 -> out [Hq,Wq,4]: mean over the 2x2 window clipped to the image (ceil_mode, pad 0), divided by 255
template <typename T>
__global__ void fgfa_pool_image_kernel(const float* __restrict__ img, int height, int width, int hq, int wq,
                                       T* __restrict__ out) {
  const int total = hq * wq;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int y = i / wq, x = i - y * wq;
    const int y0 = 2 * y, x0 = 2 * x, y1 = min(y0 + 2, height), x1 = min(x0 + 2, width);
    const float inv = 1.0f / static_cast<float>((y1 - y0) * (x1 - x0));
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < 3; ++c) {
      float s = 0.f;
      for (int yy = y0; yy < y1; ++yy)
        for (int xx = x0; xx < x1; ++xx) s += __ldg(img + (static_cast<long long>(c) * height + yy) * width + xx) / 255.0f;
      v[c] = s * inv;
    }
    T* o = out + static_cast<long long>(i) * 4;
    o[0] = from_f<T>(v[0]); o[1] = from_f<T>(v[1]); o[2] = from_f<T>(v[2]); o[3] = from_f<T>(0.f);
  }
}

// pairs [L][hq + 6][wq + 8][8]: interior (y + 3, x + 3) = (key frame c0..2, 0, frame i c0..2, 0); borders zero
template <typename T>
__global__ void fgfa_build_pairs_kernel(const T* __restrict__ ring, long long slot_stride, const int* __restrict__ slots,
                                        int n_frames, int key_pos, int hq, int wq, T* __restrict__ pairs) {
  const int hp = hq + 6, wp = wq + 8;
  const long long total = static_cast<long long>(n_frames) * hp * wp;
  const T* key = ring + static_cast<long long>(slots[key_pos]) * slot_stride;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % wp) - 3;
    const int y = static_cast<int>((i / wp) % hp) - 3;
    const int f = static_cast<int>(i / (static_cast<long long>(wp) * hp));
    T v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = from_f<T>(0.f);
    if (y >= 0 && y < hq && x >= 0 && x < wq) {
      const T* a = key + (static_cast<long long>(y) * wq + x) * 4;
      const T* b = ring + static_cast<long long>(slots[f]) * slot_stride + (static_cast<long long>(y) * wq + x) * 4;
      v[0] = a[0]; v[1] = a[1]; v[2] = a[2];
      v[4] = b[0]; v[5] = b[1]; v[6] = b[2];
    }
    T* o = pairs + i * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = v[e];
  }
}

// NHWC average pooling 2x2 / stride 2, ceil_mode, divisor = number of in-bound cells
template <typename T>
__global__ void avgpool2_nhwc_kernel(const T* __restrict__ in, int n_img, int height, int width, int channels, long long in_ld,
                                     int ho, int wo, T* __restrict__ out, long long out_ld) {
  const long long total = static_cast<long long>(n_img) * ho * wo * channels;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % channels);
    const long long pix = i / channels;
    const int x = static_cast<int>(pix % wo), y = static_cast<int>((pix / wo) % ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(wo) * ho));
    const int y0 = 2 * y, x0 = 2 * x, y1 = min(y0 + 2, height), x1 = min(x0 + 2, width);
    float s = 0.f;
    for (int yy = y0; yy < y1; ++yy)
      for (int xx = x0; xx < x1; ++xx) s += to_f<T>(in[((static_cast<long long>(n) * height + yy) * width + xx) * in_ld + c]);
    out[pix * out_ld + c] = from_f<T>(s / static_cast<float>((y1 - y0) * (x1 - x0)));
  }
}

// One CTA per output pixel. ring: [slots][h*w][ld] with feats in [0, cf) and embeddings in [cf, cf + ce).
// flow [L][h*w][flow_ld] fp32 (x, y in feature cells). Sampling = F.grid_sample(bilinear, border, align_corners=False) of
// the grid get_grid() builds: gx = (fx + x) / ((w-1)/2) - 1  ->  pixel coordinate ((gx + 1) * w - 1) / 2, clamped to
// [0, w-1].
constexpr int kAggThreads = 256;
constexpr int kAggMaxFrames = 32;

struct Corner {
  long long o00, o01, o10, o11;
  float w00, w01, w10, w11;
};

__device__ __forceinline__ Corner flow_corners(float fx, float fy, int x, int y, int w, int h, int ld) {
  const float gx = __fdiv_rn(fx + static_cast<float>(x), static_cast<float>(w - 1) * 0.5f) - 1.0f;
  const float gy = __fdiv_rn(fy + static_cast<float>(y), static_cast<float>(h - 1) * 0.5f) - 1.0f;
  float px = ((gx + 1.0f) * static_cast<float>(w) - 1.0f) * 0.5f;
  float py = ((gy + 1.0f) * static_cast<float>(h) - 1.0f) * 0.5f;
  px = fminf(fmaxf(px, 0.f), static_cast<float>(w - 1));
  py = fminf(fmaxf(py, 0.f), static_cast<float>(h - 1));
  const float x0f = floorf(px), y0f = floorf(py);
  const int x0 = static_cast<int>(x0f), y0 = static_cast<int>(y0f);
  const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
  const float lx = px - x0f, ly = py - y0f;
  Corner c;
  c.o00 = (static_cast<long long>(y0) * w + x0) * ld; c.o01 = (static_cast<long long>(y0) * w + x1) * ld;
  c.o10 = (static_cast<long long>(y1) * w + x0) * ld; c.o11 = (static_cast<long long>(y1) * w + x1) * ld;
  c.w00 = (1.f - lx) * (1.f - ly); c.w01 = lx * (1.f - ly); c.w10 = (1.f - lx) * ly; c.w11 = lx * ly;
  return c;
}

template <typename T>
__device__ __forceinline__ float sample(const T* base, const Corner& c, int ch) {
  return c.w00 * to_f<T>(base[c.o00 + ch]) + c.w01 * to_f<T>(base[c.o01 + ch]) + c.w10 * to_f<T>(base[c.o10 + ch]) +
         c.w11 * to_f<T>(base[c.o11 + ch]);
}

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < kAggThreads / 32; ++i) s += red[i];
  return s;
}

template <typename T>
__global__ void __launch_bounds__(kAggThreads)
fgfa_aggregate_kernel(const T* __restrict__ ring, long long slot_stride, int ld, int cf, int ce,
                      const int* __restrict__ slots, int n_frames, int key_pos, const float* __restrict__ flow,
                      int flow_ld, int h, int w, T* __restrict__ out, long long out_ld, float* __restrict__ weights_out) {
  __shared__ float red[kAggThreads / 32];
  __shared__ float logit[kAggMaxFrames];
  __shared__ Corner corners[kAggMaxFrames];
  const int pix = blockIdx.x;
  const int y = pix / w, x = pix - y * w;
  const int tid = threadIdx.x;
  if (tid < n_frames) {
    const float* f = flow + (static_cast<long long>(tid) * h * w + pix) * flow_ld;
    corners[tid] = flow_corners(f[0], f[1], x, y, w, h, ld);
  }
  __syncthreads();
  // warped embedding of the key frame (this thread's channels) and its norm
  const int per = (ce + kAggThreads - 1) / kAggThreads;     // channels per thread (2048 / 256 = 8)
  float ek[16];
  const T* kbase = ring + static_cast<long long>(slots[key_pos]) * slot_stride + cf;
  float kn = 0.f;
  for (int j = 0; j < per && j < 16; ++j) {
    const int ch = tid + j * kAggThreads;
    ek[j] = ch < ce ? sample<T>(kbase, corners[key_pos], ch) : 0.f;
    kn += ek[j] * ek[j];
  }
  kn = sqrtf(block_sum(kn, red)) + 1e-10f;
  for (int f = 0; f < n_frames; ++f) {
    const T* fbase = ring + static_cast<long long>(slots[f]) * slot_stride + cf;
    float dot = 0.f, nn = 0.f;
    for (int j = 0; j < per && j < 16; ++j) {
      const int ch = tid + j * kAggThreads;
      const float e = ch < ce ? sample<T>(fbase, corners[f], ch) : 0.f;
      dot += e * ek[j];
      nn += e * e;
    }
    dot = block_sum(dot, red);
    nn = sqrtf(block_sum(nn, red)) + 1e-10f;
    if (tid == 0) logit[f] = (dot / nn) / kn;      // sum of (e_ref / |e_ref|) * (e_cur / |e_cur|)
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int f = 0; f < n_frames; ++f) mx = fmaxf(mx, logit[f]);
  float den = 0.f;
  for (int f = 0; f < n_frames; ++f) den += expf(logit[f] - mx);
  const float inv = 1.0f / den;
  if (weights_out != nullptr && tid < n_frames) weights_out[static_cast<long long>(tid) * h * w + pix] = expf(logit[tid] - mx) * inv;
  for (int ch = tid; ch < cf; ch += kAggThreads) {
    float acc = 0.f;
    for (int f = 0; f < n_frames; ++f) {
      const T* fbase = ring + static_cast<long long>(slots[f]) * slot_stride;
      acc += expf(logit[f] - mx) * inv * sample<T>(fbase, corners[f], ch);
    }
    out[static_cast<long long>(pix) * out_ld + ch] = from_f<T>(acc);
  }
}

// DFF (detector/generalized_rcnn_dff.py:131-134): out = resample(key_feats, flow) * scale_map. One thread per
// (pixel, 8 channels): the four bilinear corners of a pixel are shared by its 1024 channels (consecutive threads),
// channel-fastest so every corner read / scale read / store is a coalesced 16- or 32-byte access.
template <typename T>
__global__ void dff_warp_scale_kernel(const T* __restrict__ key, int ld, int channels, const float* __restrict__ flow,
                                      int flow_ld, const T* __restrict__ scale, long long scale_ld, int h, int w,
                                      T* __restrict__ out, long long out_ld) {
  const int groups = channels / 8;
  const long long total = static_cast<long long>(h) * w * groups;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    const int pix = static_cast<int>(i / groups);
    const int y = pix / w, x = pix - y * w;
    const float* f = flow + static_cast<long long>(pix) * flow_ld;
    const Corner c = flow_corners(f[0], f[1], x, y, w, h, ld);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int ch = g * 8 + e;
      const float v = sample<T>(key, c, ch) * to_f<T>(scale[static_cast<long long>(pix) * scale_ld + ch]);
      out[static_cast<long long>(pix) * out_ld + ch] = from_f<T>(v);
    }
  }
}

static int grid_for(long long total, int block) {
  long long b = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace mega

using namespace mega;

extern "C" int mega_fgfa_pool_image(const float* image, int height, int width, void* out, int f16, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int hq = (height + 1) / 2, wq = (width + 1) / 2;
  if (f16) fgfa_pool_image_kernel<__half><<<grid_for(hq * wq, 256), 256, 0, stream>>>(image, height, width, hq, wq, static_cast<__half*>(out));
  else fgfa_pool_image_kernel<float><<<grid_for(hq * wq, 256), 256, 0, stream>>>(image, height, width, hq, wq, static_cast<float*>(out));
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_fgfa_build_pairs(const void* ring, long long slot_stride, const int* slots, int n_frames, int key_pos,
                                     int hq, int wq, void* pairs, int f16, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(n_frames > 0 && key_pos >= 0 && key_pos < n_frames, "fgfa_build_pairs: bad frame indices");
  const long long total = static_cast<long long>(n_frames) * (hq + 6) * (wq + 8);
  if (f16) fgfa_build_pairs_kernel<__half><<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const __half*>(ring), slot_stride, slots, n_frames, key_pos, hq, wq, static_cast<__half*>(pairs));
  else fgfa_build_pairs_kernel<float><<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const float*>(ring), slot_stride, slots, n_frames, key_pos, hq, wq, static_cast<float*>(pairs));
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_avgpool2_nhwc(const void* input, int n_img, int height, int width, int channels, long long in_ld,
                                  void* out, long long out_ld, int f16, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int ho = (height + 1) / 2, wo = (width + 1) / 2;
  const long long total = static_cast<long long>(n_img) * ho * wo * channels;
  if (total == 0) return MEGA_OK;
  if (f16) avgpool2_nhwc_kernel<__half><<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const __half*>(input), n_img, height, width, channels, in_ld, ho, wo, static_cast<__half*>(out), out_ld);
  else avgpool2_nhwc_kernel<float><<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const float*>(input), n_img, height, width, channels, in_ld, ho, wo, static_cast<float*>(out), out_ld);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_fgfa_aggregate(const void* ring, long long slot_stride, int ld, int feat_channels, int embed_channels,
                                   const int* slots, int n_frames, int key_pos, const float* flow, int flow_ld, int height,
                                   int width, void* out, long long out_ld, float* weights_out, int f16, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(n_frames > 0 && n_frames <= kAggMaxFrames && key_pos >= 0 && key_pos < n_frames,
                 "fgfa_aggregate: at most %d frames", kAggMaxFrames);
  MEGA_ARG_CHECK(embed_channels <= 16 * kAggThreads, "fgfa_aggregate: at most %d embedding channels", 16 * kAggThreads);
  const int pixels = height * width;
  if (f16) fgfa_aggregate_kernel<__half><<<pixels, kAggThreads, 0, stream>>>(static_cast<const __half*>(ring), slot_stride, ld, feat_channels, embed_channels, slots, n_frames, key_pos, flow, flow_ld, height, width, static_cast<__half*>(out), out_ld, weights_out);
  else fgfa_aggregate_kernel<float><<<pixels, kAggThreads, 0, stream>>>(static_cast<const float*>(ring), slot_stride, ld, feat_channels, embed_channels, slots, n_frames, key_pos, flow, flow_ld, height, width, static_cast<float*>(out), out_ld, weights_out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_dff_warp_scale(const void* key_feats, int ld, int channels, const float* flow, int flow_ld,
                                   const void* scale, long long scale_ld, int height, int width, void* out,
                                   long long out_ld, int f16, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(channels > 0 && channels % 8 == 0 && height > 0 && width > 0, "dff_warp_scale: channels must be a multiple of 8");
  const long long total = static_cast<long long>(height) * width * (channels / 8);
  if (f16) dff_warp_scale_kernel<__half><<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const __half*>(key_feats), ld, channels, flow, flow_ld, static_cast<const __half*>(scale), scale_ld, height, width, static_cast<__half*>(out), out_ld);
  else dff_warp_scale_kernel<float><<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const float*>(key_feats), ld, channels, flow, flow_ld, static_cast<const float*>(scale), scale_ld, height, width, static_cast<float*>(out), out_ld);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
