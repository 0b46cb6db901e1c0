// The remaining custom ops of mega_core/csrc that the north star names, forward (inference) side:
//   * sigmoid focal loss forward/backward   (csrc/cuda/SigmoidFocalLoss_cuda.cu:20-103)
//   * deformable / modulated deformable convolution: bilinear im2col
//     (csrc/cuda/deform_conv_kernel_cuda.cu:92-120, :197-250, :475-504, :578-640); the contraction that
//     follows (`addmm_` per group in deform_conv_cuda.cu:228-243, :545-567) runs on the wgmma GEMM,
//     so the column matrix is written K-major per output pixel: cols[b][h*Wo+w][c*kh*kw + i*kw + j];
//   * deformable position-sensitive ROI pooling forward (csrc/cuda/deform_pool_kernel_cuda.cu:31-142).
// They complete the `_C` operator surface (focal loss is RetinaNet-only). The engines' deformable backbone stages
// (MODEL.RESNETS.STAGE_WITH_DCN) do not run through mega_deform_im2col: they sample NHWC activations into a tap-major
// column operand (dcn_sample.cu); the tile kernel below shares its sample geometry with that kernel (dcn_sample.cuh).
#include <float.h>
#include "common.cuh"
#include "dcn_sample.cuh"
#include "mega_b200.h"

namespace mega {

// Sigmoid focal loss (SigmoidFocalLoss_cuda.cu:20-103) through the log-sigmoid identities
//     log p = -softplus(-x),   log(1 - p) = -softplus(x),   softplus(x) = max(x, 0) + log1p(exp(-|x|)),
// i.e. ONE exp and ONE log1p per logit (+ the two powers) instead of three exps and two logs; p itself comes from the same
// e = exp(-|x|). One thread handles four consecutive logits of a row when the class count and the pointers' alignment
// allow it (128-bit loads / stores); the target of a row is read once per thread.
struct FocalTerms {
  float p, log_p, log_1mp;
};
__device__ __forceinline__ FocalTerms focal_terms(float x) {
  const float e = __expf(-fabsf(x));
  const float l = log1pf(e);
  FocalTerms t;
  const float inv = 1.f / (1.f + e);
  t.p = x >= 0.f ? inv : e * inv;
  t.log_p = -(fmaxf(-x, 0.f) + l);
  t.log_1mp = -(fmaxf(x, 0.f) + l);
  return t;
}
// u^gamma for u in [0, 1] as exp(gamma * log u) with log u already at hand (log(1 - p) and log p are the loss's own
// terms): no powf call, one MUFU.EX2
__device__ __forceinline__ float focal_pow(float log_u, float gamma) { return __expf(gamma * log_u); }
__device__ __forceinline__ float focal_fwd_one(float x, int t, int d, float gamma, float alpha) {
  const FocalTerms f = focal_terms(x);
  if (t == d + 1) return -alpha * focal_pow(f.log_1mp, gamma) * fmaxf(f.log_p, -87.3365f);      // log(FLT_MIN)
  if (t >= 0) return -(1.f - alpha) * focal_pow(f.log_p, gamma) * f.log_1mp;
  return 0.f;
}
__device__ __forceinline__ float focal_bwd_one(float x, int t, int d, float gamma, float alpha) {
  const FocalTerms f = focal_terms(x);
  if (t == d + 1) return -alpha * focal_pow(f.log_1mp, gamma) * (1.f - f.p - f.p * gamma * fmaxf(f.log_p, -87.3365f));
  if (t >= 0) return -(1.f - alpha) * focal_pow(f.log_p, gamma) * (f.log_1mp * (1.f - f.p) * gamma - f.p);
  return 0.f;
}

// VEC: one thread per four consecutive logits of a row (128-bit loads / stores). The host picks it only when the class
// count is a multiple of 4 (a float4 never straddles two rows) and logits, d_losses and out are 16-byte aligned.
template <bool BWD, bool VEC>
__global__ void focal_loss_kernel(long long total, const float* __restrict__ logits, const int* __restrict__ targets,
                                  const float* __restrict__ d_losses, int num_classes, float gamma, float alpha,
                                  float* __restrict__ out) {
  const long long items = VEC ? total / 4 : total;
  for (long long it = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; it < items;
       it += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (VEC) {
      const long long i = it * 4;
      const long long n = i / num_classes;
      const int d = static_cast<int>(i - n * num_classes);
      const int t = __ldg(targets + n);
      const float4 x = __ldg(reinterpret_cast<const float4*>(logits + i));
      float4 r;
      if (BWD) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(d_losses + i));
        r.x = focal_bwd_one(x.x, t, d, gamma, alpha) * g.x;
        r.y = focal_bwd_one(x.y, t, d + 1, gamma, alpha) * g.y;
        r.z = focal_bwd_one(x.z, t, d + 2, gamma, alpha) * g.z;
        r.w = focal_bwd_one(x.w, t, d + 3, gamma, alpha) * g.w;
      } else {
        r.x = focal_fwd_one(x.x, t, d, gamma, alpha);
        r.y = focal_fwd_one(x.y, t, d + 1, gamma, alpha);
        r.z = focal_fwd_one(x.z, t, d + 2, gamma, alpha);
        r.w = focal_fwd_one(x.w, t, d + 3, gamma, alpha);
      }
      *reinterpret_cast<float4*>(out + i) = r;
    } else {
      const long long n = it / num_classes;
      const int d = static_cast<int>(it - n * num_classes);
      const int t = __ldg(targets + n);
      const float x = __ldg(logits + it);
      out[it] = BWD ? focal_bwd_one(x, t, d, gamma, alpha) * __ldg(d_losses + it) : focal_fwd_one(x, t, d, gamma, alpha);
    }
  }
}

__device__ __forceinline__ float dcn_bilinear(const float* __restrict__ plane, int height, int width, float h, float w) {
  const int h_low = static_cast<int>(floorf(h)), w_low = static_cast<int>(floorf(w));
  const int h_high = h_low + 1, w_high = w_low + 1;
  const float lh = h - h_low, lw = w - w_low, hh = 1.f - lh, hw = 1.f - lw;
  float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
  if (h_low >= 0 && w_low >= 0) v1 = plane[h_low * width + w_low];
  if (h_low >= 0 && w_high <= width - 1) v2 = plane[h_low * width + w_high];
  if (h_high <= height - 1 && w_low >= 0) v3 = plane[h_high * width + w_low];
  if (h_high <= height - 1 && w_high <= width - 1) v4 = plane[h_high * width + w_high];
  const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
  return w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4;
}

// Deformable im2col, tile form. A CTA (4 warps) owns 32 consecutive output pixels of one output row and kDcnCh
// channels of one deformable group:
//   1. the sample geometry of every (tap, pixel) -- offsets read once, floor / weights / the four corner indices with
//      their validity folded into the weights -- goes to shared memory; it is shared by all channels of the group (the
//      reference recomputes it per channel, deform_conv_kernel_cuda.cu:197-250);
//   2. lane = pixel, so the four gathers of a (channel, tap) read neighbouring addresses of ONE channel plane (the
//      reference layout is NCHW) -- round 1's thread-per-(pixel, channel) mapping read 32 different planes per warp;
//   3. the K-major rows cols[pixel][c*kh*kw + tap] are staged in shared memory and written with 128-bit stores, a row
//      segment of kDcnCh*kh*kw floats per pixel (round 1 wrote 4 bytes every kh*kw*4).
// The arithmetic per element is unchanged (dcn_bilinear), so results are bit-identical to the scalar kernel.
constexpr int kDcnPix = 32;
constexpr int kDcnCh = 16;
constexpr int kDcnMaxTaps = 49;     // up to 7x7 kernels in shared memory; larger ones take the scalar kernel

__global__ void __launch_bounds__(128)
deform_im2col_tile_kernel(const float* __restrict__ im, const float* __restrict__ offset, const float* __restrict__ mask,
                          int channels, int height, int width, int kh, int kw, int pad_h, int pad_w, int stride_h,
                          int stride_w, int dil_h, int dil_w, int deformable_group, int ho, int wo, int kpad,
                          float* __restrict__ cols) {
  extern __shared__ float dcn_smem[];
  const int taps = kh * kw;
  DcnTap* geo = reinterpret_cast<DcnTap*>(dcn_smem);                      // [taps][32] sample geometry
  float* mvals = dcn_smem + taps * kDcnPix * (sizeof(DcnTap) / 4);        // [taps][32] modulation scalars (DCN v2)
  float* stage = mvals + taps * kDcnPix;                                  // [32][kDcnCh * taps + 1] output rows
  const int ld = kDcnCh * taps + 1;
  const int cpg = channels / deformable_group;
  const int ch_tiles = (cpg + kDcnCh - 1) / kDcnCh;
  const int w_tiles = (wo + kDcnPix - 1) / kDcnPix;
  int bid = blockIdx.x;
  const int wt = bid % w_tiles; bid /= w_tiles;
  const int ct = bid % ch_tiles; bid /= ch_tiles;
  const int dg = bid % deformable_group; bid /= deformable_group;
  const int h_col = bid % ho;
  const int b = bid / ho;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int w_col = wt * kDcnPix + lane;
  const bool live = w_col < wo;
  const long long plane_sz = static_cast<long long>(height) * width;
  // ---- 1. geometry
  const float* off = offset + (static_cast<long long>(b) * deformable_group + dg) * 2 * taps * ho * wo;
  const float* msk = mask ? mask + (static_cast<long long>(b) * deformable_group + dg) * taps * ho * wo : nullptr;
  for (int tap = warp; tap < taps; tap += 4) {
    DcnTap g = {0, 0, 0, 0, 0.f, 0.f, 0.f, 0.f};
    if (live) {
      const int i = tap / kw, j = tap - i * kw;
      const long long o = (static_cast<long long>(2 * tap) * ho + h_col) * wo + w_col;
      const float h_im = h_col * stride_h - pad_h + i * dil_h + __ldg(off + o);
      const float w_im = w_col * stride_w - pad_w + j * dil_w + __ldg(off + o + static_cast<long long>(ho) * wo);
      g = dcn_tap_geometry(h_im, w_im, height, width);
      // the modulation scalar of DCN v2 multiplies the interpolated value (kept as a separate factor, like the reference)
      if (msk) mvals[tap * kDcnPix + lane] = __ldg(msk + (static_cast<long long>(tap) * ho + h_col) * wo + w_col);
    }
    geo[tap * kDcnPix + lane] = g;
  }
  __syncthreads();
  // ---- 2. gather: items = (channel of the tile, tap), lane = pixel
  const int c0 = dg * cpg + ct * kDcnCh;
  const int nch = min(kDcnCh, cpg - ct * kDcnCh);
  // a warp takes one tap at a time and kDcnUnroll channels per step: the geometry stays in registers and 4 x kDcnUnroll
  // independent gathers are in flight per lane (one gather chain per step left the kernel latency-bound at 0.63 TB/s)
  constexpr int kDcnUnroll = 8;
  for (int tap = warp; tap < taps; tap += 4) {
    const DcnTap g = geo[tap * kDcnPix + lane];
    const bool inside = live && g.i00 != kDcnOutside;
    const float mval = (msk && live) ? mvals[tap * kDcnPix + lane] : 1.f;
    const float* plane0 = im + (static_cast<long long>(b) * channels + c0) * plane_sz;
    for (int cl0 = 0; cl0 < nch; cl0 += kDcnUnroll) {
      float v[kDcnUnroll][4];
#pragma unroll
      for (int u = 0; u < kDcnUnroll; ++u) {
        const float* plane = plane0 + static_cast<long long>(min(cl0 + u, nch - 1)) * plane_sz;
        v[u][0] = (inside && g.i00 >= 0) ? __ldg(plane + g.i00) : 0.f;
        v[u][1] = (inside && g.i01 >= 0) ? __ldg(plane + g.i01) : 0.f;
        v[u][2] = (inside && g.i10 >= 0) ? __ldg(plane + g.i10) : 0.f;
        v[u][3] = (inside && g.i11 >= 0) ? __ldg(plane + g.i11) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kDcnUnroll; ++u) {
        if (cl0 + u < nch) {
          float val = g.w00 * v[u][0] + g.w01 * v[u][1] + g.w10 * v[u][2] + g.w11 * v[u][3];
          if (msk) val *= mval;
          stage[lane * ld + (cl0 + u) * taps + tap] = val;
        }
      }
    }
  }
  __syncthreads();
  // ---- 3. rows out: pixel p of the tile, nch*taps consecutive floats starting at column c0*taps
  const int seg = nch * taps;
  for (int p = warp; p < kDcnPix; p += 4) {
    const int wc = wt * kDcnPix + p;
    if (wc >= wo) break;
    float* row = cols + ((static_cast<long long>(b) * ho + h_col) * wo + wc) * kpad + static_cast<long long>(c0) * taps;
    const float* src = stage + p * ld;
    if (((reinterpret_cast<uintptr_t>(row) & 15) == 0) && (seg & 3) == 0) {
      for (int v = lane; v < seg / 4; v += 32) {
        float4 o = make_float4(src[4 * v], src[4 * v + 1], src[4 * v + 2], src[4 * v + 3]);
        *reinterpret_cast<float4*>(row + 4 * v) = o;
      }
    } else {
      for (int v = lane; v < seg; v += 32) row[v] = src[v];
    }
  }
}

// scalar form (kernels larger than 7x7): one thread per (b, c, h_col, w_col); writes the kh*kw taps of that channel into
// the pixel's K-major row
__global__ void deform_im2col_kernel(long long total, const float* __restrict__ im, const float* __restrict__ offset,
                                     const float* __restrict__ mask, int batch, int channels, int height, int width,
                                     int kh, int kw, int pad_h, int pad_w, int stride_h, int stride_w, int dil_h,
                                     int dil_w, int deformable_group, int ho, int wo, int kpad,
                                     float* __restrict__ cols) {
  const int cpg = channels / deformable_group;
  for (long long index = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; index < total;
       index += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(index % channels);                // channel fastest: contiguous K-major writes
    const int w_col = static_cast<int>((index / channels) % wo);
    const int h_col = static_cast<int>((index / channels / wo) % ho);
    const int b = static_cast<int>(index / channels / wo / ho);
    const int dg = c / cpg;
    const int h_in = h_col * stride_h - pad_h, w_in = w_col * stride_w - pad_w;
    const float* plane = im + (static_cast<long long>(b) * channels + c) * height * width;
    const float* off = offset + (static_cast<long long>(b) * deformable_group + dg) * 2 * kh * kw * ho * wo;
    const float* msk = mask ? mask + (static_cast<long long>(b) * deformable_group + dg) * kh * kw * ho * wo : nullptr;
    float* row = cols + ((static_cast<long long>(b) * ho + h_col) * wo + w_col) * kpad + c * kh * kw;
    for (int i = 0; i < kh; ++i) {
      for (int j = 0; j < kw; ++j) {
        const int tap = i * kw + j;
        const float offset_h = off[((2 * tap) * ho + h_col) * wo + w_col];
        const float offset_w = off[((2 * tap + 1) * ho + h_col) * wo + w_col];
        const float h_im = h_in + i * dil_h + offset_h;
        const float w_im = w_in + j * dil_w + offset_w;
        float val = 0.f;
        if (h_im > -1 && w_im > -1 && h_im < height && w_im < width) val = dcn_bilinear(plane, height, width, h_im, w_im);
        if (msk) val *= msk[(tap * ho + h_col) * wo + w_col];
        row[tap] = val;
      }
    }
  }
}

__device__ __forceinline__ float psroi_bilinear(const float* __restrict__ data, float x, float y, int width) {
  const int x1 = static_cast<int>(floorf(x)), x2 = static_cast<int>(ceilf(x));
  const int y1 = static_cast<int>(floorf(y)), y2 = static_cast<int>(ceilf(y));
  const float dist_x = x - x1, dist_y = y - y1;
  const float v11 = data[y1 * width + x1], v12 = data[y2 * width + x1];
  const float v21 = data[y1 * width + x2], v22 = data[y2 * width + x2];
  return (1 - dist_x) * (1 - dist_y) * v11 + (1 - dist_x) * dist_y * v12 + dist_x * (1 - dist_y) * v21 +
         dist_x * dist_y * v22;
}

__global__ void deform_psroi_fwd_kernel(long long count, const float* __restrict__ bottom, float spatial_scale,
                                        int channels, int height, int width, int pooled_h, int pooled_w,
                                        const float* __restrict__ rois, const float* __restrict__ trans, int no_trans,
                                        float trans_std, int sample_per_part, int output_dim, int group_size,
                                        int part_size, int num_classes, int channels_each_class,
                                        float* __restrict__ top, float* __restrict__ top_count) {
  for (long long index = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; index < count;
       index += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pw = static_cast<int>(index % pooled_w);
    const int ph = static_cast<int>((index / pooled_w) % pooled_h);
    const int ctop = static_cast<int>((index / pooled_w / pooled_h) % output_dim);
    const long long n = index / pooled_w / pooled_h / output_dim;
    const float* r = rois + n * 5;
    const int roi_batch_ind = static_cast<int>(r[0]);
    const float roi_start_w = roundf(r[1]) * spatial_scale - 0.5f;
    const float roi_start_h = roundf(r[2]) * spatial_scale - 0.5f;
    const float roi_end_w = (roundf(r[3]) + 1.f) * spatial_scale - 0.5f;
    const float roi_end_h = (roundf(r[4]) + 1.f) * spatial_scale - 0.5f;
    const float roi_width = fmaxf(roi_end_w - roi_start_w, 0.1f);
    const float roi_height = fmaxf(roi_end_h - roi_start_h, 0.1f);
    const float bin_size_h = roi_height / static_cast<float>(pooled_h);
    const float bin_size_w = roi_width / static_cast<float>(pooled_w);
    const float sub_bin_size_h = bin_size_h / static_cast<float>(sample_per_part);
    const float sub_bin_size_w = bin_size_w / static_cast<float>(sample_per_part);
    const int part_h = static_cast<int>(floorf(static_cast<float>(ph) / pooled_h * part_size));
    const int part_w = static_cast<int>(floorf(static_cast<float>(pw) / pooled_w * part_size));
    const int class_id = ctop / channels_each_class;
    const float trans_x =
        no_trans ? 0.f : trans[(((n * num_classes + class_id) * 2) * part_size + part_h) * part_size + part_w] * trans_std;
    const float trans_y =
        no_trans ? 0.f
                 : trans[(((n * num_classes + class_id) * 2 + 1) * part_size + part_h) * part_size + part_w] * trans_std;
    float wstart = static_cast<float>(pw) * bin_size_w + roi_start_w;
    wstart += trans_x * roi_width;
    float hstart = static_cast<float>(ph) * bin_size_h + roi_start_h;
    hstart += trans_y * roi_height;
    float sum = 0.f;
    int cnt = 0;
    int gw = static_cast<int>(floorf(static_cast<float>(pw) * group_size / pooled_w));
    int gh = static_cast<int>(floorf(static_cast<float>(ph) * group_size / pooled_h));
    gw = min(max(gw, 0), group_size - 1);
    gh = min(max(gh, 0), group_size - 1);
    const float* data = bottom + (static_cast<long long>(roi_batch_ind) * channels) * height * width;
    for (int ih = 0; ih < sample_per_part; ++ih) {
      for (int iw = 0; iw < sample_per_part; ++iw) {
        float w = wstart + iw * sub_bin_size_w;
        float h = hstart + ih * sub_bin_size_h;
        if (w < -0.5f || w > width - 0.5f || h < -0.5f || h > height - 0.5f) continue;
        w = fminf(fmaxf(w, 0.f), width - 1.f);
        h = fminf(fmaxf(h, 0.f), height - 1.f);
        const int c = (ctop * group_size + gh) * group_size + gw;
        sum += psroi_bilinear(data + static_cast<long long>(c) * height * width, w, h, width);
        cnt++;
      }
    }
    top[index] = cnt == 0 ? 0.f : sum / cnt;
    top_count[index] = static_cast<float>(cnt);
  }
}

static int grid_dcn(long long total, int block) {
  long long b = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace mega

using namespace mega;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <bool BWD>
static int focal_loss_launch(const float* logits, const int* targets, const float* d_losses, int num_samples,
                             int num_classes, float gamma, float alpha, float* out, cudaStream_t stream) {
  const long long total = static_cast<long long>(num_samples) * num_classes;
  if (total == 0) return MEGA_OK;
  const bool vec = (num_classes & 3) == 0 && aligned16(logits) && aligned16(out) && (!BWD || aligned16(d_losses));
  if (vec)
    focal_loss_kernel<BWD, true><<<grid_dcn(total / 2, 256), 256, 0, stream>>>(total, logits, targets, d_losses,
                                                                               num_classes, gamma, alpha, out);
  else
    focal_loss_kernel<BWD, false><<<grid_dcn(total / 2, 256), 256, 0, stream>>>(total, logits, targets, d_losses,
                                                                                num_classes, gamma, alpha, out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_sigmoid_focalloss_forward(const float* logits, const int* targets, int num_samples,
                                              int num_classes, float gamma, float alpha, float* losses,
                                              void* stream_v) {
  return focal_loss_launch<false>(logits, targets, nullptr, num_samples, num_classes, gamma, alpha, losses,
                                  static_cast<cudaStream_t>(stream_v));
}

extern "C" int mega_sigmoid_focalloss_backward(const float* logits, const int* targets, const float* d_losses,
                                               int num_samples, int num_classes, float gamma, float alpha,
                                               float* d_logits, void* stream_v) {
  return focal_loss_launch<true>(logits, targets, d_losses, num_samples, num_classes, gamma, alpha, d_logits,
                                 static_cast<cudaStream_t>(stream_v));
}

extern "C" int mega_deform_im2col(const float* input, const float* offset, const float* mask, int batch, int channels,
                                  int height, int width, int kh, int kw, int pad_h, int pad_w, int stride_h,
                                  int stride_w, int dil_h, int dil_w, int deformable_group, int kpad, float* cols,
                                  void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(deformable_group >= 1 && channels % deformable_group == 0,
                 "deform_im2col: channels must divide into deformable groups");
  MEGA_ARG_CHECK(kpad >= channels * kh * kw, "deform_im2col: kpad smaller than C*kh*kw");
  const int ho = (height + 2 * pad_h - (dil_h * (kh - 1) + 1)) / stride_h + 1;
  const int wo = (width + 2 * pad_w - (dil_w * (kw - 1) + 1)) / stride_w + 1;
  const long long total = static_cast<long long>(batch) * channels * ho * wo;
  if (total == 0) return MEGA_OK;
  const int taps = kh * kw;
  if (taps <= kDcnMaxTaps) {
    const int cpg = channels / deformable_group;
    const long long blocks = static_cast<long long>(batch) * ho * deformable_group * ((cpg + kDcnCh - 1) / kDcnCh) *
                             ((wo + kDcnPix - 1) / kDcnPix);
    MEGA_ARG_CHECK(blocks < (1LL << 31), "deform_im2col: grid too large");
    const size_t smem = (static_cast<size_t>(taps) * kDcnPix * (sizeof(DcnTap) / 4 + 1) +
                         static_cast<size_t>(kDcnPix) * (kDcnCh * taps + 1)) * sizeof(float);
    static bool configured = false;
    if (!configured) {
      MEGA_CUDA_CHECK(cudaFuncSetAttribute(deform_im2col_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
      configured = true;
    }
    deform_im2col_tile_kernel<<<static_cast<unsigned>(blocks), 128, smem, stream>>>(
        input, offset, mask, channels, height, width, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w,
        deformable_group, ho, wo, kpad, cols);
    MEGA_CUDA_CHECK(cudaGetLastError());
    return MEGA_OK;
  }
  deform_im2col_kernel<<<grid_dcn(total, 256), 256, 0, stream>>>(total, input, offset, mask, batch, channels, height,
                                                                 width, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h,
                                                                 dil_w, deformable_group, ho, wo, kpad, cols);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_deform_psroi_pooling_forward(const float* input, const float* rois, const float* trans, int num_rois,
                                                 int channels, int height, int width, int no_trans, float spatial_scale,
                                                 int output_dim, int group_size, int pooled_size, int part_size,
                                                 int sample_per_part, float trans_std, int num_classes, float* out,
                                                 float* top_count, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const long long count = static_cast<long long>(num_rois) * output_dim * pooled_size * pooled_size;
  if (count == 0) return MEGA_OK;
  MEGA_ARG_CHECK(num_classes >= 1, "deform_psroi_pooling: num_classes must be >= 1");
  const int channels_each_class = no_trans ? output_dim : output_dim / num_classes;
  deform_psroi_fwd_kernel<<<grid_dcn(count, 256), 256, 0, stream>>>(
      count, input, spatial_scale, channels, height, width, pooled_size, pooled_size, rois, trans, no_trans, trans_std,
      sample_per_part, output_dim, group_size, part_size, num_classes, channels_each_class, out, top_count);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
