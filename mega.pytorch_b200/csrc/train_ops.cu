// Training-side / non-VID entry points of the `mega_core._C` surface (SURVEY.md section 8b; 8f row 3):
//   mega_roi_align_backward_nchw          <- _C.roi_align_backward          (csrc/ROIAlign.h:27-45)
//   mega_roi_pool_forward / _backward     <- _C.roi_pool_forward / backward (csrc/ROIPool.h:11-47)
//   mega_deform_im2col_kq                 <- deformable_im2col              (deform_conv_kernel_cuda.cu:197-250, :578-640)
//   mega_deform_col2im_fused              <- deformable_col2im + deformable_col2im_coord (+ the modulated pair)
//   mega_channel_sum_nchw                 <- the grad_bias `ones` GEMM      (deform_conv_cuda.cu:667-672)
//   mega_deform_psroi_pooling_backward    <- _C.deform_psroi_pooling_backward (csrc/deform_pool.h:41-69)
// The per-item bodies live in train_ops.cuh (shared with the host build that the CPU tests check against the oracle);
// the kernels below are grid-stride loops over items, sized to a multiple of the 132 SMs. All of them are HBM / L2
// atomic bound: items are numbered so that a warp touches consecutive addresses of one plane.
#include "common.cuh"
#include "mega_b200.h"
#include "train_ops.cuh"

namespace mega {

using namespace mega_train;

struct RedAdd {
  __device__ __forceinline__ void operator()(float* p, float v) const { atomicAdd(p, v); }   // result unused: RED.ADD
};

__global__ void roi_align_bwd_kernel(long long items, const float* __restrict__ grad, const float* __restrict__ rois,
                                     float spatial_scale, int channels, int height, int width, int pooled_h,
                                     int pooled_w, int sampling_ratio, float* __restrict__ grad_in) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    roi_align_bwd_item(i, grad, rois, spatial_scale, channels, height, width, pooled_h, pooled_w, sampling_ratio,
                       grad_in, RedAdd());
}

__global__ void roi_pool_fwd_kernel(long long total, const float* __restrict__ input, const float* __restrict__ rois,
                                    float spatial_scale, int channels, int height, int width, int pooled_h,
                                    int pooled_w, float* __restrict__ out, int* __restrict__ argmax) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    roi_pool_fwd_item(i, input, rois, spatial_scale, channels, height, width, pooled_h, pooled_w, out, argmax);
}

__global__ void roi_pool_bwd_kernel(long long total, const float* __restrict__ grad, const int* __restrict__ argmax,
                                    const float* __restrict__ rois, int channels, int height, int width, int pooled_h,
                                    int pooled_w, float* __restrict__ grad_in) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    roi_pool_bwd_item(i, grad, argmax, rois, channels, height, width, pooled_h, pooled_w, grad_in, RedAdd());
}

__global__ void dcn_im2col_kq_kernel(long long total, DcnGeom g, const float* __restrict__ im,
                                     const float* __restrict__ offset, const float* __restrict__ mask,
                                     float* __restrict__ cols) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dcn_im2col_kq_item(i, g, im, offset, mask, cols);
}

__global__ void dcn_col2im_fused_kernel(long long total, DcnGeom g, const float* __restrict__ gcols,
                                        const float* __restrict__ im, const float* __restrict__ offset,
                                        const float* __restrict__ mask, float* __restrict__ grad_im,
                                        float* __restrict__ grad_offset, float* __restrict__ grad_mask) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dcn_col2im_fused_item(i, g, gcols, im, offset, mask, grad_im, grad_offset, grad_mask, RedAdd());
}

// one warp per channel: lanes stride the plane (coalesced), butterfly reduction, lane 0 accumulates into out[c]
__global__ void channel_sum_nchw_kernel(const float* __restrict__ x, int batch, int channels, int p_total,
                                        float* __restrict__ out) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int c = blockIdx.x * warps_per_block + (threadIdx.x >> 5); c < channels; c += gridDim.x * warps_per_block) {
    float s = 0.f;
    for (int b = 0; b < batch; ++b) {
      const float* row = x + (static_cast<long long>(b) * channels + c) * p_total;
      for (int p = lane; p < p_total; p += 32) s += row[p];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[c] += s;
  }
}

__global__ void deform_psroi_bwd_kernel(long long total, PsRoiGeom g, const float* __restrict__ top_diff,
                                        const float* __restrict__ top_count, const float* __restrict__ data,
                                        const float* __restrict__ rois, const float* __restrict__ trans,
                                        float* __restrict__ grad_in, float* __restrict__ grad_trans) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    deform_psroi_bwd_item(i, g, top_diff, top_count, data, rois, trans, grad_in, grad_trans, RedAdd());
}

static int grid_for(long long total, int block) {
  long long b = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

static int dcn_geom(DcnGeom* g, int batch, int channels, int height, int width, int kh, int kw, int pad_h, int pad_w,
                    int stride_h, int stride_w, int dil_h, int dil_w, int deformable_group, int ldp) {
  MEGA_ARG_CHECK(batch >= 0 && channels > 0 && height > 0 && width > 0 && kh > 0 && kw > 0 && stride_h > 0 &&
                     stride_w > 0 && dil_h > 0 && dil_w > 0,
                 "deform_conv: bad geometry");
  MEGA_ARG_CHECK(deformable_group >= 1 && channels % deformable_group == 0,
                 "deform_conv: channels must divide into deformable groups");
  g->batch = batch, g->channels = channels, g->height = height, g->width = width;
  g->kh = kh, g->kw = kw, g->pad_h = pad_h, g->pad_w = pad_w, g->stride_h = stride_h, g->stride_w = stride_w;
  g->dil_h = dil_h, g->dil_w = dil_w, g->deformable_group = deformable_group;
  g->ho = (height + 2 * pad_h - (dil_h * (kh - 1) + 1)) / stride_h + 1;
  g->wo = (width + 2 * pad_w - (dil_w * (kw - 1) + 1)) / stride_w + 1;
  MEGA_ARG_CHECK(g->ho > 0 && g->wo > 0, "deform_conv: empty output");
  MEGA_ARG_CHECK(ldp >= g->ho * g->wo, "deform_conv: ldp smaller than Ho*Wo");
  g->ldp = ldp;
  return MEGA_OK;
}

}  // namespace mega

using namespace mega;

extern "C" int mega_roi_align_backward_nchw(const float* grad, const float* rois, int num_rois, float spatial_scale,
                                            int pooled_h, int pooled_w, int batch, int channels, int height, int width,
                                            int sampling_ratio, float* grad_input, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  (void)batch;
  MEGA_ARG_CHECK(pooled_h > 0 && pooled_w > 0 && channels > 0 && height > 0 && width > 0,
                 "roi_align_backward: bad pooled size / shape");
  const long long items = roi_align_bwd_items(num_rois, channels, pooled_h, pooled_w);
  if (items == 0) return MEGA_OK;   // ROIAlign_cuda.cu:324-327: empty gradient, grad_input stays zero
  roi_align_bwd_kernel<<<grid_for(items, 256), 256, 0, stream>>>(items, grad, rois, spatial_scale, channels, height,
                                                                 width, pooled_h, pooled_w, sampling_ratio, grad_input);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_roi_pool_forward(const float* input, const float* rois, int num_rois, float spatial_scale,
                                     int channels, int height, int width, int pooled_h, int pooled_w, float* output,
                                     int* argmax, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(pooled_h > 0 && pooled_w > 0 && channels > 0, "roi_pool: bad pooled size / channels");
  const long long total = static_cast<long long>(num_rois) * channels * pooled_h * pooled_w;
  if (total == 0) return MEGA_OK;
  roi_pool_fwd_kernel<<<grid_for(total, 256), 256, 0, stream>>>(total, input, rois, spatial_scale, channels, height,
                                                                width, pooled_h, pooled_w, output, argmax);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_roi_pool_backward(const float* grad, const int* argmax, const float* rois, int num_rois,
                                      int channels, int height, int width, int pooled_h, int pooled_w,
                                      float* grad_input, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(pooled_h > 0 && pooled_w > 0 && channels > 0, "roi_pool_backward: bad pooled size / channels");
  const long long total = static_cast<long long>(num_rois) * channels * pooled_h * pooled_w;
  if (total == 0) return MEGA_OK;
  roi_pool_bwd_kernel<<<grid_for(total, 256), 256, 0, stream>>>(total, grad, argmax, rois, channels, height, width,
                                                                pooled_h, pooled_w, grad_input);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_deform_im2col_kq(const float* input, const float* offset, const float* mask, int batch,
                                     int channels, int height, int width, int kh, int kw, int pad_h, int pad_w,
                                     int stride_h, int stride_w, int dil_h, int dil_w, int deformable_group, int ldp,
                                     float* cols, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  DcnGeom g;
  const int st = dcn_geom(&g, batch, channels, height, width, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w,
                          deformable_group, ldp);
  if (st != MEGA_OK) return st;
  const long long total = static_cast<long long>(channels) * batch * g.ho * g.wo;
  if (total == 0) return MEGA_OK;
  dcn_im2col_kq_kernel<<<grid_for(total, 256), 256, 0, stream>>>(total, g, input, offset, mask, cols);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_deform_col2im_fused(const float* gcols, const float* input, const float* offset, const float* mask,
                                        int batch, int channels, int height, int width, int kh, int kw, int pad_h,
                                        int pad_w, int stride_h, int stride_w, int dil_h, int dil_w,
                                        int deformable_group, int ldp, float* grad_input, float* grad_offset,
                                        float* grad_mask, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  DcnGeom g;
  const int st = dcn_geom(&g, batch, channels, height, width, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w,
                          deformable_group, ldp);
  if (st != MEGA_OK) return st;
  MEGA_ARG_CHECK((mask == nullptr) == (grad_mask == nullptr), "deform_col2im: mask and grad_mask go together");
  const long long total = static_cast<long long>(batch) * deformable_group * kh * kw * g.ho * g.wo;
  if (total == 0) return MEGA_OK;
  dcn_col2im_fused_kernel<<<grid_for(total, 128), 128, 0, stream>>>(total, g, gcols, input, offset, mask, grad_input,
                                                                    grad_offset, grad_mask);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_channel_sum_nchw(const float* x, int batch, int channels, int plane, float* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (batch <= 0 || channels <= 0 || plane <= 0) return MEGA_OK;
  const int warps = 8;
  int blocks = (channels + warps - 1) / warps;
  if (blocks > 132 * 8) blocks = 132 * 8;
  channel_sum_nchw_kernel<<<blocks, warps * 32, 0, stream>>>(x, batch, channels, plane, out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_deform_psroi_pooling_backward(const float* out_grad, const float* input, const float* rois,
                                                  const float* trans, const float* top_count, int num_rois,
                                                  int channels, int height, int width, int no_trans,
                                                  float spatial_scale, int output_dim, int group_size, int pooled_size,
                                                  int part_size, int sample_per_part, float trans_std, int num_classes,
                                                  float* input_grad, float* trans_grad, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const long long total = static_cast<long long>(num_rois) * output_dim * pooled_size * pooled_size;
  if (total == 0) return MEGA_OK;
  MEGA_ARG_CHECK(num_classes >= 1, "deform_psroi_pooling_backward: num_classes must be >= 1");
  MEGA_ARG_CHECK(no_trans || (trans != nullptr && trans_grad != nullptr),
                 "deform_psroi_pooling_backward: trans / trans_grad missing");
  PsRoiGeom g;
  g.channels = channels, g.height = height, g.width = width, g.pooled = pooled_size, g.output_dim = output_dim;
  g.group_size = group_size, g.part_size = part_size, g.sample_per_part = sample_per_part;
  g.num_classes = num_classes, g.no_trans = no_trans ? 1 : 0;
  g.channels_each_class = no_trans ? output_dim : output_dim / num_classes;
  g.spatial_scale = spatial_scale, g.trans_std = trans_std;
  MEGA_ARG_CHECK(g.channels_each_class >= 1, "deform_psroi_pooling_backward: output_dim smaller than num_classes");
  deform_psroi_bwd_kernel<<<grid_for(total, 256), 256, 0, stream>>>(total, g, out_grad, top_count, input, rois, trans,
                                                                    input_grad, trans_grad);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}
