/* oracle_ops.c -- TEST INFRASTRUCTURE ONLY (never linked into or called by the product).
 *
 * Plain-C restatement of the reference's CPU custom ops, used as the parity checker:
 *   - oracle_nms            : greedy NMS      (mega_core/csrc/cpu/nms_cpu.cpp:6-65, and the
 *                                               CUDA variant's tie rule csrc/cuda/nms.cu:13-21,60)
 *   - oracle_roi_align_fwd  : ROIAlign forward (mega_core/csrc/cpu/ROIAlign_cpu.cpp:17-219,
 *                                               same arithmetic as csrc/cuda/ROIAlign_cuda.cu:16-122)
 * Pinned against the reference's own golden vectors (tests/test_nms.py) and against the
 * reference sources compiled verbatim into oracle/_ref (tests/test_oracle_cpu.py).
 *
 * Build: gcc -O2 -fPIC -shared -ffp-contract=off -o liboracle_ops.so oracle_ops.c -lm
 * (-ffp-contract=off: no FMA contraction, so float results match the reference build).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float score; int64_t idx; } scored_t;

/* descending by score; ties by ascending index (stable). A NaN score ranks above every number and NaNs tie with
 * each other, as in torch.sort(descending=True) and the device's key order (a positive NaN has the largest key). */
static int cmp_scored(const void* a, const void* b) {
  const scored_t* x = (const scored_t*)a;
  const scored_t* y = (const scored_t*)b;
  const int xn = isnan(x->score), yn = isnan(y->score);
  if (xn != yn) return xn ? -1 : 1;
  if (xn) return (x->idx > y->idx) - (x->idx < y->idx);
  if (x->score > y->score) return -1;
  if (x->score < y->score) return 1;
  return (x->idx > y->idx) - (x->idx < y->idx);
}

/* dets [n,4] xyxy, scores [n]; writes kept ORIGINAL indices in ascending order to keep_out,
 * returns their count. cuda_semantics=0: suppress when iou >= thr (nms_cpu.cpp:60);
 * cuda_semantics=1: suppress when iou > thr, areas recomputed per pair (nms.cu:13-21,60).
 * Both use the "+1" pixel convention. */
int64_t oracle_nms(const float* dets, const float* scores, int64_t n, float thr, int cuda_semantics,
                   int64_t* keep_out) {
  if (n <= 0) return 0;
  scored_t* order = (scored_t*)malloc(sizeof(scored_t) * (size_t)n);
  uint8_t* suppressed = (uint8_t*)calloc((size_t)n, 1);
  float* areas = (float*)malloc(sizeof(float) * (size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    order[i].score = scores[i];
    order[i].idx = i;
    areas[i] = (dets[i * 4 + 2] - dets[i * 4 + 0] + 1) * (dets[i * 4 + 3] - dets[i * 4 + 1] + 1);
  }
  qsort(order, (size_t)n, sizeof(scored_t), cmp_scored);
  for (int64_t _i = 0; _i < n; ++_i) {
    const int64_t i = order[_i].idx;
    if (suppressed[i]) continue;
    const float ix1 = dets[i * 4 + 0], iy1 = dets[i * 4 + 1], ix2 = dets[i * 4 + 2], iy2 = dets[i * 4 + 3];
    const float iarea = areas[i];
    for (int64_t _j = _i + 1; _j < n; ++_j) {
      const int64_t j = order[_j].idx;
      if (suppressed[j]) continue;
      const float xx1 = fmaxf(ix1, dets[j * 4 + 0]);
      const float yy1 = fmaxf(iy1, dets[j * 4 + 1]);
      const float xx2 = fminf(ix2, dets[j * 4 + 2]);
      const float yy2 = fminf(iy2, dets[j * 4 + 3]);
      if (cuda_semantics) {
        const float w = fmaxf(xx2 - xx1 + 1, 0.f), h = fmaxf(yy2 - yy1 + 1, 0.f);
        const float inter = w * h;
        const float iou = inter / (iarea + areas[j] - inter);
        if (iou > thr) suppressed[j] = 1;
      } else {
        const float w = fmaxf(0.f, xx2 - xx1 + 1), h = fmaxf(0.f, yy2 - yy1 + 1);
        const float inter = w * h;
        const float ovr = inter / (iarea + areas[j] - inter);
        if (ovr >= thr) suppressed[j] = 1;
      }
    }
  }
  int64_t m = 0;
  for (int64_t i = 0; i < n; ++i)
    if (!suppressed[i]) keep_out[m++] = i;
  free(order);
  free(suppressed);
  free(areas);
  return m;
}

static float bilinear(const float* data, int height, int width, float y, float x) {
  if (y < -1.0f || y > (float)height || x < -1.0f || x > (float)width) return 0.f;
  if (y <= 0) y = 0;
  if (x <= 0) x = 0;
  int y_low = (int)y, x_low = (int)x, y_high, x_high;
  if (y_low >= height - 1) { y_high = y_low = height - 1; y = (float)y_low; } else { y_high = y_low + 1; }
  if (x_low >= width - 1) { x_high = x_low = width - 1; x = (float)x_low; } else { x_high = x_low + 1; }
  const float ly = y - y_low, lx = x - x_low, hy = 1.f - ly, hx = 1.f - lx;
  const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
  return w1 * data[y_low * width + x_low] + w2 * data[y_low * width + x_high] +
         w3 * data[y_high * width + x_low] + w4 * data[y_high * width + x_high];
}

/* input NCHW [N,C,H,W]; rois [K,5] = (batch, x1, y1, x2, y2); out [K,C,ph,pw].
 * sampling_ratio <= 0 -> adaptive grid ceil(roi_size / pooled_size). */
void oracle_roi_align_fwd(const float* input, int channels, int height, int width, const float* rois,
                          int64_t num_rois, float spatial_scale, int pooled_h, int pooled_w,
                          int sampling_ratio, float* out) {
  for (int64_t n = 0; n < num_rois; ++n) {
    const float* roi = rois + n * 5;
    const int b = (int)roi[0];
    const float roi_start_w = roi[1] * spatial_scale, roi_start_h = roi[2] * spatial_scale;
    const float roi_end_w = roi[3] * spatial_scale, roi_end_h = roi[4] * spatial_scale;
    const float roi_width = fmaxf(roi_end_w - roi_start_w, 1.f);
    const float roi_height = fmaxf(roi_end_h - roi_start_h, 1.f);
    const float bin_h = roi_height / (float)pooled_h, bin_w = roi_width / (float)pooled_w;
    const int grid_h = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(roi_height / pooled_h);
    const int grid_w = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(roi_width / pooled_w);
    const float count = (float)(grid_h * grid_w);
    for (int c = 0; c < channels; ++c) {
      const float* plane = input + ((int64_t)b * channels + c) * height * width;
      for (int ph = 0; ph < pooled_h; ++ph) {
        for (int pw = 0; pw < pooled_w; ++pw) {
          float acc = 0.f;
          for (int iy = 0; iy < grid_h; ++iy) {
            const float y = roi_start_h + ph * bin_h + (iy + .5f) * bin_h / (float)grid_h;
            for (int ix = 0; ix < grid_w; ++ix) {
              const float x = roi_start_w + pw * bin_w + (ix + .5f) * bin_w / (float)grid_w;
              acc += bilinear(plane, height, width, y, x);
            }
          }
          out[((n * channels + c) * pooled_h + ph) * pooled_w + pw] = acc / count;
        }
      }
    }
  }
}
