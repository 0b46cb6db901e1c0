// Per-item bodies of the device stage of the JPEG decoder (SURVEY.md section 8f row 1): quantised coefficients ->
// the uint8 RGB pixels `PIL.Image.open(...).convert("RGB")` gives, i.e. libjpeg's default decode path (third-party
// code the reference reaches through Pillow and does not pin), restated from the algorithms:
//   * dequantise, then the integer Loeffler-Ligtenberg-Moschytz inverse DCT with 13-bit constants: a pass over the
//     columns descaled by 11 bits (2 fractional bits kept), a pass over the rows descaled by 18, then +128 and
//     saturation to 0..255. The host stage only passes blocks whose intermediates fit the library's 16-bit SIMD lanes
//     (jpeg_host.cuh: kMaxColumnSum), so 32-bit arithmetic here gives the same values. The library's shortcuts for columns / rows
//     without AC terms give the value of the full butterfly, so there is none here;
//   * chroma upsampling with the triangle filter: horizontally (3a + b + 1) >> 2 towards the left neighbour and
//     (3a + b + 2) >> 2 towards the right one; for 2x2 the vertical 3a + b first (the nearer row weighs 3), then
//     (3s + t + 8) >> 4 / (3s + t + 7) >> 4. The one-sided forms the library uses in the first and last column and
//     its repeated first / last row equal the same formulas with the neighbour index clamped to the component's TRUE
//     size, which is how they are written here; components at most 2 samples wide are replicated instead;
//   * YCbCr -> RGB in 16-bit fixed point: R = Y + ((91881 Cr' + 32768) >> 16), B = Y + ((116130 Cb' + 32768) >> 16),
//     G = Y + ((-22554 Cb' - 46802 Cr' + 32768) >> 16) with Cb' = Cb - 128, Cr' = Cr - 128, clamped to 0..255.
// oracle/jpeg_oracle.py is the numpy statement of the same arithmetic, pinned to Pillow bit for bit.
// Same __host__ __device__ arrangement as image_ops.cuh: the CPU tests run these bodies through a g++ build.
#pragma once
#include <stdint.h>

#include "mega_b200.h"

#if defined(__CUDACC__)
#define MEGA_JPEG_HD __host__ __device__ __forceinline__
#else
#define MEGA_JPEG_HD static inline
#endif

namespace mega_jpeg {

constexpr int kWsStride = 72;   // ints of intermediate per 8x8 block: 64 + 8 so that the 4 blocks of a warp use disjoint banks

// index of the image whose [start, next start) holds key; `start` picks the prefix (block_start or quad_start)
MEGA_JPEG_HD int find_image(const mega_jpeg_desc* descs, int n, long long key, long long mega_jpeg_desc::*start) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (descs[mid].*start <= key)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// position (r, c) of the 8x8 intermediate, rotated by the row so that column writes and row reads of the 8 threads of
// a block fall into 8 different shared-memory banks
MEGA_JPEG_HD int ws_index(int r, int c) { return r * 8 + ((c + r) & 7); }

// one 1-D pass; unsigned arithmetic so that a hand-built coefficient buffer wraps instead of overflowing
MEGA_JPEG_HD void idct_1d(const int* x, int shift, int* out) {
  typedef uint32_t u;
  const u x0 = x[0], x1 = x[1], x2 = x[2], x3 = x[3], x4 = x[4], x5 = x[5], x6 = x[6], x7 = x[7];
  u z1 = (x2 + x6) * 4433u;
  const u t2 = z1 - x6 * 15137u;
  const u t3 = z1 + x2 * 6270u;
  const u t0 = (x0 + x4) << 13, t1 = (x0 - x4) << 13;
  const u t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  u o0 = x7, o1 = x5, o2 = x3, o3 = x1;
  z1 = o0 + o3;
  u z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const u z5 = (z3 + z4) * 9633u;
  o0 *= 2446u, o1 *= 16819u, o2 *= 25172u, o3 *= 12299u;
  z1 *= static_cast<u>(-7373), z2 *= static_cast<u>(-20995);
  z3 = z3 * static_cast<u>(-16069) + z5, z4 = z4 * static_cast<u>(-3196) + z5;
  o0 += z1 + z3, o1 += z2 + z4, o2 += z2 + z3, o3 += z1 + z4;
  const u half = 1u << (shift - 1);
  out[0] = static_cast<int>(t10 + o3 + half) >> shift;
  out[7] = static_cast<int>(t10 - o3 + half) >> shift;
  out[1] = static_cast<int>(t11 + o2 + half) >> shift;
  out[6] = static_cast<int>(t11 - o2 + half) >> shift;
  out[2] = static_cast<int>(t12 + o1 + half) >> shift;
  out[5] = static_cast<int>(t12 - o1 + half) >> shift;
  out[3] = static_cast<int>(t13 + o0 + half) >> shift;
  out[4] = static_cast<int>(t13 - o0 + half) >> shift;
}

// +128 and saturation to 0..255, as the SIMD IDCT of the library Pillow ships does (its portable C path would wrap
// beyond +-512 instead; Pillow's pixels on x86-64 show the saturation)
MEGA_JPEG_HD int range_limit(int v) {
  v += 128;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// column `col` of one block: dequantise, first pass, into the block's intermediate ws[kWsStride]
MEGA_JPEG_HD void idct_column(const int16_t* coef, const unsigned short* quant, int col, int* ws) {
  int x[8], o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) x[k] = static_cast<int>(coef[k * 8 + col]) * static_cast<int>(quant[k * 8 + col]);
  idct_1d(x, 11, o);
#pragma unroll
  for (int k = 0; k < 8; ++k) ws[ws_index(k, col)] = o[k];
}

// row `row` of one block: second pass, range limit; the 8 samples packed little-endian (sample 0 in the low byte)
MEGA_JPEG_HD uint64_t idct_row(const int* ws, int row) {
  int x[8], o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) x[k] = ws[ws_index(row, k)];
  idct_1d(x, 18, o);
  uint64_t r = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) r |= static_cast<uint64_t>(range_limit(o[k])) << (8 * k);
  return r;
}

// where block b (batch-wide index) lives: its image, its coefficients, its 8 sample rows in the component plane
struct BlockPlace {
  const mega_jpeg_desc* d;
  int comp;
  long long plane_off;    // byte offset of the block's first sample in the plane workspace
  int stride;             // bytes between sample rows of the component plane
};

MEGA_JPEG_HD BlockPlace place_block(const mega_jpeg_desc* descs, int n, long long b) {
  const mega_jpeg_desc* d = descs + find_image(descs, n, b, &mega_jpeg_desc::block_start);
  const long long local = b - d->block_start;
  int c = 0;
  if (d->ncomp == 3) c = local >= d->comp_block_off[2] ? 2 : (local >= d->comp_block_off[1] ? 1 : 0);
  const long long in_comp = local - d->comp_block_off[c];
  const int by = static_cast<int>(in_comp / d->comp_bw[c]), bx = static_cast<int>(in_comp % d->comp_bw[c]);
  BlockPlace p;
  p.d = d, p.comp = c, p.stride = d->comp_bw[c] * 8;
  p.plane_off = (d->block_start + d->comp_block_off[c]) * 64 + static_cast<long long>(by) * 8 * p.stride + bx * 8;
  return p;
}

// sample (x, y) of the full-size image from a component subsampled by (hs, vs) in {1, 2}; dw x dh: its true size
MEGA_JPEG_HD int upsampled(const uint8_t* plane, int stride, int dw, int dh, int hs, int vs, int x, int y) {
  if (hs == 1) return plane[static_cast<long long>(y) * stride + x];
  if (dw <= 2) return plane[static_cast<long long>(y >> (vs - 1)) * stride + (x >> 1)];
  const int c = x >> 1, odd = x & 1;
  const int nb = odd ? (c + 1 < dw ? c + 1 : dw - 1) : (c > 0 ? c - 1 : 0);
  if (vs == 1) {
    const uint8_t* row = plane + static_cast<long long>(y) * stride;
    return (3 * row[c] + row[nb] + 1 + odd) >> 2;
  }
  const int r = y >> 1;
  const int rn = (y & 1) ? (r + 1 < dh ? r + 1 : dh - 1) : (r > 0 ? r - 1 : 0);
  const uint8_t* near = plane + static_cast<long long>(r) * stride;
  const uint8_t* far = plane + static_cast<long long>(rn) * stride;
  const int s = 3 * near[c] + far[c], t = 3 * near[nb] + far[nb];
  return (3 * s + t + 8 - odd) >> 4;
}

MEGA_JPEG_HD int clamp_u8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// colour work item q (batch-wide): 4 pixels of one row of one image, planar uint8 [3, H, W] out
MEGA_JPEG_HD void color_item(const mega_jpeg_desc* descs, int n, long long q, const uint8_t* planes, uint8_t* out) {
  const mega_jpeg_desc& d = descs[find_image(descs, n, q, &mega_jpeg_desc::quad_start)];
  const long long local = q - d.quad_start;
  const int y = static_cast<int>(local / d.quads_per_row), x0 = static_cast<int>(local % d.quads_per_row) * 4;
  const uint8_t* p0 = planes + (d.block_start + d.comp_block_off[0]) * 64;
  const int s0 = d.comp_bw[0] * 8;
  uint8_t px[3][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int x = x0 + i < d.width ? x0 + i : d.width - 1;          // lanes past the row repeat its last pixel; not stored
    const int yy = p0[static_cast<long long>(y) * s0 + x];
    if (d.color == MEGA_JPEG_GREY) {
      px[0][i] = px[1][i] = px[2][i] = static_cast<uint8_t>(yy);
      continue;
    }
    int c12[2];
#pragma unroll
    for (int c = 1; c < 3; ++c)
      c12[c - 1] = upsampled(planes + (d.block_start + d.comp_block_off[c]) * 64, d.comp_bw[c] * 8, d.comp_dw[c],
                             d.comp_dh[c], d.hmax, d.vmax, x, y);
    if (d.color == MEGA_JPEG_RGB) {
      px[0][i] = static_cast<uint8_t>(yy), px[1][i] = static_cast<uint8_t>(c12[0]), px[2][i] = static_cast<uint8_t>(c12[1]);
      continue;
    }
    const int cb = c12[0] - 128, cr = c12[1] - 128;
    px[0][i] = static_cast<uint8_t>(clamp_u8(yy + ((91881 * cr + 32768) >> 16)));
    px[1][i] = static_cast<uint8_t>(clamp_u8(yy + ((-22554 * cb - 46802 * cr + 32768) >> 16)));
    px[2][i] = static_cast<uint8_t>(clamp_u8(yy + ((116130 * cb + 32768) >> 16)));
  }
  const long long plane = static_cast<long long>(d.width) * d.height;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    uint8_t* o = out + d.out_off + c * plane + static_cast<long long>(y) * d.width + x0;
    if (x0 + 4 <= d.width && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
      *reinterpret_cast<uint32_t*>(o) = px[c][0] | px[c][1] << 8 | px[c][2] << 16 | static_cast<uint32_t>(px[c][3]) << 24;
    } else {
      for (int i = 0; i < 4 && x0 + i < d.width; ++i) o[i] = px[c][i];
    }
  }
}

// ---- host-side planning and validation (shared by the library and the host build used in the CPU tests)

static inline int plan_batch(const mega_jpeg_info* infos, int n, mega_jpeg_desc* descs, long long* totals) {
  long long blocks = 0, quads = 0, bytes = 0;
  for (int i = 0; i < n; ++i) {
    const mega_jpeg_info& f = infos[i];
    mega_jpeg_desc& d = descs[i];
    if (f.width <= 0 || f.height <= 0 || f.width > 65535 || f.height > 65535 || (f.ncomp != 1 && f.ncomp != 3) || f.total_blocks <= 0) return 1;
    if (!((f.hmax == 1 && f.vmax == 1) || (f.hmax == 2 && f.vmax == 1) || (f.hmax == 2 && f.vmax == 2))) return 1;
    if (f.color < MEGA_JPEG_GREY || f.color > MEGA_JPEG_RGB || (f.ncomp == 1) != (f.color == MEGA_JPEG_GREY)) return 1;
    long long off = 0;
    for (int c = 0; c < f.ncomp; ++c) {
      const int h = c == 0 ? f.hmax : 1, v = c == 0 ? f.vmax : 1;
      if (f.comp_dw[c] != (f.width * h + f.hmax - 1) / f.hmax || f.comp_dh[c] != (f.height * v + f.vmax - 1) / f.vmax) return 1;
      if (f.comp_bw[c] * 8 < f.comp_dw[c] || f.comp_bh[c] * 8 < f.comp_dh[c] || f.comp_block_off[c] != off) return 1;
      off += static_cast<long long>(f.comp_bw[c]) * f.comp_bh[c];
    }
    if (off != f.total_blocks) return 1;
    d.width = f.width, d.height = f.height, d.ncomp = f.ncomp, d.hmax = f.hmax, d.vmax = f.vmax, d.color = f.color;
    for (int c = 0; c < 3; ++c) {
      d.comp_dw[c] = f.comp_dw[c], d.comp_dh[c] = f.comp_dh[c], d.comp_bw[c] = f.comp_bw[c];
      d.comp_block_off[c] = f.comp_block_off[c];
      for (int k = 0; k < 64; ++k) d.quant[c][k] = f.quant[c][k];
    }
    d.quads_per_row = (f.width + 3) / 4;
    d.block_start = blocks, d.total_blocks = f.total_blocks, d.quad_start = quads, d.out_off = bytes;
    blocks += f.total_blocks;
    quads += static_cast<long long>(d.quads_per_row) * f.height;
    bytes += (3LL * f.width * f.height + 15) / 16 * 16;
  }
  totals[0] = blocks, totals[1] = quads, totals[2] = bytes;
  return 0;
}

// the descriptors are consistent with each other and with the buffer sizes: what the launch relies on
static inline bool batch_fits(const mega_jpeg_desc* descs, int n, long long planes_bytes, long long out_bytes,
                              long long* blocks, long long* quads) {
  long long b = 0, q = 0;
  for (int i = 0; i < n; ++i) {
    const mega_jpeg_desc& d = descs[i];
    if (d.width <= 0 || d.height <= 0 || d.width > 65535 || d.height > 65535) return false;   // JPEG's own limit
    if (d.block_start != b || d.quad_start != q || d.total_blocks <= 0) return false;
    if (d.color < MEGA_JPEG_GREY || d.color > MEGA_JPEG_RGB || (d.ncomp == 1) != (d.color == MEGA_JPEG_GREY)) return false;
    if (d.quads_per_row != (d.width + 3) / 4 || (d.ncomp != 1 && d.ncomp != 3) || d.hmax < 1 || d.hmax > 2 || d.vmax < 1 || d.vmax > d.hmax) return false;
    for (int c = 0; c < d.ncomp; ++c) {      // each component's region: whole block rows, enough of them, in order
      const int h = c == 0 ? d.hmax : 1, v = c == 0 ? d.vmax : 1;
      const int dw = (d.width * h + d.hmax - 1) / d.hmax, dh = (d.height * v + d.vmax - 1) / d.vmax;
      const long long begin = d.comp_block_off[c], end = c + 1 < d.ncomp ? d.comp_block_off[c + 1] : d.total_blocks;
      if (d.comp_dw[c] != dw || d.comp_dh[c] != dh || d.comp_bw[c] <= 0 || d.comp_bw[c] * 8 < dw) return false;
      if (begin < 0 || end < begin || (end - begin) % d.comp_bw[c] != 0) return false;
      if ((end - begin) / d.comp_bw[c] * 8 < dh) return false;
    }
    if (d.comp_block_off[0] != 0) return false;
    if (d.out_off < 0 || (d.out_off & 3) || d.out_off + 3LL * d.width * d.height > out_bytes) return false;
    b += d.total_blocks;
    q += static_cast<long long>(d.quads_per_row) * d.height;
  }
  if (b * 64 > planes_bytes) return false;
  *blocks = b, *quads = q;
  return true;
}

}  // namespace mega_jpeg
