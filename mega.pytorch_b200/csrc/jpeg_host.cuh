// Host stage of the baseline JPEG decoder (SURVEY.md section 8f row 1): marker parsing and Huffman decoding, the part
// of the format that is serial. Plain C++ (no CUDA), written from ITU-T T.81; every read is checked against the end of
// the caller's buffer, every table index against the table, every coefficient write against the block count of the
// frame header. Output: mega_jpeg_info + quantised coefficients in natural order (see include/mega_b200.h).
// A stream is either decoded completely or refused with MEGA_JPEG_UNSUPPORTED / MEGA_JPEG_CORRUPT: where libjpeg would
// warn and guess (data after a marker, a missing restart marker), this refuses, and the caller lets Pillow decide.
#pragma once
#include <stdint.h>
#include <string.h>

#include "mega_b200.h"

#ifndef MEGA_OK                             // host-only builds do not see common.cuh
#define MEGA_OK 0
#define MEGA_ERR_ARG 1
#endif

namespace mega_jpeg {

constexpr int kMaxBlocks = 1 << 22;       // 2^28 samples: larger frames are refused as unsupported
// Largest sum of |dequantised coefficient| over one column of a block that is decoded here. The library Pillow uses
// runs the IDCT in 16-bit SIMD lanes: products, the sums in0 + in4 etc. and the values between the two passes
// (at most 5.66 x this sum) are int16 there and wrap or saturate beyond it, which the 32-bit arithmetic of
// jpeg_decode.cuh does not reproduce. Below this bound every intermediate of the row pass stays under 2^14 and
// both agree; an 8-bit image gives a few hundred to ~2000. Blocks above it are left to Pillow (MEGA_JPEG_CORRUPT).
constexpr int kMaxColumnSum = 2800;

static const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Huff {
  bool defined = false;
  uint16_t fast[1 << 10];      // 10-bit prefix -> (length << 8 | symbol), 0: no code of <= 10 bits
  uint32_t bound[17];          // codes of length l are < bound[l] when left-aligned in 16 bits
  int valoff[17];              // symbol index of a length-l code c: valoff[l] + c
  uint8_t vals[256];
  int nvals = 0;
};

// counts[16], then the symbols; false: over-subscribed, too many symbols, or a table libjpeg refuses
static inline bool build_huff(Huff& h, const uint8_t* counts, const uint8_t* symbols, int nsym) {
  if (nsym > 256) return false;
  memset(h.fast, 0, sizeof(h.fast));
  memcpy(h.vals, symbols, nsym);
  h.nvals = nsym;
  uint32_t code = 0;
  int k = 0, maxlen = 0;
  for (int len = 1; len <= 16; ++len)
    if (counts[len - 1]) maxlen = len;
  for (int len = 1; len <= 16; ++len) {
    h.valoff[len] = k - static_cast<int>(code);
    for (int i = 0; i < counts[len - 1]; ++i, ++code, ++k) {
      if (code >= (1u << len)) return false;
      if (len <= 10) {
        const uint32_t lo = code << (10 - len);
        for (uint32_t j = 0; j < (1u << (10 - len)); ++j) h.fast[lo + j] = static_cast<uint16_t>(len << 8 | symbols[k]);
      }
    }
    h.bound[len] = code << (16 - len);
    if (len <= maxlen && code >= (1u << len)) return false;   // as libjpeg: no code of a used length may be all ones
    code <<= 1;
  }
  h.defined = true;
  return true;
}

// Bit reader over one restart segment. Bytes are taken up to the next marker (or the end of the buffer) and never
// past it; after that zero bits are supplied and counted in `pad`, so "the data ran out" is `n < pad`.
struct Bits {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc = 0;            // left-aligned: the top n bits are valid
  int n = 0;
  int pad = 0;

  inline void fill() {
    while (n <= 56) {
      uint64_t b = 0;
      if (p < end && *p != 0xFF) {
        b = *p++;
      } else if (p + 1 < end && p[0] == 0xFF && p[1] == 0x00) {
        b = 0xFF;
        p += 2;
      } else if (pad < (1 << 20)) {
        pad += 8;
      }
      acc |= b << (56 - n);
      n += 8;
    }
  }
  inline uint32_t peek16() const { return static_cast<uint32_t>(acc >> 48); }
  inline void drop(int k) { acc <<= k, n -= k; }
  inline bool overrun() const { return n < pad; }
  // -1: invalid code
  inline int decode(const Huff& h) {
    fill();
    const uint32_t v = peek16();
    const uint16_t e = h.fast[v >> 6];
    if (e) {
      drop(e >> 8);
      return e & 255;
    }
    for (int len = 11; len <= 16; ++len) {
      if (v < h.bound[len]) {
        const int idx = h.valoff[len] + static_cast<int>(v >> (16 - len));
        if (idx < 0 || idx >= h.nvals) return -1;
        drop(len);
        return h.vals[idx];
      }
    }
    return -1;
  }
  // s in 1..15: s raw bits, sign-extended as T.81 F.2.2.1 does
  inline int receive_extend(int s) {
    fill();
    const int v = static_cast<int>(acc >> (64 - s));
    drop(s);
    return v >= (1 << (s - 1)) ? v : v - (1 << s) + 1;
  }
};

struct Component {
  int id, h, v, tq;
};

struct Decoder {
  const uint8_t* data;
  const uint8_t* end;
  mega_jpeg_info* info;
  int16_t* coef;               // null: headers only
  long long capacity;
  uint16_t qt[4][64];
  bool qt_defined[4] = {false, false, false, false};
  Huff dc[4], ac[4];
  Component comp[3];
  bool have_frame = false, jfif = false, adobe = false;
  int adobe_transform = 0;
  int restart = 0;
  bool done[3] = {false, false, false};

  static inline int be16(const uint8_t* p) { return p[0] << 8 | p[1]; }

  int frame(const uint8_t* s, int len) {
    if (have_frame || len < 6) return MEGA_JPEG_CORRUPT;
    if (s[0] != 8) return MEGA_JPEG_UNSUPPORTED;
    const int height = be16(s + 1), width = be16(s + 3), nc = s[5];
    if (nc != 1 && nc != 3) return MEGA_JPEG_UNSUPPORTED;
    if (len != 6 + 3 * nc || width == 0 || height == 0) return MEGA_JPEG_CORRUPT;
    for (int c = 0; c < nc; ++c) {
      comp[c] = Component{s[6 + 3 * c], s[7 + 3 * c] >> 4, s[7 + 3 * c] & 15, s[8 + 3 * c]};
      if (comp[c].tq > 3 || comp[c].h < 1 || comp[c].h > 4 || comp[c].v < 1 || comp[c].v > 4) return MEGA_JPEG_CORRUPT;
      for (int d = 0; d < c; ++d)
        if (comp[d].id == comp[c].id) return MEGA_JPEG_CORRUPT;
    }
    if (nc == 1) {
      comp[0].h = comp[0].v = 1;          // a lone component is never interleaved: its factors do not matter
    } else {
      const int h = comp[0].h, v = comp[0].v;
      if (!((h == 1 && v == 1) || (h == 2 && v == 1) || (h == 2 && v == 2))) return MEGA_JPEG_UNSUPPORTED;
      for (int c = 1; c < 3; ++c)
        if (comp[c].h != 1 || comp[c].v != 1) return MEGA_JPEG_UNSUPPORTED;
    }
    mega_jpeg_info& f = *info;
    memset(&f, 0, sizeof(f));
    f.width = width, f.height = height, f.ncomp = nc, f.hmax = comp[0].h, f.vmax = comp[0].v;
    f.mcus_x = (width + 8 * f.hmax - 1) / (8 * f.hmax);
    f.mcus_y = (height + 8 * f.vmax - 1) / (8 * f.vmax);
    long long off = 0;
    for (int c = 0; c < nc; ++c) {
      f.comp_dw[c] = (width * comp[c].h + f.hmax - 1) / f.hmax;
      f.comp_dh[c] = (height * comp[c].v + f.vmax - 1) / f.vmax;
      f.comp_bw[c] = f.mcus_x * comp[c].h;
      f.comp_bh[c] = f.mcus_y * comp[c].v;
      f.comp_block_off[c] = off;
      off += static_cast<long long>(f.comp_bw[c]) * f.comp_bh[c];
    }
    f.total_blocks = off;
    if (off > kMaxBlocks) return MEGA_JPEG_UNSUPPORTED;
    if (coef) {
      if (off > capacity) return MEGA_ERR_ARG;                    // the caller's buffer is smaller than this frame
      memset(coef, 0, static_cast<size_t>(off) * 64 * sizeof(int16_t));
    }
    have_frame = true;
    return MEGA_OK;
  }

  int tables_dqt(const uint8_t* s, int len) {
    int i = 0;
    while (i < len) {
      const int pq = s[i] >> 4, tq = s[i] & 15;
      ++i;
      if (pq > 1 || tq > 3 || i + 64 * (pq + 1) > len) return MEGA_JPEG_CORRUPT;
      for (int k = 0; k < 64; ++k) qt[tq][kZigzag[k]] = static_cast<uint16_t>(pq ? be16(s + i + 2 * k) : s[i + k]);
      qt_defined[tq] = true;
      i += 64 * (pq + 1);
    }
    return MEGA_OK;
  }

  int tables_dht(const uint8_t* s, int len) {
    int i = 0;
    while (i < len) {
      if (i + 17 > len) return MEGA_JPEG_CORRUPT;
      const int tc = s[i] >> 4, th = s[i] & 15;
      int total = 0;
      for (int k = 0; k < 16; ++k) total += s[i + 1 + k];
      if (tc > 1 || th > 3 || total > 256 || i + 17 + total > len) return MEGA_JPEG_CORRUPT;
      if (!build_huff(tc ? ac[th] : dc[th], s + i + 1, s + i + 17, total)) return MEGA_JPEG_CORRUPT;
      if (!tc)
        for (int k = 0; k < total; ++k)
          if (s[i + 17 + k] > 15) return MEGA_JPEG_CORRUPT;       // a DC symbol is a bit count
      i += 17 + total;
    }
    return MEGA_OK;
  }

  // one 8x8 block: false on an invalid code, a run past the block or a value no 8-bit encoder produces
  inline bool block(Bits& bits, const Huff& hd, const Huff& ha, const uint16_t* q, int& pred, int16_t* out) {
    int t = bits.decode(hd);
    if (t < 0 || t > 15) return false;
    if (t) pred += bits.receive_extend(t);
    if (pred < -32768 || pred > 32767) return false;
    int colsum[8] = {0, 0, 0, 0, 0, 0, 0, 0};     // sum of |dequantised coefficient| per column of the block
    colsum[0] = (pred < 0 ? -pred : pred) * static_cast<int>(q[0]);
    out[0] = static_cast<int16_t>(pred);
    for (int k = 1; k < 64;) {
      const int rs = bits.decode(ha);
      if (rs < 0) return false;
      const int r = rs >> 4, s = rs & 15;
      if (s) {
        k += r;
        if (k > 63) return false;
        const int v = bits.receive_extend(s);
        const int z = kZigzag[k];
        colsum[z & 7] += (v < 0 ? -v : v) * static_cast<int>(q[z]);
        if (colsum[z & 7] > kMaxColumnSum) return false;
        out[z] = static_cast<int16_t>(v);
        ++k;
      } else if (r == 15) {
        k += 16;
      } else {
        break;
      }
    }
    return colsum[0] <= kMaxColumnSum && !bits.overrun();
  }

  // entropy-coded data of one scan starting at p; on success *next is where marker parsing resumes
  int scan(const uint8_t* s, int len, const uint8_t* p, const uint8_t** next) {
    mega_jpeg_info& f = *info;
    if (!have_frame || len < 1) return MEGA_JPEG_CORRUPT;
    const int ns = s[0];
    if (ns < 1 || ns > f.ncomp || len != 4 + 2 * ns) return MEGA_JPEG_CORRUPT;
    if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return MEGA_JPEG_UNSUPPORTED;
    if (ns != 1 && ns != f.ncomp) return MEGA_JPEG_UNSUPPORTED;
    int ci[3], td[3], ta[3];
    for (int k = 0; k < ns; ++k) {
      ci[k] = -1;
      for (int c = 0; c < f.ncomp; ++c)
        if (comp[c].id == s[1 + 2 * k]) ci[k] = c;
      if (ci[k] < 0 || done[ci[k]]) return MEGA_JPEG_CORRUPT;
      for (int d = 0; d < k; ++d)
        if (ci[d] == ci[k]) return MEGA_JPEG_CORRUPT;
      td[k] = s[2 + 2 * k] >> 4, ta[k] = s[2 + 2 * k] & 15;
      if (td[k] > 3 || ta[k] > 3 || !dc[td[k]].defined || !ac[ta[k]].defined || !qt_defined[comp[ci[k]].tq])
        return MEGA_JPEG_CORRUPT;
      memcpy(f.quant[ci[k]], qt[comp[ci[k]].tq], sizeof(f.quant[0]));
    }
    int mx, my;
    if (ns == 1) {                          // non-interleaved: the component's own grid of true-size blocks
      mx = (f.comp_dw[ci[0]] + 7) / 8, my = (f.comp_dh[ci[0]] + 7) / 8;
    } else {
      mx = f.mcus_x, my = f.mcus_y;
    }
    const long long total = static_cast<long long>(mx) * my;
    long long mcu = 0;
    int rst = 0;
    while (mcu < total) {
      Bits bits;
      bits.p = p, bits.end = end;
      int pred[3] = {0, 0, 0};
      const long long stop = restart ? (mcu + restart < total ? mcu + restart : total) : total;
      for (; mcu < stop; ++mcu) {
        const int row = static_cast<int>(mcu / mx), col = static_cast<int>(mcu % mx);
        for (int k = 0; k < ns; ++k) {
          const int c = ci[k];
          const int hh = ns == 1 ? 1 : comp[c].h, vv = ns == 1 ? 1 : comp[c].v;
          for (int by = 0; by < vv; ++by)
            for (int bx = 0; bx < hh; ++bx) {
              const long long b = f.comp_block_off[c] + static_cast<long long>(row * vv + by) * f.comp_bw[c] + col * hh + bx;
              if (b < 0 || b >= f.total_blocks) return MEGA_JPEG_CORRUPT;
              if (!block(bits, dc[td[k]], ac[ta[k]], f.quant[c], pred[k], coef + b * 64)) return MEGA_JPEG_CORRUPT;
            }
        }
      }
      if (bits.n - bits.pad >= 8) return MEGA_JPEG_CORRUPT;       // whole bytes left in front of the marker
      p = bits.p;
      if (mcu < total) {                    // a restart marker must follow, in sequence
        while (p + 1 < end && p[0] == 0xFF && p[1] == 0xFF) ++p;
        if (p + 1 >= end || p[0] != 0xFF || p[1] != 0xD0 + rst) return MEGA_JPEG_CORRUPT;
        p += 2;
        rst = (rst + 1) & 7;
      }
    }
    for (int k = 0; k < ns; ++k) done[ci[k]] = true;
    *next = p;
    return MEGA_OK;
  }

  int run() {
    if (end - data < 4 || data[0] != 0xFF || data[1] != 0xD8) return MEGA_JPEG_CORRUPT;
    const uint8_t* p = data + 2;
    for (;;) {
      if (p >= end || *p != 0xFF) return MEGA_JPEG_CORRUPT;       // a marker must follow at once (fill bytes aside)
      while (p < end && *p == 0xFF) ++p;
      if (p >= end) return MEGA_JPEG_CORRUPT;
      const int m = *p++;
      if (m < 0xC0 || m == 0xDE || m == 0xDF || (m >= 0xF0 && m != 0xFE)) return MEGA_JPEG_CORRUPT;   // reserved / hierarchical: Pillow refuses
      if (m == 0xD9) return MEGA_JPEG_CORRUPT;                    // EOI before every component was decoded
      if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7)) return MEGA_JPEG_CORRUPT;   // SOI / RSTn outside a scan
      if (end - p < 2) return MEGA_JPEG_CORRUPT;
      const int len = be16(p);
      if (len < 2 || end - p < len) return MEGA_JPEG_CORRUPT;
      const uint8_t* s = p + 2;
      const int n = len - 2;
      p += len;
      int st = MEGA_OK;
      switch (m) {
        case 0xDB: st = tables_dqt(s, n); break;
        case 0xC4: st = tables_dht(s, n); break;
        case 0xC0:
        case 0xC1: st = frame(s, n); break;
        case 0xC2: case 0xC3: case 0xC5: case 0xC6: case 0xC7: case 0xC8: case 0xC9: case 0xCA: case 0xCB: case 0xCC:
        case 0xCD: case 0xCE: case 0xCF:
          return MEGA_JPEG_UNSUPPORTED;
        case 0xDD:
          if (n != 2) return MEGA_JPEG_CORRUPT;
          restart = be16(s);
          break;
        case 0xE0: jfif = jfif || (n >= 5 && memcmp(s, "JFIF\0", 5) == 0); break;
        case 0xEE:
          if (n >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = true, adobe_transform = s[11];
          break;
        case 0xDA: {
          if (!have_frame) return MEGA_JPEG_CORRUPT;
          if (!coef) return finish();
          st = scan(s, n, p, &p);
          if (st == MEGA_OK) {
            bool all = true;
            for (int c = 0; c < info->ncomp; ++c) all = all && done[c];
            if (all) {                       // EOI must follow: Pillow refuses a stream whose end is damaged
              while (p + 1 < end && p[0] == 0xFF && p[1] == 0xFF) ++p;
              if (p + 1 >= end || p[0] != 0xFF || p[1] != 0xD9) return MEGA_JPEG_CORRUPT;
              return finish();
            }
          }
          break;
        }
        default: break;                     // APPn, COM, DNL, ...: skipped by their length
      }
      if (st != MEGA_OK) return st;
    }
  }

  int finish() {
    mega_jpeg_info& f = *info;
    if (f.ncomp == 1)
      f.color = MEGA_JPEG_GREY;
    else if (jfif)
      f.color = MEGA_JPEG_YCBCR;
    else if (adobe)
      f.color = adobe_transform == 0 ? MEGA_JPEG_RGB : MEGA_JPEG_YCBCR;
    else
      f.color = (comp[0].id == 'R' && comp[1].id == 'G' && comp[2].id == 'B') ? MEGA_JPEG_RGB : MEGA_JPEG_YCBCR;
    return MEGA_OK;
  }
};

// coef == nullptr: headers only (mega_jpeg_probe)
static inline int decode_host(const uint8_t* data, long long size, mega_jpeg_info* info, int16_t* coef, long long capacity) {
  if (!data || size < 0 || !info) return MEGA_ERR_ARG;
  Decoder* d = new Decoder();               // ~12 KB of tables: kept off the (possibly small) thread stack
  d->data = data, d->end = data + size, d->info = info, d->coef = coef, d->capacity = capacity;
  const int st = d->run();
  delete d;
  return st;
}

}  // namespace mega_jpeg
