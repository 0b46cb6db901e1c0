// Implicit-GEMM convolution / GEMM on the Hopper tensor cores (wgmma, TF32 / FP16 operands,
// FP32 accumulate in registers), fed by TMA with the 128-byte shared-memory swizzle.
//
// One kernel serves every dense contraction of the MEGA hot path:
//   * backbone / res5 / RPN-head convolutions (1x1, 3x3, 3x3 dilated) over NHWC maps
//     (reference: mega_core/modeling/backbone/resnet.py:324-344, rpn/rpn.py:99-106),
//     with FrozenBatchNorm scale/bias (layers/batch_norm.py:26-31), residual add and ReLU
//     folded into the epilogue;
//   * Linear layers (make_layers.py:80-92) as a 1x1 "convolution" over an H=1 image;
//   * the per-head Q.K^T and P.V' products of the relation module
//     (roi_box_feature_extractors.py:602-646) through the batch (grid.z) offsets.
//
// Tiling: the M tile is a th x tw rectangle of 128 output pixels, so the A operand of filter
// tap (r,s) is the same rectangle shifted by (r,s)*dilation - pad: a plain 4-D tiled TMA load
// with out-of-bounds zero fill supplies the padding. K is consumed in slabs of 32 floats
// (= one 128 B swizzle row) per tap. Warp roles: warp 0 TMA producer, warp 1 barrier init, warps 2-5 epilogue
// (accumulator ring -> registers -> global); 3xTF32 adds warps 6-9, the operand splitters. Two MMA warpgroups follow the
// last of these warps (kMmaWarp0): warpgroup g issues the wgmma of tile rows [64 g, 64 g + 64) and keeps that accumulator
// in registers.
// 3xFP16 (split-fp16 tensors, the mode the strict engine runs; see kModeF16x3 below) keeps each role in whole warpgroups
// and moves registers between them with setmaxnreg (512 threads start at 128 registers each): warpgroup 0 (warps 0-3:
// producer, barrier init, two idle warps) drops to 40, warpgroup 1 (warps 4-7: the epilogue) to 104, and the two MMA
// warpgroups (warps 8-15) rise to 184, so that the wgmma accumulator and the round-to-nearest master accumulator (64 + 64
// registers per thread at block_n 128) stay in registers.
#include "common.cuh"
#pragma once
#include "mega_b200.h"
#include "wgmma.cuh"

namespace mega {

constexpr int kBM = 128;        // M tile of one CTA (two m64 warpgroups)
// operand arithmetic of a launch
constexpr int kModeTf32 = 0;    // fp32 operands in HBM, rounded to TF32 by the TMA load; K slab = 32 floats
constexpr int kModeSplit3 = 1;  // "3xTF32": fp32 operands split hi/lo in shared memory
constexpr int kModeF16 = 2;     // fp16 operands in HBM (10-bit mantissa like TF32, half the bytes, twice the
                                // tensor-pipe rate); K slab = 64 halves
constexpr int kModeF16x3 = 3;   // "3xFP16": operands stored SPLIT in HBM -- every group of 32 K-values is one 128-byte row
                                // [32 hi halves | 32 lo halves] with hi = fp16(x), lo = fp16(x - hi): the same 4 bytes per
                                // value as fp32 and 22 mantissa bits like 3xTF32, but NO split work in the kernel (the
                                // producing epilogue / the weight packer did it) and kind::f16 MMAs; K slab = 32 values
// every mode stages K slabs of 128 bytes per row (one swizzle row) and issues 4 MMAs of 32 bytes of K each
// (3xFP16: 2 k-steps x 3 products over the hi / lo halves of the row; 3xTF32: 4 k-steps x 3 products)
__host__ __device__ constexpr int mode_bk(int mode) { return mode == kModeF16 ? 64 : 32; }
constexpr int kThreads = 192;   // 6 warps before the MMA warpgroups (10 in the 3xTF32 mode)
constexpr int kMaxCtas = 132;   // persistent grid: one CTA per SM of an H100 SXM
// The MMA warpgroups hand finished accumulators to the epilogue warps through a ring of shared-memory slots of 32 columns
// x 128 rows fp32 (row r = 128 bytes, 16-byte groups swizzled by r & 7: conflict-free for both sides). Every slot is read by
// four epilogue warps (one per 32-row quarter) and produced in column order, tile after tile.
constexpr int kRingSlots = 2;
constexpr int kRingSlotBytes = kBM * 128;
// 3xFP16 holds a whole tile in its ring (chunk c of every tile in slot c), so that the MMA warpgroups hand over a finished
// tile without waiting for the epilogue of the one before; the epilogue writes its result in place, into the rows it read.
__host__ __device__ constexpr int ring_slots(int mode, int bn) { return mode == kModeF16x3 ? bn / 32 : kRingSlots; }
__host__ __device__ constexpr int mma_warp0(int mode) { return mode == kModeSplit3 ? 12 : 8; }
__host__ __device__ constexpr int conv_gemm_threads(int mode) { return (mma_warp0(mode) + 8) * 32; }
// 3xFP16 registers per thread of warpgroup 0 (producer), 1 (epilogue) and 2-3 (MMA): the 64K registers of the SM
constexpr int kF16x3RegsProducer = 40, kF16x3RegsEpilogue = 104, kF16x3RegsMma = 184;
static_assert(128 * kF16x3RegsProducer + 128 * kF16x3RegsEpilogue + 256 * kF16x3RegsMma == 65536 &&
                  conv_gemm_threads(kModeF16x3) == 512,
              "3xFP16 register split");
// An N tile wider than 128 columns is computed in two passes over the same k-blocks (columns [0, P0), then [P0, block_n)):
// a pass keeps at most 64 accumulator registers per MMA thread. Both widths are multiples of 32 (whole ring chunks).
__host__ __device__ constexpr int pass_n(int bn) { return bn <= 128 ? bn : (bn == 160 ? 96 : bn / 2); }
// Pipeline stages of the (mode, block_n) kernel, grouped launches (block_n 64) included; conv_gemm_kernel checks that they
// fit the 227 KB of shared memory next to the ring and the epilogue staging.
constexpr int conv_gemm_stages(int mode, int bn) {
  if (mode == kModeSplit3) return bn == 64 ? 4 : 2;
  if (mode == kModeF16x3) return bn == 64 ? 6 : 4;
  return bn == 32 ? 6 : bn == 64 ? 5 : bn <= 128 ? 4 : bn <= 192 ? 3 : 2;
}

struct ConvGemmParams {
  int tiles_w, tiles_h, tile_w, tile_h;
  int out_h, out_w, n_img;
  int taps_r, taps_s, dil, pad;
  int pad_w;                  // left padding (pad applies to the rows)
  int stride_h, stride_w;     // convolution stride: output (h, w) reads input (h*stride_h + r*dil - pad, ...)
  int k_chunks;  // ceil(Cin / BK)
  int cout;
  const float* scale;
  const float* bias;
  int has_residual;
  int relu;
  int a_c_off, a_n_off, b_k_off, b_n_off;
  int out_c_off, out_n_off;   // per-batch coordinate offsets of the output / residual tensors
  int res_c_off, res_n_off;
  int bias_z_off;
  int box_w, box_h;           // per-warp store box: 32 output pixels = box_h x box_w
  // stream-K decomposition
  int m_tiles, n_tiles;      // per batch entry
  int kb_per_tile;           // taps * k_chunks
  long long total_units;     // batch * m_tiles * n_tiles * kb_per_tile
  long long total_tiles;     // batch * m_tiles * n_tiles
  int stream_k;              // 1: k-block granular split across CTAs, 0: whole tiles round-robin
  int n_fast;                // 3xFP16 whole-tile launches only: tiles ordered with the n-tile fastest (decode_tile)
  float* part_ws;            // [grid][2][128][BN] partial accumulators
  int* counters;             // [tiles], zero between launches
  int seg_len;               // 3xTF32 / 3xFP16: k-blocks accumulated by the tensor core before the RN fold into the master accumulator
  int b_lo_tap_off;          // 3xTF32 only: > 0: B's low parts are stored as taps [b_lo_tap_off, 2 * b_lo_tap_off) of the B tensor
  int res_split;             // 3xFP16 only: the residual tensor is in the split-fp16 format (else fp32)
  float acc_scale;           // 3xFP16 only: the accumulator is multiplied by this power of two first (weights are stored
                             // scaled by its inverse so that their low halves stay normal fp16 numbers)
  // The TMA unit clips a store's innermost (channel) extent at 16-byte granularity. tmOut therefore ends at out_tail0, the
  // last 16-byte boundary at or before the channel extent out_cext; the channels [out_tail0, out_cext) of a pixel are
  // written with plain stores (store_tail), so that nothing past out_cext changes.
  void* out_ptr;
  long long out_ld, out_str_h, out_str_n;   // element strides of the output pixels / rows / images
  int out_tail0, out_cext;
};

template <int BN, int STAGES, int MODE = kModeTf32>
struct SmemLayout {
  static constexpr bool SPLIT3 = MODE == kModeSplit3;
  static constexpr int kABytes = kBM * 128;
  static constexpr int kBBytes = pass_n(BN) * 128;     // B rows of one pass
  static constexpr int kHalf = kABytes + kBBytes;                 // bytes the two TMA loads of a k-block deliver
  // 3xTF32: [A raw | B hi (masked in place by the splitters) | B lo]; the MMA warpgroups split A in registers
  static constexpr int kStageBytes = SPLIT3 ? kHalf + kBBytes : kHalf;
  static constexpr int kRingOffset = STAGES * kStageBytes;
  static constexpr int kEpiOffset = kRingOffset + ring_slots(MODE, BN) * kRingSlotBytes;
  // 4 warps x (2 out + 2 residual) x 4 KB (3xFP16: 4 warps x 2 residual x 4 KB; its results go back into the ring)
  static constexpr int kEpiBytes = MODE == kModeF16x3 ? 4 * 2 * 4096 : 4 * 4 * 4096;
  static constexpr int kBarOffset = kEpiOffset + kEpiBytes;
  static constexpr int kSbCols = BN <= 128 ? 128 : 256;
  static constexpr int kSbOffset = kBarOffset + 512;              // [scale | bias][kSbCols] floats of the tile being finished
  static constexpr int kTotal = kSbOffset + 8 * kSbCols + 1024;   // + align slack
};

struct TileCoord {
  int img, h0, w0, n0, batch;
};

// Work-list indices are 32-bit (the host checks total_units * grid < 2^31): 64-bit divisions cost hundreds of cycles
// on the single-thread critical paths of the producer / MMA roles.
// Tiles are ordered (batch, n-tile, m-tile) with m fastest, or, with n_fast, (batch, m-tile, n-tile) with n fastest.
__device__ __forceinline__ TileCoord decode_tile(const ConvGemmParams& p, int t, int bn, bool n_fast = false) {
  TileCoord c;
  int m_tile, n_tile;
  if (n_fast) {
    n_tile = t % p.n_tiles;
    const int rest = t / p.n_tiles;
    m_tile = rest % p.m_tiles;
    c.batch = rest / p.m_tiles;
  } else {
    m_tile = t % p.m_tiles;
    const int rest = t / p.m_tiles;
    n_tile = rest % p.n_tiles;
    c.batch = rest / p.n_tiles;
  }
  const int tw_i = m_tile % p.tiles_w;
  const int th_i = (m_tile / p.tiles_w) % p.tiles_h;
  c.img = m_tile / (p.tiles_w * p.tiles_h);
  c.h0 = th_i * p.tile_h;
  c.w0 = tw_i * p.tile_w;
  c.n0 = n_tile * bn;
  return c;
}

__device__ __forceinline__ int cta_first_unit(int total, int grid, int c) {
  return static_cast<int>((static_cast<unsigned>(total) * static_cast<unsigned>(c)) / static_cast<unsigned>(grid));
}

// the CTA whose unit range [first(c), first(c+1)) contains unit u
__device__ __forceinline__ int unit_owner(int total, int grid, int u) {
  int c = static_cast<int>((static_cast<unsigned>(u) * static_cast<unsigned>(grid)) / static_cast<unsigned>(total));
  if (c >= grid) c = grid - 1;
  while (c + 1 < grid && cta_first_unit(total, grid, c + 1) <= u) ++c;
  while (c > 0 && cta_first_unit(total, grid, c) > u) --c;
  return c;
}

// the (tile, k-block range) items of one CTA, identical for the three warp roles
struct WorkIter {
  int u, u_end, tile, tiles;
  int KB, grid;
  bool sk;
  __device__ __forceinline__ WorkIter(const ConvGemmParams& p, int cta, int grid_)
      : tile(cta), tiles(static_cast<int>(p.total_tiles)), KB(p.kb_per_tile), grid(grid_), sk(p.stream_k != 0) {
    u = cta_first_unit(static_cast<int>(p.total_units), grid_, cta);
    u_end = cta_first_unit(static_cast<int>(p.total_units), grid_, cta + 1);
  }
  __device__ __forceinline__ bool next(int& t, int& kb0, int& kb1) {
    if (sk) {
      if (u >= u_end) return false;
      t = u / KB;
      kb0 = u - t * KB;
      kb1 = min(KB, kb0 + (u_end - u));
      u += kb1 - kb0;
      return true;
    }
    if (tile >= tiles) return false;
    t = tile;
    kb0 = 0;
    kb1 = KB;
    tile += grid;
    return true;
  }
  // the tile of the item next() returns next
  __device__ __forceinline__ bool peek(int& t) const {
    if (sk) {
      t = u / KB;
      return u < u_end;
    }
    t = tile;
    return tile < tiles;
  }
};

// named barrier of the THREADS epilogue threads
template <int THREADS>
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(THREADS) : "memory"); }

// ------------------------------------------------------------------ stream-K fix-up
// A tile whose k-blocks straddle CTAs c_first .. c_last is finished by the last of them to arrive. Each publishes its partial
// accumulator to part_ws[cta][slot][kBM][bn]. Only the first and the last work item of a CTA's unit range can be partial, so
// two slots per CTA suffice: slot 0 holds the CTA's first item, slot 1 any later one. The finisher derives the slot of CTA
// oc's part of tile t from where oc's range starts (inside t: t was its first item), and sums the parts in CTA order, so
// the result does not depend on which CTA arrives last.
__device__ __forceinline__ float* sk_part_row(const ConvGemmParams& p, int c, int slot, int row, int bn) {
  return p.part_ws + ((static_cast<long long>(c) * 2 + slot) * kBM + row) * bn;
}

// tile row `row` of this CTA's part of its tile_item-th work item
__device__ __forceinline__ float* sk_own_part_row(const ConvGemmParams& p, int cta, int tile_item, int row, int bn) {
  return sk_part_row(p, cta, tile_item == 0 ? 0 : 1, row, bn);
}

// columns [col0, col0 + 32) of a row of this CTA's part (callers take `part` from sk_own_part_row once per item, before
// they wait for their first chunk: computed after the wait, the address costs the 3xFP16 epilogue spills)
__device__ __forceinline__ void sk_publish(float* part, int col0, const uint32_t (&acc)[32]) {
  float* ws = part + col0;
#pragma unroll
  for (int j = 0; j < 32; j += 4)
    __stcg(reinterpret_cast<float4*>(ws + j), make_float4(__uint_as_float(acc[j]), __uint_as_float(acc[j + 1]),
                                                          __uint_as_float(acc[j + 2]), __uint_as_float(acc[j + 3])));
}

// Called by all THREADS epilogue threads once they have published their chunks of tile t. Counts this CTA's arrival; the
// last of the c_first .. c_last arrivals resets the counter for the next launch. True in every thread of the finisher.
template <int THREADS>
__device__ __forceinline__ bool sk_elect_finisher(const ConvGemmParams& p, int U, int grid, int KB, int t, int epi_tid,
                                                  int* flag, int& c_first, int& c_last) {
  __threadfence();
  epi_bar_sync<THREADS>();
  c_first = unit_owner(U, grid, t * KB);
  c_last = unit_owner(U, grid, t * KB + KB - 1);
  if (epi_tid == 0) {
    const int parts = c_last - c_first + 1;
    const int old = atomicAdd(&p.counters[t], 1);
    const int last = (old == parts - 1);
    if (last) p.counters[t] = 0;
    *flag = last;
  }
  epi_bar_sync<THREADS>();
  const bool finisher = *flag != 0;
  if (finisher) __threadfence();
  return finisher;
}

// columns [col0, col0 + 32) of tile row `row` of tile t: the parts of CTAs c_first .. c_last summed in CTA order
__device__ __forceinline__ void sk_reduce(const ConvGemmParams& p, int U, int grid, int KB, int t, int c_first, int c_last,
                                          int row, int bn, int col0, float (&acc)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int oc = c_first; oc <= c_last; ++oc) {
    const int slot = (cta_first_unit(U, grid, oc) >= t * KB) ? 0 : 1;
    const float* ws = sk_part_row(p, oc, slot, row, bn) + col0;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(ws + j));
      acc[j] += v.x; acc[j + 1] += v.y; acc[j + 2] += v.z; acc[j + 3] += v.w;
    }
  }
}

// ------------------------------------------------------------------ epilogue staging
// Origin of the store / residual box of the warps of 32-row quarter q (tile rows [32 q, 32 q + 32) = box_h x box_w output
// pixels), and the residual's image index.
struct StoreBox {
  int w, h, res_n;
};
__device__ __forceinline__ StoreBox store_box(const ConvGemmParams& p, const TileCoord& tc, int q) {
  const int r0 = q * 32;
  const int bh0 = r0 / p.tile_w, bw0 = r0 - bh0 * p.tile_w;
  return {tc.w0 + bw0, tc.h0 + bh0, tc.img + tc.batch * p.res_n_off};
}

// Channels [out_tail0, out_cext) of this lane's pixel that fall in a staged output chunk (128-byte swizzled row `rowp`,
// global channel gc0 at its column 0, cw columns): plain stores of what the TMA store would clip at 16-byte granularity.
template <bool HALF>
__device__ __forceinline__ void store_tail(const ConvGemmParams& p, const uint8_t* rowp, int gc0, int cw, const StoreBox& box,
                                          int out_n, int lane) {
  const int h = box.h + lane / p.box_w, w = box.w + lane % p.box_w;
  if (h >= p.out_h || w >= p.out_w) return;
  const int j0 = max(p.out_tail0 - gc0, 0), j1 = min(p.out_cext - gc0, cw);
  const uint32_t sw = static_cast<uint32_t>(lane & 7);
  const long long pix = static_cast<long long>(out_n) * p.out_str_n + static_cast<long long>(h) * p.out_str_h +
                        static_cast<long long>(w) * p.out_ld + gc0;
  for (int j = j0; j < j1; ++j) {
    if (HALF)
      static_cast<uint16_t*>(p.out_ptr)[pix + j] =     // fp16 bits
          *reinterpret_cast<const uint16_t*>(rowp + ((static_cast<uint32_t>(j >> 3) ^ sw) << 4) + (j & 7) * 2);
    else
      static_cast<float*>(p.out_ptr)[pix + j] =
          *reinterpret_cast<const float*>(rowp + ((static_cast<uint32_t>(j >> 2) ^ sw) << 4) + (j & 3) * 4);
  }
}

// Column i of the tile's scale / bias slice into shared memory (scale at sb, bias at sb + bias_off), so that the chunk loops
// read them with broadcast loads; columns past cout get scale 1 and bias 0.
__device__ __forceinline__ void stage_scale_bias(float* sb, int bias_off, const ConvGemmParams& p, const TileCoord& tc, int i) {
  const int n = tc.n0 + i;
  const int zoff = tc.batch * p.bias_z_off;
  sb[i] = (p.scale && n < p.cout) ? __ldg(p.scale + zoff + n) : 1.f;
  sb[bias_off + i] = (p.bias && n < p.cout) ? __ldg(p.bias + zoff + n) : 0.f;
}

// 4 bytes from global to shared memory without a register in between (cp.async); zero-filled unless `valid`, in which case
// nothing is read from src. Complete for the issuing thread after cp_async_wait_all.
__device__ __forceinline__ void cp_async_f32(float* dst, const float* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 4 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// ------------------------------------------------------------------ TMA producer
struct PipeState {
  int stage;
  uint32_t phase;
};

// The loads of k-blocks [kb0, kb1) of one tile pass into the STAGES-deep ring of stages stage_bytes apart from stage0, by
// lanes 0 and 1 of the producer warp, so that the two descriptor-based copies of a k-block are issued in parallel. Lane 0
// posts the stage's tx_bytes and loads the A tile (the tile's pixel rectangle shifted to filter tap (r, s)); lane 1 loads
// B rows n0 .. to b_off and, if b_lo_off != 0, their pre-split low parts (taps + p.b_lo_tap_off) to b_lo_off. bk: K slab
// width in elements. on_stage(kb) runs once the stage of k-block kb is free.
template <int STAGES, class F>
__device__ __forceinline__ void produce_pass(const CUtensorMap* tmA, const CUtensorMap* tmB, uint64_t* full_bar,
                                             uint64_t* empty_bar, PipeState& ps, uint8_t* stage0, int stage_bytes, int b_off,
                                             int b_lo_off, int bk, uint32_t tx_bytes, const ConvGemmParams& p,
                                             const TileCoord& tc, int n0, int kb0, int kb1, int lane, F&& on_stage) {
  const int k_chunks = p.k_chunks, taps_s = p.taps_s;
  int tap = kb0 / k_chunks;
  int kc = kb0 - tap * k_chunks;
  int r = tap / taps_s;
  int sx = tap - r * taps_s;
  const int a_c0 = tc.batch * p.a_c_off, a_n = tc.img + tc.batch * p.a_n_off;
  const int b_k0 = tc.batch * p.b_k_off, b_n = n0 + tc.batch * p.b_n_off;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&empty_bar[ps.stage], ps.phase ^ 1);
    on_stage(kb);
    uint8_t* dst = stage0 + ps.stage * stage_bytes;
    if (lane == 0) {
      mbar_arrive_expect_tx(&full_bar[ps.stage], tx_bytes);
      tma_load_4d(dst, tmA, &full_bar[ps.stage], kc * bk + a_c0, tc.w0 * p.stride_w + sx * p.dil - p.pad_w,
                  tc.h0 * p.stride_h + r * p.dil - p.pad, a_n);
    } else {
      tma_load_3d(dst + b_off, tmB, &full_bar[ps.stage], kc * bk + b_k0, b_n, tap);
      if (b_lo_off != 0) tma_load_3d(dst + b_lo_off, tmB, &full_bar[ps.stage], kc * bk + b_k0, b_n, tap + p.b_lo_tap_off);
    }
    if (++kc == k_chunks) {
      kc = 0;
      ++tap;
      if (++sx == taps_s) {
        sx = 0;
        ++r;
      }
    }
    if (++ps.stage == STAGES) {
      ps.stage = 0;
      ps.phase ^= 1;
    }
  }
}

// epilogue side of the accumulator ring: this thread's tile row `row`, the 32 columns of the `use`-th chunk that goes through
// ring slot `slot`; the slot is handed back once the warp has read it (all 32 lanes call this).
// A parity wait only tells the phase it names from its neighbours, so every warp that reads a slot must read EVERY chunk
// of that slot, in order: then neither side can be more than one phase away from the other.
__device__ __forceinline__ void ring_take(const uint8_t* ring, uint64_t* full, uint64_t* empty, uint32_t slot, uint32_t use,
                                          int row, uint32_t (&r)[32]) {
  mbar_wait(&full[slot], use & 1u);
  const uint8_t* rowp = ring + slot * kRingSlotBytes + row * 128;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint4 v = *reinterpret_cast<const uint4*>(rowp + ((j ^ (row & 7)) << 4));
    r[4 * j] = v.x; r[4 * j + 1] = v.y; r[4 * j + 2] = v.z; r[4 * j + 3] = v.w;
  }
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[slot]);
}
// chunk number `seq` of a ring whose slots alternate (every reader warp of a slot reads all of its chunks)
__device__ __forceinline__ void ring_take(const uint8_t* ring, uint64_t* full, uint64_t* empty, uint32_t seq, int row,
                                          uint32_t (&r)[32]) {
  ring_take(ring, full, empty, seq % kRingSlots, seq / kRingSlots, row, r);
}
__device__ __forceinline__ void ring_skip(const uint8_t* ring, uint64_t* full, uint64_t* empty, uint32_t slot, uint32_t use,
                                          int row) {
  uint32_t r[32];
  ring_take(ring, full, empty, slot, use, row, r);
}
__device__ __forceinline__ void ring_skip(const uint8_t* ring, uint64_t* full, uint64_t* empty, uint32_t seq, int row) {
  ring_skip(ring, full, empty, seq % kRingSlots, seq / kRingSlots, row);
}

// MMA side: the fragment of warpgroup-thread `wtid` (0..127) of accumulator columns [32 c, 32 c + 32) as the `use`-th chunk of
// ring slot `slot` (rows 64 wg .. 64 wg + 63); every MMA thread arrives on the slot's full barrier
template <int NR>
__device__ __forceinline__ void ring_put(uint8_t* ring, uint64_t* full, uint64_t* empty, uint32_t slot, uint32_t use, int wg,
                                         int wtid, const float (&d)[NR], const int c) {
  if (use > 0) mbar_wait(&empty[slot], (use - 1) & 1u);
  const int r0 = wg * 64 + (wtid >> 5) * 16 + ((wtid & 31) >> 2);
  const int t = wtid & 3;
  uint8_t* base = ring + slot * kRingSlotBytes;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = 2 * i + (t >> 1);                 // 16-byte group of columns 8 i + 2 t, + 1
    const int off = (t & 1) * 8;
    *reinterpret_cast<float2*>(base + r0 * 128 + ((j ^ (r0 & 7)) << 4) + off) =
        make_float2(d[4 * (4 * c + i)], d[4 * (4 * c + i) + 1]);
    const int r1 = r0 + 8;
    *reinterpret_cast<float2*>(base + r1 * 128 + ((j ^ (r1 & 7)) << 4) + off) =
        make_float2(d[4 * (4 * c + i) + 2], d[4 * (4 * c + i) + 3]);
  }
  mbar_arrive(&full[slot]);
}

// one k-block of MMAs of warpgroup wg: the 64 x BN slab of the tile, K = one 128-byte swizzle row
template <int BN, int MODE>
__device__ __forceinline__ void mma_kblock(float (&d)[BN / 2], uint32_t a_addr, uint32_t b_addr, uint32_t b_lo_addr,
                                           const int wtid, const bool first) {
  const uint64_t adesc = wgmma_desc_sw128(a_addr);
  const uint64_t bdesc = wgmma_desc_sw128(b_addr);
  if constexpr (MODE == kModeSplit3) {
    // A from registers: hi = fp32 truncated to TF32, lo = x - hi (exact); B hi / lo from shared memory
    // fragment of k-step k: rows g, g + 8 (g = 16 warp + lane / 4), K columns 8 k + lane % 4 and + 4
    const int g = (wtid >> 5) * 16 + ((wtid & 31) >> 2), t = wtid & 3;
    const uint64_t blo = wgmma_desc_sw128(b_lo_addr);
    uint32_t ahi[4][4], alo[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = g + (e & 1) * 8, col = 8 * k + t + (e >> 1) * 4;
        float x;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(a_addr + r * 128 + ((((col >> 2) ^ (r & 7)) << 4) | ((col & 3) << 2))));
        const uint32_t h = __float_as_uint(x) & 0xffffe000u;
        ahi[k][e] = h;
        alo[k][e] = __float_as_uint(x - __uint_as_float(h));
      }
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      Wgmma<BN>::tf32_rs(d, ahi[k], bdesc + 2 * k, (first && k == 0) ? 0 : 1);
      Wgmma<BN>::tf32_rs(d, ahi[k], blo + 2 * k, 1);
      Wgmma<BN>::tf32_rs(d, alo[k], bdesc + 2 * k, 1);
    }
  } else if constexpr (MODE == kModeF16x3) {
    // a staged row = [32 hi halves | 32 lo halves] of 32 K-values: k-step j (16 values) reads hi at byte 32 j and
    // lo at byte 64 + 32 j of the swizzle row (descriptor units of 16 bytes); hi.hi + hi.lo + lo.hi
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      Wgmma<BN>::f16_ss(d, adesc + 2 * k, bdesc + 2 * k, (first && k == 0) ? 0 : 1);
      Wgmma<BN>::f16_ss(d, adesc + 2 * k, bdesc + 4 + 2 * k, 1);
      Wgmma<BN>::f16_ss(d, adesc + 4 + 2 * k, bdesc + 2 * k, 1);
    }
  } else {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // advance 32 B (8 floats / 16 halves) inside the swizzle row: +2 in 16-byte units
      if (MODE == kModeF16) Wgmma<BN>::f16_ss(d, adesc + 2 * k, bdesc + 2 * k, (first && k == 0) ? 0 : 1);
      else Wgmma<BN>::tf32_ss(d, adesc + 2 * k, bdesc + 2 * k, (first && k == 0) ? 0 : 1);
    }
  }
  wgmma_commit();
}

// One k-block of a grouped convolution (mega_conv_gemm_desc::group_width = GW in {8, 16, 32}; block_n 64 and 64 channels per
// batch entry, so the staged weight tile is block-diagonal): k-step K, whose KS channels ch0 .. ch0 + KS feed only the
// output columns of their own groups, issues one wgmma of width N = max(GW, KS) over those columns -- B rows [col0, col0 + N)
// (8-row swizzle atoms: +8 col0 in descriptor units) into accumulator registers [col0 / 2, col0 / 2 + N / 2) (the m64nNk*
// fragment keeps every 8-column block in 4 consecutive registers). The products it leaves out are exact zeros, so the
// accumulator equals the dense k-block's. A k-block touches only some columns: mma_pass clears the accumulator at the start
// of a segment and every MMA accumulates. KC: which 32-channel half of the tap the k-block holds (32-value K slabs).
// Grouped launches run their own kernel instantiations (GW template argument): a runtime choice between this issue and
// the dense one inside a kernel would make ptxas serialise all of its wgmma groups.
template <int V>
struct IntC {
  static constexpr int value = V;
};
template <int K, int KN, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (K < KN) {
    f(IntC<K>());
    static_for<K + 1, KN>(f);
  }
}

template <int MODE, int GW, int KC>
__device__ __forceinline__ void mma_kblock_grouped(float (&d)[32], uint32_t a_addr, uint32_t b_addr, uint32_t b_lo_addr,
                                                   const int wtid) {
  constexpr int KS = (MODE == kModeF16 || MODE == kModeF16x3) ? 16 : 8;    // channels per k-step
  constexpr int N = GW > KS ? GW : KS;
  constexpr int NK = MODE == kModeF16x3 ? 2 : 4;                           // k-steps per k-block
  const uint64_t adesc = wgmma_desc_sw128(a_addr);
  const uint64_t bdesc = wgmma_desc_sw128(b_addr);
  if constexpr (MODE == kModeSplit3) {
    const int g = (wtid >> 5) * 16 + ((wtid & 31) >> 2), t = wtid & 3;
    const uint64_t blo = wgmma_desc_sw128(b_lo_addr);
    uint32_t ahi[4][4], alo[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = g + (e & 1) * 8, col = 8 * k + t + (e >> 1) * 4;
        float x;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(a_addr + r * 128 + ((((col >> 2) ^ (r & 7)) << 4) | ((col & 3) << 2))));
        const uint32_t h = __float_as_uint(x) & 0xffffe000u;
        ahi[k][e] = h;
        alo[k][e] = __float_as_uint(x - __uint_as_float(h));
      }
    }
    wgmma_fence();
    static_for<0, NK>([&](auto kc) {
      constexpr int k = decltype(kc)::value;
      constexpr int col0 = (32 * KC + KS * k) / N * N;
      float(&dd)[N / 2] = *reinterpret_cast<float(*)[N / 2]>(&d[col0 / 2]);
      Wgmma<N>::tf32_rs(dd, ahi[k], bdesc + 2 * k + 8 * col0, 1);
      Wgmma<N>::tf32_rs(dd, ahi[k], blo + 2 * k + 8 * col0, 1);
      Wgmma<N>::tf32_rs(dd, alo[k], bdesc + 2 * k + 8 * col0, 1);
    });
  } else {
    wgmma_fence();
    static_for<0, NK>([&](auto kc) {
      constexpr int k = decltype(kc)::value;
      constexpr int col0 = (32 * KC + KS * k) / N * N;
      float(&dd)[N / 2] = *reinterpret_cast<float(*)[N / 2]>(&d[col0 / 2]);
      if constexpr (MODE == kModeF16x3) {
        Wgmma<N>::f16_ss(dd, adesc + 2 * k, bdesc + 2 * k + 8 * col0, 1);
        Wgmma<N>::f16_ss(dd, adesc + 2 * k, bdesc + 4 + 2 * k + 8 * col0, 1);
        Wgmma<N>::f16_ss(dd, adesc + 4 + 2 * k, bdesc + 2 * k + 8 * col0, 1);
      } else if constexpr (MODE == kModeF16) {
        Wgmma<N>::f16_ss(dd, adesc + 2 * k, bdesc + 2 * k + 8 * col0, 1);
      } else {
        Wgmma<N>::tf32_ss(dd, adesc + 2 * k, bdesc + 2 * k + 8 * col0, 1);
      }
    });
  }
  wgmma_commit();
}

// kb = the k-block's index in its tile (tap * k_chunks + half): which half of the tap's 64 channels it holds
template <int MODE, int GW>
__device__ __forceinline__ void mma_kblock_grouped(float (&d)[32], uint32_t a_addr, uint32_t b_addr, uint32_t b_lo_addr,
                                                   const int wtid, const int kb) {
  if (mode_bk(MODE) == 64 || (kb & 1) == 0) mma_kblock_grouped<MODE, GW, 0>(d, a_addr, b_addr, b_lo_addr, wtid);
  else mma_kblock_grouped<MODE, GW, 1>(d, a_addr, b_addr, b_lo_addr, wtid);
}

struct MmaState {
  int stage;
  uint32_t phase;
  uint32_t uses[kRingSlots];   // accumulator chunks handed to each ring slot so far (3xFP16: uses[0] counts whole tiles)
};

// 3xFP16: the two MMA warpgroups issue their k-blocks in turn (named barriers 2 and 3 of the 256 MMA threads). Warpgroup 1
// issues k-block n after warpgroup 0 has issued it, and warpgroup 0 issues k-block n + 1 after warpgroup 1 has issued n, so
// the tensor pipe runs their MMAs one k-block apart: at every segment end one warpgroup folds into its master accumulator
// while the other's MMAs keep the pipe busy. Warpgroup 1 arrives once before its first k-block and warpgroup 0 waits once
// after its last, so that every arrival is matched.
__device__ __forceinline__ void mma_turn_wait(int wg) { asm volatile("bar.sync %0, 256;" ::"r"(3 - wg)); }
__device__ __forceinline__ void mma_turn_pass(int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(2 + wg)); }

// The MMAs of one work item (k-blocks [kb0, kb1)) for PN columns of the tile (one pass), by MMA warpgroup wg; the result
// goes to the ring in 32-column chunks. SPLIT3 / 3xFP16 restart the accumulator every seg_len k-blocks and fold the segments
// into a master accumulator with round-to-nearest adds.
// Ring slots: hpc == 0: consecutive chunks alternate over the slots (conv_gemm: every reader of a slot reads all its chunks);
// hpc > 0: the chunk of columns [32 c, 32 c + 32) goes to slot (c / hpc) & 1, the slot of the epilogue half that finishes
// those columns in a chain layer (hpc = 32-column chunks per epilogue chunk).
template <int PN, int STAGES, int MODE, class L, int GW = 0>
__device__ __forceinline__ void mma_pass(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, uint64_t* split_bar,
                                         uint8_t* ring, uint64_t* ring_full, uint64_t* ring_empty, MmaState& ms, int kb0,
                                         int kb1, int seg_len, int wg, int wtid, int hpc) {
  static_assert(GW == 0 || PN == 64, "grouped k-blocks need a 64-column pass");
  constexpr bool SPLIT3 = MODE == kModeSplit3;
  constexpr bool SEG = SPLIT3 || MODE == kModeF16x3;
  const int lane = wtid & 31;
  float d[PN / 2];
  float master[SEG ? PN / 2 : 1];
  if constexpr (MODE == kModeF16x3) {
#pragma unroll
    for (int i = 0; i < PN / 2; ++i) master[i] = -0.f;
  }
  bool has_master = false;
  for (int s0 = kb0, s1 = 0; s0 < kb1; s0 = s1) {
    s1 = (kb1 - s0 > seg_len) ? s0 + seg_len : kb1;
    int pending = -1;                            // stage whose MMAs may still be in flight
    if constexpr (GW > 0) {
#pragma unroll
      for (int i = 0; i < PN / 2; ++i) d[i] = 0.f;
    }
    for (int kb = s0; kb < s1; ++kb) {
      mbar_wait(SPLIT3 ? &split_bar[ms.stage] : &full_bar[ms.stage], ms.phase);
      const uint32_t a_addr = smem_u32(smem + ms.stage * L::kStageBytes);
      if constexpr (MODE == kModeF16x3) mma_turn_wait(wg);
      if constexpr (GW > 0)
        mma_kblock_grouped<MODE, GW>(d, a_addr + wg * 64 * 128, a_addr + L::kABytes, a_addr + L::kABytes + L::kBBytes, wtid,
                                     kb);
      else
        mma_kblock<PN, MODE>(d, a_addr + wg * 64 * 128, a_addr + L::kABytes, a_addr + L::kABytes + L::kBBytes, wtid, kb == s0);
      if constexpr (MODE == kModeF16x3) mma_turn_pass(wg);
      // SPLIT3 reads its A fragments into registers for every k-block: nothing stays in flight across them
      if (SPLIT3) wgmma_wait<0>(); else wgmma_wait<1>();
      if (pending >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[pending]);   // frees the smem slot: its MMAs have retired
      }
      pending = ms.stage;
      if (++ms.stage == STAGES) {
        ms.stage = 0;
        ms.phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_wait_regs(d);
    if (pending >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[pending]);
    }
    if constexpr (MODE == kModeF16x3) {
      // master starts at -0, and -0 + x == x for every non-NaN x (zeros and infinities included): the values the select
      // below gives. Written as that select, the fold made ptxas build each new master beside the old one (64 + 64 + 64
      // registers at PN = 128) and spill.
#pragma unroll
      for (int i = 0; i < PN / 2; ++i) master[i] = __fadd_rn(d[i], master[i]);
    } else if constexpr (SEG) {
#pragma unroll
      for (int i = 0; i < PN / 2; ++i) master[i] = has_master ? __fadd_rn(d[i], master[i]) : d[i];
      has_master = true;
    }
  }
  if constexpr (MODE == kModeF16x3) {   // chunk c of the tile -> slot c (the ring holds a whole tile)
#pragma unroll
    for (int c = 0; c < PN / 32; ++c) ring_put(ring, ring_full, ring_empty, c, ms.uses[0], wg, wtid, master, c);
    ++ms.uses[0];
  } else {
#pragma unroll
    for (int c = 0; c < PN / 32; ++c) {
      uint32_t slot;
      if (hpc == 0) slot = (ms.uses[0] == ms.uses[1]) ? 0u : 1u;    // alternate
      else slot = static_cast<uint32_t>((c / hpc) & 1);
      const uint32_t use = ms.uses[slot]++;
      if constexpr (SEG) ring_put(ring, ring_full, ring_empty, slot, use, wg, wtid, master, c);
      else ring_put(ring, ring_full, ring_empty, slot, use, wg, wtid, d, c);
    }
  }
}

// Persistent stream-K kernel. The work is the list of (tile, k-block) units, tiles ordered
// (batch, n-tile, m-tile) with m fastest; CTA c owns the contiguous unit range
// [c*U/G, (c+1)*U/G). A tile whose k-blocks straddle CTAs is finished by the last CTA to
// arrive, which sums the partial accumulators (in CTA order -> deterministic) and runs the
// epilogue. The MMA warpgroups compute item i+1 in registers while the epilogue warps finish
// item i from the accumulator ring.
// SPLIT3 ("3xTF32"): operands arrive as full fp32; four splitter warps rewrite every staged B tile as hi = fp32 truncated
// to TF32 (in place) and lo = x - hi (behind it), the MMA warpgroups split their A fragments the same way in registers, and
// each k-step issues hi*hi + hi*lo + lo*hi into the same accumulator: ~2^-19 relative error instead of 2^-11, for the
// strict-parity mode.
// OUT16: output (and residual) tensors are fp16; the epilogue then works in chunks of 64 columns (= one 128-byte
// swizzle row of halves) instead of 32.
// Programmatic dependent launch: the prologue (barrier init, descriptor prefetch) runs before griddepcontrol.wait, i.e.
// overlapped with the tail of the previous kernel on the stream; nothing before the wait touches global memory.
template <int BN, int STAGES, int MODE, bool OUT16, int GW = 0>
__global__ void __launch_bounds__(conv_gemm_threads(MODE), 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmRes,
                      const ConvGemmParams p) {
  constexpr bool SPLIT3 = MODE == kModeSplit3;
  constexpr bool PK = MODE == kModeF16x3;       // split-fp16 operands; OUT16 then means "split-fp16 output" (else fp32)
  constexpr bool SEG = SPLIT3 || PK;            // segmented accumulation with a round-to-nearest master accumulator
  constexpr bool OUTH = OUT16 && !PK;           // plain fp16 output
  constexpr int kBK = mode_bk(MODE);
  constexpr int CW = OUTH ? 64 : 32;   // epilogue chunk: columns per 128-byte output row segment
  constexpr int kMmaWarp0 = mma_warp0(MODE);
  constexpr int RS = ring_slots(MODE, BN);
  static_assert(!OUTH || BN % 64 == 0, "fp16 output needs block_n % 64 == 0");
  static_assert(SmemLayout<BN, STAGES, MODE>::kTotal <= 227 * 1024, "pipeline + staging exceed the 227 KB of a CTA");
  using L = SmemLayout<BN, STAGES, MODE>;
  // The tensor core adds into its fp32 accumulator with truncation, a bias that grows with the length of the
  // accumulation chain (~2e-5 relative after 32 k-blocks, which the chaotic position embedding of the relation module
  // amplifies to 5e-3 on the final logits). The strict modes therefore restart the accumulator every kSegLen k-blocks
  // and fold the segments into a master accumulator (registers of the MMA warpgroups) with round-to-nearest fp32 adds.
  const int kSegLen = SEG ? p.seg_len : 0x7fffffff;   // k-blocks per accumulator segment (mega_set_split3_seg_len, default 4)
  extern __shared__ uint8_t smem_raw[];
  // the 128B swizzle pattern is a function of the absolute smem address: align to 1024 B
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* split_bar = empty_bar + STAGES;       // [STAGES] (3xTF32 only)
  uint64_t* ring_full = split_bar + STAGES;       // [RS]
  uint64_t* ring_empty = ring_full + RS;          // [RS]
  uint64_t* res_bar = ring_empty + RS;            // [4 warps][2]
  int* epi_flag = reinterpret_cast<int*>(res_bar + 16);
  uint8_t* ring = smem + L::kRingOffset;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int grid = gridDim.x;
  const int cta = blockIdx.x;
  const int U = static_cast<int>(p.total_units);
  const int KB = p.kb_per_tile;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmOut);
    if (p.has_residual) prefetch_tmap(&tmRes);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);      // one arrival per MMA warp
      mbar_init(&split_bar[s], 4);
    }
    for (int b = 0; b < RS; ++b) {
      mbar_init(&ring_full[b], 256);    // every MMA thread
      mbar_init(&ring_empty[b], 4);     // the four epilogue warps that read a slot
    }
    for (int b = 0; b < 16; ++b) mbar_init(&res_bar[b], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();               // the previous kernel's results (and its reads of our outputs) are complete
  griddep_launch_dependents();  // let the next kernel's prologue overlap this kernel
  if (warp == 0) {
    // ===================== TMA producer =====================
    if (PK) setmaxnreg_dec<kF16x3RegsProducer>();
    if (lane < 2) {
      PipeState ps = {0, 0};
      WorkIter it(p, PK ? ctaid_x_here() : cta, grid);
      int t;
      int kb0, kb1;
      const bool b_lo = SPLIT3 && p.b_lo_tap_off > 0;    // pre-split weights: the low parts come by TMA too
      while (it.next(t, kb0, kb1)) {
        const TileCoord tc = decode_tile(p, t, BN, PK && p.n_fast);
        for (int pass = 0; pass < (BN > pass_n(BN) ? 2 : 1); ++pass)
          produce_pass<STAGES>(&tmA, &tmB, full_bar, empty_bar, ps, smem, L::kStageBytes, L::kABytes,
                               b_lo ? L::kABytes + L::kBBytes : 0, kBK, L::kHalf + (b_lo ? L::kBBytes : 0), p, tc,
                               tc.n0 + pass * pass_n(BN), kb0, kb1, lane, [](int) {});
      }
    }
  } else if (warp >= kMmaWarp0) {
    // ===================== MMA warpgroups =====================
    if (PK) setmaxnreg_inc<kF16x3RegsMma>();
    const int wg = (warp - kMmaWarp0) >> 2;          // tile rows [64 wg, 64 wg + 64)
    const int wtid = threadIdx.x - (kMmaWarp0 + 4 * wg) * 32;
    constexpr int P0 = pass_n(BN), P1 = BN - P0;
    MmaState ms = {0, 0, {0, 0}};
    WorkIter it(p, PK ? ctaid_x_here() : cta, grid);
    int t;
    int kb0, kb1;
    if (PK && wg == 1) mma_turn_pass(wg);
    while (it.next(t, kb0, kb1)) {
      mma_pass<P0, STAGES, MODE, L, GW>(smem, full_bar, empty_bar, split_bar, ring, ring_full, ring_empty, ms, kb0, kb1,
                                        kSegLen, wg, wtid, 0);
      if constexpr (P1 > 0)
        mma_pass<P1, STAGES, MODE, L>(smem, full_bar, empty_bar, split_bar, ring, ring_full, ring_empty, ms, kb0, kb1,
                                      kSegLen, wg, wtid, 0);
    }
    if (PK && wg == 0) mma_turn_wait(wg);
  } else if (warp >= 6 && warp < 10 && !PK) {
    // ===================== operand splitter (3xTF32 only, warps 6..9) =====================
    // B: hi = x truncated to TF32 written back in place, lo = x - hi into the region behind the raw tile (pre-split weights
    // bring lo by TMA: only the hi mask is applied). A is split by the MMA warpgroups while they load their fragments.
    if (SPLIT3) {
      const int stid = threadIdx.x - kThreads;            // 0..127
      int stage = 0;
      uint32_t phase = 0;
      WorkIter it(p, cta, grid);
      int t;
      int kb0, kb1;
      const bool need_lo = p.b_lo_tap_off == 0;
      while (it.next(t, kb0, kb1)) {
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          uint8_t* bb = smem + stage * L::kStageBytes + L::kABytes;
          constexpr int kVecs = L::kBBytes / 16;
#pragma unroll 4
          for (int v = stid; v < kVecs; v += 128) {
            float4 x = *reinterpret_cast<const float4*>(bb + v * 16);
            float4 h;
            h.x = __uint_as_float(__float_as_uint(x.x) & 0xffffe000u);
            h.y = __uint_as_float(__float_as_uint(x.y) & 0xffffe000u);
            h.z = __uint_as_float(__float_as_uint(x.z) & 0xffffe000u);
            h.w = __uint_as_float(__float_as_uint(x.w) & 0xffffe000u);
            *reinterpret_cast<float4*>(bb + v * 16) = h;
            if (need_lo)
              *reinterpret_cast<float4*>(bb + L::kBBytes + v * 16) = make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
          }
          fence_async_smem();
          __syncwarp();
          if (lane == 0) mbar_arrive(&split_bar[stage]);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else if (PK && warp >= 4 && warp < 8) {
    // ===================== epilogue, 3xFP16 (warps 4..7) =====================
    // One warp per 32-row quarter of the tile finishes all of its 32-column chunks: every ring slot is read by all four
    // warps. The BN scale is folded into the packed weights, and the bias slice of the NEXT tile is fetched during the
    // current one (double-buffered, one barrier per tile). The ring holds the whole tile (chunk j in slot j): each warp
    // writes its result back into the rows of the slot it read (every thread reads its 128-byte row into registers before
    // it writes the same row), stores it from there, and hands the tile's slots back once those stores have read them. The
    // residual arrives in two 4 KB buffers per warp: chunks 0 and 1 at the start of the tile, chunk j + 2 once j is read.
    setmaxnreg_dec<kF16x3RegsEpilogue>();
    constexpr int kCPW = BN / 32;          // 32-column chunks per warp
    const int q = warp & 3;                // 32-row quarter of the tile
    const int row = q * 32 + lane;
    const int epi_tid = (warp - 4) * 32 + lane;                              // 0 .. 127
    uint8_t* res_buf = smem + L::kEpiOffset + (warp - 4) * 8192;             // 2 x 4 KB residual staging
    uint64_t* rbar = res_bar + (warp - 4) * 2;
    float* bias_s = reinterpret_cast<float*>(smem + L::kSbOffset);           // [2][BN]
    uint32_t rphase = 0;
    const int cta_e = ctaid_x_here();
    WorkIter it(p, cta_e, grid);
    int t;
    int kb0, kb1;
    const uint32_t sw = static_cast<uint32_t>(lane & 7);
    const bool res_split = p.res_split != 0;
    const float slope = p.relu == 2 ? 0.1f : 0.f;
    for (int tile_item = 0; it.next(t, kb0, kb1); ++tile_item) {
      const TileCoord tc = decode_tile(p, t, BN, p.n_fast);
      const bool complete = (kb0 == 0 && kb1 == KB);
      const StoreBox box = store_box(p, tc, q);
      const int nchunks = min(BN / 32, (p.cout - tc.n0 + 31) / 32);
      const int bsel = tile_item & 1;
      // ---- bias slices: [bsel] holds this tile's (written at the end of the previous tile, or right here for the first)
      epi_bar_sync<128>();     // every warp is done with the tile before: its bias buffer may be refilled, this one's is visible
      if (tile_item == 0) {
        if (epi_tid < BN) {
          const int n = tc.n0 + epi_tid;
          bias_s[epi_tid] = (p.bias && n < p.cout) ? __ldg(p.bias + tc.batch * p.bias_z_off + n) : 0.f;
        }
        epi_bar_sync<128>();
      }
      {   // the next tile's slice into [bsel ^ 1], which no warp reads before the next tile's barrier
        int t2;
        if (it.peek(t2) && epi_tid < BN) {
          const TileCoord tc2 = decode_tile(p, t2, BN, p.n_fast);
          const int n = tc2.n0 + epi_tid;
          const bool valid = p.bias && n < p.cout;
          cp_async_f32(bias_s + (bsel ^ 1) * BN + epi_tid,
                       valid ? p.bias + tc2.batch * p.bias_z_off + n : static_cast<const float*>(p.out_ptr), valid);
        }
      }
      // ---- residual chunk j into buffer j & 1 (read by the time chunk j + 2 is issued: the reads precede a fence and a
      //      __syncwarp)
      const int res_c0 = tc.n0 + tc.batch * p.res_c_off;
      auto issue_residual = [&](const int j) {
        if (p.has_residual && lane == 0 && j < nchunks) {
          mbar_arrive_expect_tx(&rbar[j & 1], 4096);
          tma_load_4d(res_buf + (j & 1) * 4096, &tmRes, &rbar[j & 1], res_c0 + j * 32, box.w, box.h, box.res_n);
        }
      };
      if (complete) {
        issue_residual(0);
        issue_residual(1);
      }
      // Every warp waits for every chunk of every tile, columns past cout included: a parity wait only tells the phase it
      // names from its neighbours, so neither side may run more than one phase ahead of the other.
      auto take_chunk = [&](const int j, uint32_t (&r)[32]) {
        mbar_wait(&ring_full[j], bsel);
        const uint8_t* rowp = ring + j * kRingSlotBytes + row * 128;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const uint4 v = *reinterpret_cast<const uint4*>(rowp + ((static_cast<uint32_t>(i) ^ sw) << 4));
          r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
        }
      };
      bool finalize = complete;
      int c_first = cta_e, c_last = cta_e;
      if (!complete) {
        // ---- publish this CTA's partial accumulator (this warp's rows), then find out whether it arrived last
        float* part = sk_own_part_row(p, cta_e, tile_item, row, BN);
#pragma unroll
        for (int j = 0; j < kCPW; ++j) {
          uint32_t raw[32];
          take_chunk(j, raw);
          sk_publish(part, j * 32, raw);
        }
        finalize = sk_elect_finisher<128>(p, U, grid, KB, t, epi_tid, epi_flag, c_first, c_last);
        if (finalize) {
          issue_residual(0);
          issue_residual(1);
        }
      }
      if (finalize) {
        const int out_n = tc.img + tc.batch * p.out_n_off;
#pragma unroll
        for (int j = 0; j < kCPW; ++j) {
          if (j < nchunks) {
            float acc[32];
            if (complete) {
              uint32_t raw[32];
              take_chunk(j, raw);
#pragma unroll
              for (int i = 0; i < 32; ++i) acc[i] = __uint_as_float(raw[i]);
            } else {
              sk_reduce(p, U, grid, KB, t, c_first, c_last, row, BN, j * 32, acc);
            }
            uint8_t* rowp = ring + j * kRingSlotBytes + row * 128;        // the result goes back to the row it came from
            const uint8_t* resp = res_buf + (j & 1) * 4096 + lane * 128;
            const float4* biv = reinterpret_cast<const float4*>(bias_s + bsel * BN + j * 32);
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              const float4 bi = biv[i >> 2];
              acc[i] = fmaf(acc[i], p.acc_scale, bi.x); acc[i + 1] = fmaf(acc[i + 1], p.acc_scale, bi.y);
              acc[i + 2] = fmaf(acc[i + 2], p.acc_scale, bi.z); acc[i + 3] = fmaf(acc[i + 3], p.acc_scale, bi.w);
            }
            if (p.has_residual) {
              mbar_wait(&rbar[j & 1], (rphase >> (j & 1)) & 1u);
              rphase ^= (1u << (j & 1));
              if (res_split) {    // 16-byte chunks 0..3: hi halves of values 8c .. 8c+7, chunks 4..7: their lo halves
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                  const uint4 rh = *reinterpret_cast<const uint4*>(resp + ((static_cast<uint32_t>(c) ^ sw) << 4));
                  const uint4 rl = *reinterpret_cast<const uint4*>(resp + ((static_cast<uint32_t>(4 + c) ^ sw) << 4));
                  const uint32_t hs[4] = {rh.x, rh.y, rh.z, rh.w}, ls[4] = {rl.x, rl.y, rl.z, rl.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 a2 = h2_to_f2(hs[e]), b2 = h2_to_f2(ls[e]);
                    acc[8 * c + 2 * e] += a2.x + b2.x;
                    acc[8 * c + 2 * e + 1] += a2.y + b2.y;
                  }
                }
              } else {
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                  const float4 rr = *reinterpret_cast<const float4*>(resp + ((static_cast<uint32_t>(c) ^ sw) << 4));
                  acc[4 * c] += rr.x; acc[4 * c + 1] += rr.y; acc[4 * c + 2] += rr.z; acc[4 * c + 3] += rr.w;
                }
              }
            }
            if (p.relu) {
#pragma unroll
              for (int i = 0; i < 32; ++i) acc[i] = fmaxf(acc[i], slope * acc[i]);
            }
            if (OUT16) {      // split-fp16 result
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                uint32_t hh[4], ll[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  hh[e] = f2_to_h2_sat(acc[8 * c + 2 * e], acc[8 * c + 2 * e + 1]);
                  const float2 back = h2_to_f2(hh[e]);
                  ll[e] = f2_to_h2_sat(acc[8 * c + 2 * e] - back.x, acc[8 * c + 2 * e + 1] - back.y);
                }
                *reinterpret_cast<uint4*>(rowp + ((static_cast<uint32_t>(c) ^ sw) << 4)) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
                *reinterpret_cast<uint4*>(rowp + ((static_cast<uint32_t>(4 + c) ^ sw) << 4)) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
              }
            } else {
#pragma unroll
              for (int c = 0; c < 8; ++c)
                *reinterpret_cast<float4*>(rowp + ((static_cast<uint32_t>(c) ^ sw) << 4)) =
                    make_float4(acc[4 * c], acc[4 * c + 1], acc[4 * c + 2], acc[4 * c + 3]);
            }
            fence_async_smem();
            __syncwarp();
            if (j + 2 < kCPW) issue_residual(j + 2);
            const int gc0 = tc.n0 + j * 32 + tc.batch * p.out_c_off;
            if (!OUT16 && gc0 + 32 > p.out_tail0) store_tail<false>(p, rowp, gc0, 32, box, out_n, lane);
            if (lane == 0 && gc0 < p.out_tail0) {
              tma_store_4d(&tmOut, ring + j * kRingSlotBytes + q * 4096, gc0, box.w, box.h, out_n);
              tma_store_commit();
            }
          } else if (complete) {
            mbar_wait(&ring_full[j], bsel);   // columns past cout: nothing to read
          }
        }
      }
      // ---- the tile's slots go back to the MMA warpgroups once this warp's stores have read its rows
      if (lane == 0) tma_store_wait_read<0>();
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < kCPW; ++j) mbar_arrive(&ring_empty[j]);
      }
      cp_async_wait_all();
    }
    if (lane == 0) tma_store_wait<0>();   // global writes complete before the CTA retires
  } else if (PK) {
    // warps 1..3 (barrier init done): their registers go to the MMA warpgroups
    setmaxnreg_dec<kF16x3RegsProducer>();
  } else if (warp >= 2 && warp < 6) {
    // ===================== epilogue (warps 2..5) =====================
    const int q = warp & 3;  // 32-row quarter of the tile
    const int row = q * 32 + lane;
    const int epi_tid = (warp - 2) * 32 + lane;
    uint8_t* epi_out = smem + L::kEpiOffset + (warp - 2) * 16384;   // 2 x 4 KB store staging
    uint8_t* epi_res = epi_out + 8192;                              // 2 x 4 KB residual staging
    uint64_t* rbar = res_bar + (warp - 2) * 2;
    float* sb_s = reinterpret_cast<float*>(smem + L::kSbOffset);
    uint32_t rphase = 0;
    WorkIter it(p, cta, grid);
    int t;
    int kb0, kb1;
    uint32_t seq0 = 0;    // ring chunk number of this item's column 0
    for (int tile_item = 0; it.next(t, kb0, kb1); ++tile_item, seq0 += BN / 32) {
      const TileCoord tc = decode_tile(p, t, BN);
      const bool complete = (kb0 == 0 && kb1 == KB);
      // ---- while the MMAs of this tile run: stage its scale / bias slice in shared memory (the chunk loop then reads
      //      them with broadcast LDS instead of L1-missing global loads) and start the first residual load
      const StoreBox box = store_box(p, tc, q);
      const int nchunks = min(BN / CW, (p.cout - tc.n0 + CW - 1) / CW);
      epi_bar_sync<128>();   // every warp is done with the previous tile's scale / bias
      for (int i = epi_tid; i < BN; i += 128) stage_scale_bias(sb_s, L::kSbCols, p, tc, i);
      if (complete && p.has_residual && lane == 0 && nchunks > 0) {
        mbar_arrive_expect_tx(&rbar[0], 4096);
        tma_load_4d(epi_res, &tmRes, &rbar[0], tc.n0 + tc.batch * p.res_c_off, box.w, box.h, box.res_n);
      }
      epi_bar_sync<128>();
      bool finalize = complete;
      int c_first = cta, c_last = cta;
      if (!complete) {
        // ---- publish this CTA's partial accumulator, then find out whether it arrived last
        float* part = sk_own_part_row(p, cta, tile_item, row, BN);
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
          uint32_t raw[32];
          ring_take(ring, ring_full, ring_empty, seq0 + c, row, raw);
          sk_publish(part, c * 32, raw);
        }
        finalize = sk_elect_finisher<128>(p, U, grid, KB, t, epi_tid, epi_flag, c_first, c_last);
      }
      if (finalize) {
        // Output pixels of this warp: tile rows [32q, 32q+32) = a box_h x box_w rectangle. Results go
        // registers -> 128B-swizzled smem -> one TMA store per 32-column chunk (full-line writes,
        // image-edge and channel-edge clipping by the TMA unit); the residual arrives the same way.
        const int out_n = tc.img + tc.batch * p.out_n_off;
        const bool has_sb = (p.scale != nullptr) || (p.bias != nullptr);
        const uint32_t sw = static_cast<uint32_t>(lane & 7);
        if (!complete && p.has_residual && lane == 0 && nchunks > 0) {   // (whole tiles started this load earlier)
          mbar_arrive_expect_tx(&rbar[0], 4096);
          tma_load_4d(epi_res, &tmRes, &rbar[0], tc.n0 + tc.batch * p.res_c_off, box.w, box.h, box.res_n);
        }
        auto finish_chunk = [&](const int c) {
          const int nb = tc.n0 + c * CW;
          const uint8_t* rsrc = nullptr;
          if (p.has_residual) {
            const int rb = c & 1;
            if (c + 1 < nchunks && lane == 0) {   // prefetch the next residual chunk into the other buffer
              mbar_arrive_expect_tx(&rbar[rb ^ 1], 4096);
              tma_load_4d(epi_res + (rb ^ 1) * 4096, &tmRes, &rbar[rb ^ 1], nb + CW + tc.batch * p.res_c_off, box.w, box.h,
                          box.res_n);
            }
            mbar_wait(&rbar[rb], (rphase >> rb) & 1u);
            rphase ^= (1u << rb);
            rsrc = epi_res + rb * 4096 + lane * 128;
          }
          // the out staging buffer (c & 1) was handed to a TMA store two chunks ago: wait until read
          if (lane == 0) tma_store_wait_read<1>();
          __syncwarp();
          uint8_t* dst = epi_out + (c & 1) * 4096 + lane * 128;
          // 32 accumulator columns at a time (keeps the live registers at 32 + a handful: the 64-wide form spilled)
        #pragma unroll
          for (int h = 0; h < CW / 32; ++h) {
            const int col0 = c * CW + h * 32;     // first column of this half inside the tile
            float acc[32];
            if (complete) {
              uint32_t raw[32];
              ring_take(ring, ring_full, ring_empty, seq0 + col0 / 32, row, raw);
        #pragma unroll
              for (int j = 0; j < 32; ++j) acc[j] = __uint_as_float(raw[j]);
            } else {
              sk_reduce(p, U, grid, KB, t, c_first, c_last, row, BN, col0, acc);
            }
            if (has_sb) {
              const float4* scv = reinterpret_cast<const float4*>(sb_s + col0);
              const float4* biv = reinterpret_cast<const float4*>(sb_s + L::kSbCols + col0);
        #pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float4 sc = scv[j >> 2], bi = biv[j >> 2];
                acc[j] = fmaf(acc[j], sc.x, bi.x); acc[j + 1] = fmaf(acc[j + 1], sc.y, bi.y);
                acc[j + 2] = fmaf(acc[j + 2], sc.z, bi.z); acc[j + 3] = fmaf(acc[j + 3], sc.w, bi.w);
              }
            }
            const float slope = p.relu == 2 ? 0.1f : 0.f;
            if (OUTH) {
              // 64 halves per staging row: 16-byte groups of 8 halves, swizzled like the TMA box
        #pragma unroll
              for (int j = 0; j < 32; j += 8) {
                const uint32_t chunk = (static_cast<uint32_t>((h * 32 + j) >> 3) ^ sw) << 4;
                float v[8];
        #pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = acc[j + e];
                if (rsrc) {
                  const uint4 rr = *reinterpret_cast<const uint4*>(rsrc + chunk);
                  const float2 r0v = h2_to_f2(rr.x), r1v = h2_to_f2(rr.y), r2v = h2_to_f2(rr.z), r3v = h2_to_f2(rr.w);
                  v[0] += r0v.x; v[1] += r0v.y; v[2] += r1v.x; v[3] += r1v.y;
                  v[4] += r2v.x; v[5] += r2v.y; v[6] += r3v.x; v[7] += r3v.y;
                }
                if (p.relu) {
        #pragma unroll
                  for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], slope * v[e]);
                }
                uint4 o;
                o.x = f2_to_h2(v[0], v[1]); o.y = f2_to_h2(v[2], v[3]);
                o.z = f2_to_h2(v[4], v[5]); o.w = f2_to_h2(v[6], v[7]);
                *reinterpret_cast<uint4*>(dst + chunk) = o;
              }
            } else {
        #pragma unroll
              for (int j = 0; j < 32; j += 4) {
                float4 v = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
                const uint32_t chunk = (static_cast<uint32_t>(j >> 2) ^ sw) << 4;
                if (rsrc) {
                  const float4 rr = *reinterpret_cast<const float4*>(rsrc + chunk);
                  v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
                }
                if (p.relu) {
                  v.x = fmaxf(v.x, slope * v.x); v.y = fmaxf(v.y, slope * v.y);
                  v.z = fmaxf(v.z, slope * v.z); v.w = fmaxf(v.w, slope * v.w);
                }
                *reinterpret_cast<float4*>(dst + chunk) = v;
              }
            }
          }
          fence_async_smem();
          __syncwarp();
          const int gc0 = nb + tc.batch * p.out_c_off;
          if (gc0 + CW > p.out_tail0) store_tail<OUTH>(p, dst, gc0, CW, box, out_n, lane);
          if (lane == 0 && gc0 < p.out_tail0) {
            tma_store_4d(&tmOut, epi_out + (c & 1) * 4096, gc0, box.w, box.h, out_n);
            tma_store_commit();
          }
        };
#pragma unroll 1
        for (int c = 0; c < nchunks; ++c) finish_chunk(c);
      }
      if (complete) {
        // columns past cout: hand their ring slots back unread
#pragma unroll 1
        for (int c = nchunks * (CW / 32); c < BN / 32; ++c) ring_skip(ring, ring_full, ring_empty, seq0 + c, row);
      }
    }
    if (lane == 0) tma_store_wait<0>();   // global writes complete before the CTA retires
  }
}

// ------------------------------------------------------------------ launch
// pdl != 0: launched with programmatic stream serialization, i.e. this kernel's prologue may start while the
// previous kernel on the stream drains (the kernel itself orders its memory accesses with griddepcontrol.wait).
template <int BN, int STAGES, int MODE, bool OUT16, int GW = 0>
static int launch_cfg(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                      const CUtensorMap& tmRes, const ConvGemmParams& p, dim3 grid, cudaStream_t stream, int pdl) {
  using L = SmemLayout<BN, STAGES, MODE>;
  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(conv_gemm_kernel<BN, STAGES, MODE, OUT16, GW>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(conv_gemm_threads(MODE), 1, 1);
  cfg.dynamicSmemBytes = L::kTotal;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  MEGA_CUDA_CHECK(cudaLaunchKernelEx(&cfg, conv_gemm_kernel<BN, STAGES, MODE, OUT16, GW>, tmA, tmB, tmOut, tmRes, p));
  return MEGA_OK;
}

// The kernel instantiation of one launch of operand mode MODE: block_n, out16 (fp16 output for kModeF16, which needs
// block_n % 64 == 0; split-fp16 output for kModeF16x3) and the group width gw (0: dense; 8 / 16 / 32: block_n 64).
// Each mode is instantiated in one translation unit (conv_gemm.cu: tf32 and 3xTF32, conv_gemm_f16.cu, conv_gemm_f16x3.cu),
// so that nvcc builds them in parallel.
template <int MODE>
int launch_mode(int block_n, bool out16, int gw, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                const CUtensorMap& tmRes, const ConvGemmParams& p, dim3 grid, cudaStream_t stream, int pdl) {
  auto launch = [&](auto bn, auto gw_c) -> int {
    constexpr int BN = decltype(bn)::value, GW = decltype(gw_c)::value, ST = conv_gemm_stages(MODE, BN);
    if constexpr (MODE == kModeF16x3 || (MODE == kModeF16 && BN % 64 == 0)) {
      if (out16) return launch_cfg<BN, ST, MODE, true, GW>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
    } else if (out16) {
      mega_set_error("conv_gemm: fp16 output needs fp16 operands and block_n %% 64 == 0 (got precision %d, block_n %d)",
                     MODE, BN);
      return MEGA_ERR_ARG;
    }
    return launch_cfg<BN, ST, MODE, false, GW>(tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
  };
  switch (gw) {
    case 8: return launch(IntC<64>(), IntC<8>());
    case 16: return launch(IntC<64>(), IntC<16>());
    case 32: return launch(IntC<64>(), IntC<32>());
  }
  switch (block_n) {
    case 64: return launch(IntC<64>(), IntC<0>());
    case 128: return launch(IntC<128>(), IntC<0>());
  }
  if constexpr (MODE == kModeTf32 || MODE == kModeF16) {   // the strict modes run block_n 64 and 128 only
    switch (block_n) {
      case 32: return launch(IntC<32>(), IntC<0>());
      case 96: return launch(IntC<96>(), IntC<0>());
      case 160: return launch(IntC<160>(), IntC<0>());
      case 192: return launch(IntC<192>(), IntC<0>());
      case 256: return launch(IntC<256>(), IntC<0>());
    }
  }
  mega_set_error("conv_gemm: unsupported block_n %d for precision %d", block_n, MODE);
  return MEGA_ERR_ARG;
}

// declarator of launch_mode<M> for its explicit instantiations
#define MEGA_LAUNCH_MODE(M)                                                                                                \
  int launch_mode<M>(int, bool, int, const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,     \
                     const ConvGemmParams&, dim3, cudaStream_t, int)
extern template MEGA_LAUNCH_MODE(kModeTf32);
extern template MEGA_LAUNCH_MODE(kModeSplit3);
extern template MEGA_LAUNCH_MODE(kModeF16);
extern template MEGA_LAUNCH_MODE(kModeF16x3);

}  // namespace mega
