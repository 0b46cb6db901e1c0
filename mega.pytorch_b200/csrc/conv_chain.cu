// A whole chain of dependent convolutions / GEMMs in ONE persistent kernel.
//
// The backbone of the MEGA hot path is a strictly sequential chain of ~100 small implicit GEMMs per frame pair
// (ResNet-101 res2..res5, modeling/backbone/resnet.py:324-344; RPN head, rpn/rpn.py:99-106). Each of them is 2-10 us
// of tensor-core work at M = 4788 output pixels, so one-kernel-per-layer execution is dominated by what surrounds
// the math: launch, barrier set-up, descriptor fetch, pipeline fill and drain.
//
// Here the per-layer kernel body (TMA producer warp / two wgmma warpgroups / 8 epilogue warps fed through the
// accumulator ring, persistent stream-K work list -- see conv_gemm_kernel.cuh) is wrapped in a loop over a device-side
// table of layers. One CTA per SM stays resident for the whole chain; mbarriers and the smem rings are set up once;
// layers are separated by a grid-wide barrier (one atomic counter, release/acquire) instead of a kernel boundary.
// Tensor maps live in the layer table in global memory.
//
// Barrier depth. With depth 1 layer l starts when every CTA has finished layer l-1: the tensor pipe idles through every
// layer's tail (last epilogue, store drain + gpu-scope release, barrier, first operand fetch). With depth 2 layer l only waits for layer l-2 (one arrival counter per layer parity), so a table that INTERLEAVES two
// independent chains A0 B0 A1 B1 ... (the per-frame branch of two halves of an image batch) keeps the TMA / MMA warps of
// every CTA streaming chain B's layer while chain A's tail drains, and vice versa. Stream-K partial sums and tile
// counters of odd layers live in the second half of the workspace (a CTA may already publish partials of layer l+1
// while a slower CTA still reduces layer l).
//
// Restrictions of a chain: fp16 operands, block_n <= 128 (one 32 KB smem stage holds A 128 x 64 and B
// block_n x 64 halves), output fp16 or fp32 per layer.
#include "conv_gemm_kernel.cuh"

namespace mega {

constexpr int kChainStages = 4;
constexpr int kChainStageBytes = 32768;     // A tile 16 KB + B tile (<= 128 rows) 16 KB
constexpr int kChainABytes = 16384;
constexpr int kChainRingOffset = kChainStages * kChainStageBytes;
constexpr int kChainEpiOffset = kChainRingOffset + kRingSlots * kRingSlotBytes;
constexpr int kChainEpiBytes = 4 * 4 * 4096;
constexpr int kChainBarOffset = kChainEpiOffset + kChainEpiBytes;
constexpr int kChainSbOffset = kChainBarOffset + 256;      // [scale | bias][128] floats of the tile being finished
constexpr int kChainSmem = kChainSbOffset + 1024 + 1024;
static_assert(kChainSmem <= 227 * 1024, "chain pipeline + staging exceed the 227 KB of a CTA");
struct ChainSmemLayout {     // what mma_pass needs to know of a stage
  static constexpr int kStageBytes = kChainStageBytes;
  static constexpr int kABytes = kChainABytes;
  static constexpr int kBBytes = kChainStageBytes - kChainABytes;
};

struct alignas(128) ChainLayer {
  CUtensorMap tmA, tmB, tmOut, tmRes;
  ConvGemmParams p;
  int block_n;
  int out16;
  int active_ctas;   // CTAs that take part in this layer's work list (<= grid); the others only pass the barrier
  int cta_rot;       // physical CTA (cta_rot + i) % grid plays logical CTA i of this layer's work list (depth-2 chains:
                     // the work lists of consecutive layers start where the previous one ended, so a layer whose tile
                     // count is not a multiple of the grid does not leave the same SMs idle every time)
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// generic <-> async proxy ordering (TMA loads of data other CTAs wrote with TMA stores / generic stores)
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// all CTAs of the grid have finished `target / grid` layers
__device__ __forceinline__ void grid_wait(const unsigned* ctr, unsigned target) {
  if (ld_acquire_u32(ctr) >= target) {
    fence_proxy_async_all();
    return;
  }
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (ld_acquire_u32(ctr) < target) {
    __nanosleep(40);
    if ((++spins & 0x3ff) == 0 && globaltimer_ns() - t0 > 2000000000ull) __trap();   // (no printf: see mbar_wait)
  }
  fence_proxy_async_all();
}

// optional in-kernel event trace of ONE CTA (diagnostics): (tag, SM clock) pairs per role
struct ChainTrace {
  unsigned long long* buf;   // [3 roles][kTraceCap][2] or NULL
  int cta;
  int level;                 // 0: every event; 1: per-layer events only (a 100-layer chain fits the buffer);
                             // 2 + l: every event of layer l only
};
constexpr int kTraceCap = 4096;
struct TraceCursor {
  unsigned long long* p;
  int n;
  int level;
  __device__ __forceinline__ void put(unsigned long long tag) {
    if (p != nullptr && n < kTraceCap) {
      const unsigned code = static_cast<unsigned>(tag & 0xff);
      if (level == 1 && code >= 3 && code <= 7) return;      // per-k-block / per-tile events
      if (level >= 2 && static_cast<int>(tag >> 32) != level - 2) return;
      p[2 * n] = tag;
      p[2 * n + 1] = static_cast<unsigned long long>(clock64());
      ++n;
    }
  }
};
__device__ __forceinline__ TraceCursor trace_cursor(const ChainTrace& tr, int role, int cta) {
  TraceCursor c;
  c.p = (tr.buf != nullptr && cta == tr.cta) ? tr.buf + static_cast<long long>(role) * kTraceCap * 2 : nullptr;
  c.n = 0;
  c.level = tr.level;
  return c;
}
#define TR_TAG(layer, idx, code) ((static_cast<unsigned long long>(layer) << 32) | (static_cast<unsigned long long>(idx) << 8) | (code))

// ------------------------------------------------------------------ epilogue of one layer (8 warps)
// Eight epilogue warps: warp w finishes tile rows 32 (w & 3) .. +31, and of the tile's 64-column (fp16 out) / 32-column
// (fp32 out) chunks it takes those with chunk % 2 == (w - 2) / 4, so every accumulator ring slot is read by the four warps
// of one parity. The layer's flags are template parameters of the inner loop, staging goes through explicit ld/st.shared
// with precomputed swizzled offsets, and two warps share a row quarter.
constexpr int kEpiWarps = 8;
constexpr int kEpiThreads = kEpiWarps * 32;
// warps 0..7: the two MMA warpgroups; 8..15: epilogue; 16: TMA producer. 544 threads leave 120 registers per thread, which
// the MMA warpgroups need to keep a 64 x 128 accumulator live across their asynchronous wgmma groups
constexpr int kChainMmaWarp0 = 0;
constexpr int kChainEpiWarp0 = 8;
constexpr int kChainProducerWarp = 16;
constexpr int kChainThreads = (kChainProducerWarp + 1) * 32;

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// 32 accumulator columns (one thread = one output pixel) -> scale / bias -> (+ residual) -> activation -> staging row.
// sb: shared address of scale[col0 ..] (bias at +512 bytes); dst / rsrc: shared addresses of this lane's 128-byte staging
// rows; off[g]: byte offset of 16-byte group g inside the swizzled row. H: which 32-column half of a 64-half row (OUT16).
template <bool OUT16, bool RES, int RELU>
__device__ __forceinline__ void epi_half(const uint32_t (&raw)[32], uint32_t sb, uint32_t dst, uint32_t rsrc,
                                         const uint32_t (&off)[8], const int H) {
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const uint4 sc = lds128(sb + j * 4), bi = lds128(sb + 512 + j * 4);
    v[j] = fmaf(__uint_as_float(raw[j]), __uint_as_float(sc.x), __uint_as_float(bi.x));
    v[j + 1] = fmaf(__uint_as_float(raw[j + 1]), __uint_as_float(sc.y), __uint_as_float(bi.y));
    v[j + 2] = fmaf(__uint_as_float(raw[j + 2]), __uint_as_float(sc.z), __uint_as_float(bi.z));
    v[j + 3] = fmaf(__uint_as_float(raw[j + 3]), __uint_as_float(sc.w), __uint_as_float(bi.w));
  }
  if (OUT16) {
#pragma unroll
    for (int g = 0; g < 4; ++g) {          // 8 halves = 16 bytes per group
      const int j = g * 8;
      if (RES) {
        const uint4 rr = lds128(rsrc + off[H * 4 + g]);
        const float2 r0 = h2_to_f2(rr.x), r1 = h2_to_f2(rr.y), r2 = h2_to_f2(rr.z), r3 = h2_to_f2(rr.w);
        v[j] += r0.x; v[j + 1] += r0.y; v[j + 2] += r1.x; v[j + 3] += r1.y;
        v[j + 4] += r2.x; v[j + 5] += r2.y; v[j + 6] += r3.x; v[j + 7] += r3.y;
      }
      if (RELU == 1) {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[j + e] = fmaxf(v[j + e], 0.f);
      } else if (RELU == 2) {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[j + e] = fmaxf(v[j + e], 0.1f * v[j + e]);
      }
      uint4 o;
      o.x = f2_to_h2(v[j], v[j + 1]); o.y = f2_to_h2(v[j + 2], v[j + 3]);
      o.z = f2_to_h2(v[j + 4], v[j + 5]); o.w = f2_to_h2(v[j + 6], v[j + 7]);
      sts128(dst + off[H * 4 + g], o);
    }
  } else {
#pragma unroll
    for (int g = 0; g < 8; ++g) {          // 4 floats = 16 bytes per group
      const int j = g * 4;
      if (RES) {
        const uint4 rr = lds128(rsrc + off[g]);
        v[j] += __uint_as_float(rr.x); v[j + 1] += __uint_as_float(rr.y);
        v[j + 2] += __uint_as_float(rr.z); v[j + 3] += __uint_as_float(rr.w);
      }
      if (RELU == 1) {
#pragma unroll
        for (int e = 0; e < 4; ++e) v[j + e] = fmaxf(v[j + e], 0.f);
      } else if (RELU == 2) {
#pragma unroll
        for (int e = 0; e < 4; ++e) v[j + e] = fmaxf(v[j + e], 0.1f * v[j + e]);
      }
      uint4 o;
      o.x = __float_as_uint(v[j]); o.y = __float_as_uint(v[j + 1]); o.z = __float_as_uint(v[j + 2]); o.w = __float_as_uint(v[j + 3]);
      sts128(dst + off[g], o);
    }
  }
}

template <bool OUT16>
__device__ __forceinline__ void epi_half_dispatch(const uint32_t (&raw)[32], uint32_t sb, uint32_t dst, uint32_t rsrc,
                                                  const uint32_t (&off)[8], const int H, const bool res, const int relu) {
  // the flags are uniform over the layer: one branch per 32 columns instead of one per element
  if (relu == 1) {
    if (res) epi_half<OUT16, true, 1>(raw, sb, dst, rsrc, off, H);
    else epi_half<OUT16, false, 1>(raw, sb, dst, rsrc, off, H);
  } else if (relu == 0) {
    if (res) epi_half<OUT16, true, 0>(raw, sb, dst, rsrc, off, H);
    else epi_half<OUT16, false, 0>(raw, sb, dst, rsrc, off, H);
  } else {
    if (res) epi_half<OUT16, true, 2>(raw, sb, dst, rsrc, off, H);
    else epi_half<OUT16, false, 2>(raw, sb, dst, rsrc, off, H);
  }
}

template <bool OUT16>
__device__ __forceinline__ void chain_epilogue_layer(const ChainLayer* L, const ConvGemmParams& p, const int BN, uint8_t* smem,
                                                  uint64_t* ring_full, uint64_t* ring_empty, uint64_t* res_bar,
                                                  int* epi_flag, int warp, int lane, int cta,
                                                  int grid, uint32_t& ruse, uint32_t& rphase, TraceCursor& tr, int layer) {
  constexpr int CW = OUT16 ? 64 : 32;          // columns per chunk (= one 128-byte staging row)
  constexpr int HPC = CW / 32;                 // 32-column halves per chunk
  const int ew = warp - kChainEpiWarp0;        // epilogue warp 0..7
  const int q = warp & 3;                      // 32-row quarter of the tile
  const int half = ew >> 2;                    // parity of the chunks this warp takes
  const int row = q * 32 + lane;
  const int epi_tid = ew * 32 + lane;
  const uint32_t stage_base = smem_u32(smem + kChainEpiOffset + ew * 8192);
  const uint8_t* ring = smem + kChainRingOffset;
  const uint32_t out_row = stage_base + lane * 128;          // 4 KB store staging | 4 KB residual staging per warp
  const uint32_t res_row = out_row + 4096;
  uint64_t* rbar = res_bar + ew;
  const uint32_t sb_u32 = smem_u32(smem + kChainSbOffset);
  float* sb_s = reinterpret_cast<float*>(smem + kChainSbOffset);
  const int U = static_cast<int>(p.total_units);
  const int KB = p.kb_per_tile;
  const CUtensorMap* tmOut = &L->tmOut;
  const CUtensorMap* tmRes = &L->tmRes;
  const bool has_res = p.has_residual != 0;
  const int relu = p.relu;
  uint32_t off[8];
#pragma unroll
  for (int g = 0; g < 8; ++g) off[g] = (static_cast<uint32_t>(g) ^ static_cast<uint32_t>(lane & 7)) << 4;
  WorkIter it(p, cta, grid);
  int t;
  int kb0, kb1;
  // every 32-column accumulator chunk of this warp's epilogue chunks arrives in ring slot `half`; ruse counts them
  for (int tile_item = 0; it.next(t, kb0, kb1); ++tile_item) {
    const TileCoord tc = decode_tile(p, t, BN);
    const bool complete = (kb0 == 0 && kb1 == KB);
    const StoreBox box = store_box(p, tc, q);
    const int nchunks = min(BN / CW, (p.cout - tc.n0 + CW - 1) / CW);
    // ---- while the MMAs of this tile run: stage its scale / bias slice in shared memory and start this warp's first
    //      residual load
    epi_bar_sync<kEpiThreads>();   // every warp is done with the previous tile's scale / bias
    if (epi_tid < BN) stage_scale_bias(sb_s, 128, p, tc, epi_tid);
    if (complete && has_res && lane == 0 && half < nchunks) {
      mbar_arrive_expect_tx(rbar, 4096);
      tma_load_4d(reinterpret_cast<void*>(smem + kChainEpiOffset + ew * 8192 + 4096), tmRes, rbar,
                  tc.n0 + half * CW + tc.batch * p.res_c_off, box.w, box.h, box.res_n);
    }
    epi_bar_sync<kEpiThreads>();
    tr.put(TR_TAG(layer, tile_item, 4));
    bool finalize = complete;
    int c_first = cta, c_last = cta;
    if (!complete) {
      // ---- publish this CTA's partial accumulator (each warp its own columns), then find out whether it arrived last
      float* part = sk_own_part_row(p, cta, tile_item, row, BN);
      for (int c = half; c < BN / CW; c += 2) {
#pragma unroll 1
        for (int h = 0; h < HPC; ++h) {
          uint32_t acc[32];
          ring_take(ring, ring_full, ring_empty, half, ruse++, row, acc);
          sk_publish(part, (c * HPC + h) * 32, acc);
        }
      }
      finalize = sk_elect_finisher<kEpiThreads>(p, U, grid, KB, t, epi_tid, epi_flag, c_first, c_last);
    }
    if (finalize) {
      const int out_n = tc.img + tc.batch * p.out_n_off;
#pragma unroll 1
      for (int c = half; c < nchunks; c += 2) {
        const int nb = tc.n0 + c * CW;
        if (has_res) {
          if ((!complete || c != half) && lane == 0) {   // (whole tiles started their first load before the MMAs)
            mbar_arrive_expect_tx(rbar, 4096);
            tma_load_4d(reinterpret_cast<void*>(smem + kChainEpiOffset + ew * 8192 + 4096), tmRes, rbar,
                        nb + tc.batch * p.res_c_off, box.w, box.h, box.res_n);
          }
          mbar_wait(rbar, (rphase >> ew) & 1u);
          rphase ^= (1u << ew);
          tr.put(TR_TAG(layer, tile_item, 5));
        }
        // this warp's store staging was handed to a TMA store one chunk (usually one tile) ago: wait until it was read
        if (lane == 0) tma_store_wait_read<0>();
        __syncwarp();
#pragma unroll
        for (int h = 0; h < HPC; ++h) {
          const int col0 = c * CW + h * 32;     // first column of this half inside the tile
          uint32_t raw[32];
          if (complete) {
            ring_take(ring, ring_full, ring_empty, half, ruse++, row, raw);
          } else {
            float sum[32];
            sk_reduce(p, U, grid, KB, t, c_first, c_last, row, BN, col0, sum);
#pragma unroll
            for (int j = 0; j < 32; ++j) raw[j] = __float_as_uint(sum[j]);
          }
          epi_half_dispatch<OUT16>(raw, sb_u32 + col0 * 4, out_row, res_row, off, h, has_res, relu);
        }
        fence_async_smem();
        __syncwarp();
        const int gc0 = nb + tc.batch * p.out_c_off;
        if (gc0 + CW > p.out_tail0) store_tail<OUT16>(p, smem + kChainEpiOffset + ew * 8192 + lane * 128, gc0, CW, box, out_n, lane);
        if (lane == 0 && gc0 < p.out_tail0) {
          tma_store_4d(tmOut, smem + kChainEpiOffset + ew * 8192, gc0, box.w, box.h, out_n);
          tma_store_commit();
        }
      }
    }
    if (complete) {
      // chunks of this warp's parity past cout: hand their ring slots back unread
      const int c0 = nchunks + ((nchunks & 1) != half ? 1 : 0);
      for (int c = c0; c < BN / CW; c += 2)
#pragma unroll
        for (int h = 0; h < HPC; ++h) ring_skip(ring, ring_full, ring_empty, half, ruse++, row);
    }
    tr.put(TR_TAG(layer, tile_item, 6));
  }
}

__global__ void __launch_bounds__(kChainThreads, 1)
conv_chain_kernel(const ChainLayer* __restrict__ layers, const int n_layers, unsigned* sync, const ChainTrace trace,
                  const int depth) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (the 128B swizzle pattern is a function of the absolute address) as an OFFSET into the shared
  // array, so that the compiler keeps the shared address space (ld/st.shared instead of generic accesses)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kChainBarOffset);
  uint64_t* empty_bar = full_bar + kChainStages;
  uint64_t* ring_full = empty_bar + kChainStages;       // [kRingSlots]
  uint64_t* ring_empty = ring_full + kRingSlots;         // [kRingSlots]
  uint64_t* res_bar = ring_empty + kRingSlots;           // [8 epilogue warps]
  int* epi_flag = reinterpret_cast<int*>(res_bar + 8);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int grid = gridDim.x;
  const int cta = blockIdx.x;

  if (warp == kChainProducerWarp && lane == 31) {
    for (int s = 0; s < kChainStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);      // one arrival per MMA warp
    }
    for (int b = 0; b < kRingSlots; ++b) {
      mbar_init(&ring_full[b], 256);    // every MMA thread
      mbar_init(&ring_empty[b], 4);     // the four epilogue warps of one chunk parity
    }
    for (int b = 0; b < kEpiWarps; ++b) mbar_init(&res_bar[b], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  griddep_launch_dependents();

  if (warp == kChainProducerWarp) {
    // ===================== TMA producer =====================
    if (lane < 2) {
      PipeState ps = {0, 0};
      TraceCursor tr = trace_cursor(trace, 0, cta);
      if (lane != 0) tr.p = nullptr;
      for (int l = 0; l < n_layers; ++l) {
        const ChainLayer* L = layers + l;
        if (lane == 0) prefetch_tmap(&L->tmA); else prefetch_tmap(&L->tmB);
        // everything the loop needs from the layer table is fetched BEFORE the grid barrier
        const ConvGemmParams p = L->p;
        const int BN = L->block_n;
        const int act = L->active_ctas;
        const uint32_t tx_bytes = static_cast<uint32_t>((kBM + BN) * 128);
        tr.put(TR_TAG(l, 0, 1));
        // layer l may read what layers <= l - depth wrote: all CTAs have arrived l / depth times at counter l % depth
        if (l >= depth) grid_wait(sync + (l % depth), static_cast<unsigned>(l / depth) * grid);
        tr.put(TR_TAG(l, 0, 2));
        int lc = cta - L->cta_rot;
        if (lc < 0) lc += grid;
        if (lc >= act) continue;
        WorkIter it(p, lc, act);
        int t;
        int kb0, kb1;
        while (it.next(t, kb0, kb1)) {
          const TileCoord tc = decode_tile(p, t, BN);
          produce_pass<kChainStages>(&L->tmA, &L->tmB, full_bar, empty_bar, ps, smem, kChainStageBytes, kChainABytes, 0, 64,
                                     tx_bytes, p, tc, tc.n0, kb0, kb1, lane, [&](int kb) { tr.put(TR_TAG(l, kb, 3)); });
        }
      }
    }
  } else if (warp >= kChainMmaWarp0 && warp < kChainMmaWarp0 + 8) {
    // ===================== MMA warpgroups =====================
    const int wg = (warp - kChainMmaWarp0) >> 2;     // tile rows [64 wg, 64 wg + 64)
    const int wtid = threadIdx.x - (kChainMmaWarp0 + 4 * wg) * 32;
    MmaState ms = {0, 0, {0, 0}};
    TraceCursor tr = trace_cursor(trace, 1, cta);
    if (wtid != 0 || wg != 0) tr.p = nullptr;
    uint8_t* ring = smem + kChainRingOffset;
    for (int l = 0; l < n_layers; ++l) {
      const ChainLayer* L = layers + l;
      const ConvGemmParams p = L->p;
      const int BN = L->block_n;
      const int act = L->active_ctas;
      int lc = cta - L->cta_rot;
      if (lc < 0) lc += grid;
      if (lc >= act) continue;
      WorkIter it(p, lc, act);
      int t;
      int kb0, kb1;
      const int hpc = L->out16 ? 2 : 1;       // 32-column chunks per epilogue chunk of this layer
      while (it.next(t, kb0, kb1)) {
        tr.put(TR_TAG(l, kb0, 7));
        switch (BN) {
          case 32: mma_pass<32, kChainStages, kModeF16, ChainSmemLayout>(smem, full_bar, empty_bar, empty_bar, ring, ring_full,
                                                                          ring_empty, ms, kb0, kb1, 0x7fffffff, wg, wtid, hpc); break;
          case 64: mma_pass<64, kChainStages, kModeF16, ChainSmemLayout>(smem, full_bar, empty_bar, empty_bar, ring, ring_full,
                                                                          ring_empty, ms, kb0, kb1, 0x7fffffff, wg, wtid, hpc); break;
          case 96: mma_pass<96, kChainStages, kModeF16, ChainSmemLayout>(smem, full_bar, empty_bar, empty_bar, ring, ring_full,
                                                                          ring_empty, ms, kb0, kb1, 0x7fffffff, wg, wtid, hpc); break;
          default: mma_pass<128, kChainStages, kModeF16, ChainSmemLayout>(smem, full_bar, empty_bar, empty_bar, ring, ring_full,
                                                                           ring_empty, ms, kb0, kb1, 0x7fffffff, wg, wtid, hpc); break;
        }
      }
    }
  } else if (warp >= kChainEpiWarp0 && warp < kChainEpiWarp0 + kEpiWarps) {
    // ===================== epilogue (warps 8..15) =====================
    const int epi_tid = (warp - kChainEpiWarp0) * 32 + lane;
    uint32_t ruse = 0;    // chunks this warp took from its ring slot
    uint32_t rphase = 0;
    TraceCursor tr = trace_cursor(trace, 2, cta);
    if (epi_tid != 0) tr.p = nullptr;
    for (int l = 0; l < n_layers; ++l) {
      const ChainLayer* L = layers + l;
      if (lane == 0) {
        prefetch_tmap(&L->tmOut);
        prefetch_tmap(&L->tmRes);
      }
      // residual / partial-sum reads of this layer must see what the other CTAs wrote in earlier layers
      // (one poller per CTA; the named barrier passes the acquired state on to the other epilogue threads)
      if (l >= depth) {
        if (epi_tid == 0) grid_wait(sync + (l % depth), static_cast<unsigned>(l / depth) * grid);
        epi_bar_sync<kEpiThreads>();
        fence_proxy_async_all();
      }
      const ConvGemmParams p = L->p;
      const int act = L->active_ctas;
      int lc = cta - L->cta_rot;
      if (lc < 0) lc += grid;
      if (lc < act) {
        if (L->out16) {
          chain_epilogue_layer<true>(L, p, L->block_n, smem, ring_full, ring_empty, res_bar, epi_flag,
                                     warp, lane, lc, act, ruse, rphase, tr, l);
        } else {
          chain_epilogue_layer<false>(L, p, L->block_n, smem, ring_full, ring_empty, res_bar, epi_flag,
                                      warp, lane, lc, act, ruse, rphase, tr, l);
        }
      }
      tr.put(TR_TAG(l, 0, 8));
      // this CTA's part of layer l is complete and visible: arrive at the grid barrier
      // (stream-K partial sums were fenced by their writers; the TMA stores of every warp are complete after its
      //  wait_group; the named barrier orders all of that before thread 0's single gpu-scope release)
      if (lane == 0) tma_store_wait<0>();
      tr.put(TR_TAG(l, 0, 9));
      epi_bar_sync<kEpiThreads>();
      if (epi_tid == 0) {
        fence_proxy_async_all();
        __threadfence();
        atomicAdd(sync + (l % depth), 1u);
      }
      tr.put(TR_TAG(l, 0, 10));
    }
    // last CTA out resets the barrier words for the next launch (every CTA has passed every barrier by then)
    if (epi_tid == 0) {
      const unsigned old = atomicAdd(sync + depth, 1u);
      if (old == static_cast<unsigned>(grid) - 1) {
        for (int i = 0; i <= depth; ++i) sync[i] = 0;
        __threadfence();
      }
    }
  }
}

// defined in conv_gemm.cu: validates a descriptor and encodes its tensor maps / kernel parameters
int encode_conv_gemm_problem(const mega_conv_gemm_desc* d, CUtensorMap* tmA, CUtensorMap* tmB, CUtensorMap* tmOut,
                             CUtensorMap* tmRes, ConvGemmParams* p, int* ctas);

}  // namespace mega

using namespace mega;

extern "C" long long mega_conv_chain_plan_bytes(int n_layers) {
  return static_cast<long long>(n_layers) * static_cast<long long>(sizeof(ChainLayer));
}

extern "C" int mega_conv_chain_encode2(const mega_conv_gemm_desc* descs, int n_layers, void* plan_host,
                                       long long plan_bytes, int* grid_out, int depth) {
  MEGA_ARG_CHECK(descs != nullptr && plan_host != nullptr && n_layers > 0, "conv_chain: bad arguments");
  MEGA_ARG_CHECK(depth == 1 || depth == 2, "conv_chain: barrier depth must be 1 or 2 (got %d)", depth);
  MEGA_ARG_CHECK(plan_bytes >= mega_conv_chain_plan_bytes(n_layers), "conv_chain: plan buffer too small");
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(plan_host) & 127) == 0, "conv_chain: plan buffer must be 128-byte aligned");
  ChainLayer* out = static_cast<ChainLayer*>(plan_host);
  int grid = 1;
  for (int l = 0; l < n_layers; ++l) {
    const mega_conv_gemm_desc* d = descs + l;
    MEGA_ARG_CHECK(d->precision == kModeF16, "conv_chain: layer %d: chains run fp16 operands only", l);
    MEGA_ARG_CHECK(d->block_n <= 128, "conv_chain: layer %d: block_n %d > 128", l, d->block_n);
    MEGA_ARG_CHECK(d->workspace == descs[0].workspace, "conv_chain: every layer must name the same workspace");
    ChainLayer* L = out + l;
    int ctas = 0;
    const int rc = encode_conv_gemm_problem(d, &L->tmA, &L->tmB, &L->tmOut, &L->tmRes, &L->p, &ctas);
    if (rc != MEGA_OK) return rc;
    L->block_n = d->block_n;
    L->out16 = d->out_f16 ? 1 : 0;
    L->active_ctas = ctas;
    L->cta_rot = 0;
    if (ctas > grid) grid = ctas;
    if (depth == 2) {
      // two layers are in flight: odd layers take the second half of the tile counters and of the partial-sum area
      // (block_n <= 128 in a chain, so one half holds kMaxCtas x 2 x 128 x 128 floats)
      MEGA_ARG_CHECK(L->p.total_tiles <= 32768, "conv_chain: layer %d: %lld tiles exceed the 32768 counters of a depth-2 chain", l,
                     L->p.total_tiles);
      if (l & 1) {
        L->p.counters += 32768;
        L->p.part_ws += static_cast<long long>(kMaxCtas) * 2 * kBM * 128;
      }
    }
  }
  if (depth == 2) {
    // rolling work lists: layer l starts at the physical CTA where layer l-1's list ended
    long long start = 0;
    for (int l = 0; l < n_layers; ++l) {
      out[l].cta_rot = static_cast<int>(start % grid);
      // whole-tile layers occupy min(tiles, ctas) CTAs for (about) one tile time each; advance by the tiles of the last,
      // partial wave so that the next layer begins on the CTAs this one leaves idle
      const long long tiles = out[l].p.total_tiles;
      const int act = out[l].active_ctas;
      start += out[l].p.stream_k ? act : (tiles % act == 0 ? act : tiles % act);
    }
  }
  if (grid_out) *grid_out = grid;
  return MEGA_OK;
}

extern "C" int mega_conv_chain_encode(const mega_conv_gemm_desc* descs, int n_layers, void* plan_host,
                                      long long plan_bytes, int* grid_out) {
  return mega_conv_chain_encode2(descs, n_layers, plan_host, plan_bytes, grid_out, 1);
}

static ChainTrace g_chain_trace = {nullptr, 0, 0};

/* diagnostics: the next launches record an in-kernel event trace of CTA `cta` into trace_dev
 * (3 * 4096 * 2 uint64, zero it first); trace_dev == NULL switches tracing off */
extern "C" int mega_conv_chain_set_trace(void* trace_dev, int cta) {
  g_chain_trace.buf = static_cast<unsigned long long*>(trace_dev);
  g_chain_trace.cta = cta;
  g_chain_trace.level = 0;
  return MEGA_OK;
}

/* level 1: only the per-layer events (layer begin / barrier passed / tiles done / stores drained / arrived) */
extern "C" int mega_conv_chain_set_trace2(void* trace_dev, int cta, int level) {
  g_chain_trace.buf = static_cast<unsigned long long*>(trace_dev);
  g_chain_trace.cta = cta;
  g_chain_trace.level = level;
  return MEGA_OK;
}

extern "C" int mega_conv_chain_launch2(const void* plan_device, int n_layers, int grid, void* sync_words, void* stream_v,
                                       int pdl, int depth) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(plan_device != nullptr && sync_words != nullptr && n_layers > 0 && grid > 0 && grid <= kMaxCtas,
                 "conv_chain_launch: bad arguments (grid %d)", grid);
  MEGA_ARG_CHECK(depth == 1 || depth == 2, "conv_chain_launch: barrier depth must be 1 or 2 (got %d)", depth);
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(plan_device) & 127) == 0, "conv_chain_launch: plan must be 128-byte aligned");
  static bool configured = false;
  if (!configured) {
    MEGA_CUDA_CHECK(cudaFuncSetAttribute(conv_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmem));
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(grid), 1, 1);
  cfg.blockDim = dim3(kChainThreads, 1, 1);
  cfg.dynamicSmemBytes = kChainSmem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  MEGA_CUDA_CHECK(cudaLaunchKernelEx(&cfg, conv_chain_kernel, static_cast<const ChainLayer*>(plan_device), n_layers,
                                     static_cast<unsigned*>(sync_words), g_chain_trace, depth));
  return MEGA_OK;
}

extern "C" int mega_conv_chain_launch(const void* plan_device, int n_layers, int grid, void* sync_words, void* stream_v,
                                      int pdl) {
  return mega_conv_chain_launch2(plan_device, n_layers, grid, sync_words, stream_v, pdl, 1);
}
