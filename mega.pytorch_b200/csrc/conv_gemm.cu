#include "conv_gemm_kernel.cuh"

namespace mega {

template MEGA_LAUNCH_MODE(kModeTf32);
template MEGA_LAUNCH_MODE(kModeSplit3);

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || p == nullptr) {
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

static int g_tf32_round = 1;  // TMA converts fp32 -> tf32 (round to nearest) while loading

static int g_num_sms = 0;
static int g_seg_len = 4;      // 3xTF32 / 3xFP16: k-blocks per accumulator segment (tools/strict_probe.py: 2 / 4 / 8 -> logits p99 1.8e-4 / 2.3e-4 / 5.3e-4)
constexpr int kCounterSlots = 65536;   // ints at the head of the workspace
constexpr int kMinUnits = 4;

}  // namespace mega

using namespace mega;

extern "C" long long mega_conv_gemm_workspace_bytes(void) {
  return static_cast<long long>(kCounterSlots) * sizeof(int) +
         static_cast<long long>(kMaxCtas) * 2 * kBM * 256 * sizeof(float);
}

extern "C" int mega_set_split3_seg_len(int k_blocks) {
  int old = g_seg_len;
  if (k_blocks >= 1 && k_blocks <= 64) g_seg_len = k_blocks;
  return old;
}

extern "C" int mega_set_tf32_rounding(int enable) {
  int old = g_tf32_round;
  g_tf32_round = enable ? 1 : 0;
  return old;
}

namespace mega {

// validates a descriptor, encodes its four tensor maps and fills the kernel parameters; *ctas = CTAs of the
// persistent work list (shared by the single-launch path below and the layer chains of conv_chain.cu)
int encode_conv_gemm_problem(const mega_conv_gemm_desc* d, CUtensorMap* tmA_p, CUtensorMap* tmB_p, CUtensorMap* tmOut_p,
                             CUtensorMap* tmRes_p, ConvGemmParams* p_out, int* ctas_out) {
  MEGA_ARG_CHECK(d != nullptr, "conv_gemm: null descriptor");
  MEGA_ARG_CHECK(d->precision >= 0 && d->precision <= 3,
                 "conv_gemm: precision must be 0 (tf32), 1 (3xtf32), 2 (fp16 operands) or 3 (3xfp16, split-fp16 operands)");
  const bool strict = d->precision == kModeSplit3;
  const bool f16 = d->precision == kModeF16;
  const bool pk = d->precision == kModeF16x3;  // split-fp16 tensors are addressed like fp32 tensors (4 bytes per value)
  const bool out16 = d->out_f16 != 0 && !pk;
  const int esz = f16 ? 2 : 4;                 // operand element size
  const int osz = out16 ? 2 : 4;               // output / residual element size
  const int ealign = 16 / esz, oalign = 16 / osz;
  const int bk = mode_bk(d->precision);
  MEGA_ARG_CHECK(d->tile_h > 0 && d->tile_w > 0 && d->tile_h * d->tile_w == kBM,
                 "conv_gemm: tile_h*tile_w must be 128 (got %dx%d)", d->tile_h, d->tile_w);
  MEGA_ARG_CHECK(d->tile_w <= 256 && d->tile_h <= 256, "conv_gemm: tile too large for a TMA box");
  const int stride_h = d->stride_h > 0 ? d->stride_h : 1, stride_w = d->stride_w > 0 ? d->stride_w : 1;
  MEGA_ARG_CHECK((d->tile_w - 1) * stride_w + 1 <= 256 && (d->tile_h - 1) * stride_h + 1 <= 256,
                 "conv_gemm: strided tile %dx%d (stride %dx%d) exceeds the 256-element TMA box", d->tile_h, d->tile_w,
                 stride_h, stride_w);
  MEGA_ARG_CHECK(d->block_n == 32 || d->block_n == 64 || d->block_n == 96 || d->block_n == 128 ||
                     d->block_n == 160 || d->block_n == 192 || d->block_n == 256,
                 "conv_gemm: block_n must be one of 32/64/96/128/160/192/256");
  MEGA_ARG_CHECK(!out16 || (f16 && d->block_n % 64 == 0),
                 "conv_gemm: fp16 output needs fp16 operands and block_n %% 64 == 0 (got precision %d, block_n %d)",
                 d->precision, d->block_n);
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(d->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->b) & 15) == 0,
                 "conv_gemm: operand base pointers must be 16-byte aligned");
  MEGA_ARG_CHECK((d->a_stride_w % ealign) == 0 && (d->a_stride_h % ealign) == 0 && (d->a_stride_n % ealign) == 0,
                 "conv_gemm: activation strides must be multiples of 16 bytes");
  MEGA_ARG_CHECK(d->out != nullptr && (reinterpret_cast<uintptr_t>(d->out) & 15) == 0 && (d->out_ld % oalign) == 0,
                 "conv_gemm: output must be 16-byte aligned with a row pitch multiple of 16 bytes");
  MEGA_ARG_CHECK(d->residual == nullptr ||
                     ((reinterpret_cast<uintptr_t>(d->residual) & 15) == 0 && (d->res_ld % oalign) == 0),
                 "conv_gemm: residual must be 16-byte aligned with a row pitch multiple of 16 bytes");
  MEGA_ARG_CHECK(d->out_c_off == 0 || d->cout == d->block_n,
                 "conv_gemm: channel-offset batching needs cout == block_n (got %d vs %d)", d->cout, d->block_n);
  MEGA_ARG_CHECK((d->b_stride_n % ealign) == 0 && (d->b_stride_tap % ealign) == 0,
                 "conv_gemm: weight strides must be multiples of 16 bytes");
  MEGA_ARG_CHECK(d->batch >= 1, "conv_gemm: batch must be >= 1");
  MEGA_ARG_CHECK(d->workspace != nullptr && d->workspace_bytes >= mega_conv_gemm_workspace_bytes(),
                 "conv_gemm: workspace missing or smaller than mega_conv_gemm_workspace_bytes()");
  MEGA_ARG_CHECK((reinterpret_cast<uintptr_t>(d->workspace) & 255) == 0, "conv_gemm: workspace must be 256-byte aligned");
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    mega_set_error("conv_gemm: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return MEGA_ERR_CUDA;
  }
  MEGA_ARG_CHECK(!(strict || pk) || d->block_n == 64 || d->block_n == 128, "conv_gemm: 3xtf32 / 3xfp16 support block_n 64 / 128");
  if (pk) {
    MEGA_ARG_CHECK((d->a_c & 31) == 0 && (d->b_k & 31) == 0 && (d->k_per_tap & 31) == 0 && (d->a_c_off & 31) == 0 &&
                       (d->b_k_off & 31) == 0,
                   "conv_gemm: split-fp16 operands need channel counts / offsets in multiples of 32 (a_c %d, b_k %d, k %d)",
                   d->a_c, d->b_k, d->k_per_tap);
    // a ragged cout is rounded up to whole 32-value groups (the extra columns are computed from zero-filled B rows and must
    // fit inside the row pitch); batched launches address whole groups only
    const int cout_r = (d->cout + 31) & ~31;
    MEGA_ARG_CHECK(d->out_f16 == 0 || ((d->out_c_off & 31) == 0 && (d->cout == cout_r || (d->batch == 1 && d->out_ld >= cout_r))),
                   "conv_gemm: split-fp16 output needs cout (%d) in multiples of 32 (or batch 1 and a row pitch >= the rounded cout)", d->cout);
    MEGA_ARG_CHECK(d->res_split == 0 || d->residual == nullptr ||
                       ((d->res_c_off & 31) == 0 && (d->cout == cout_r || (d->batch == 1 && d->res_ld >= cout_r))),
                   "conv_gemm: split-fp16 residual needs cout (%d) in multiples of 32", d->cout);
    MEGA_ARG_CHECK((d->a_stride_w & 31) == 0 && (d->b_stride_n & 31) == 0 && (reinterpret_cast<uintptr_t>(d->a) & 127) == 0 &&
                       (reinterpret_cast<uintptr_t>(d->b) & 127) == 0,
                   "conv_gemm: split-fp16 operands need 128-byte aligned rows");
    MEGA_ARG_CHECK(d->scale == nullptr,
                   "conv_gemm: precision 3 takes no per-channel scale: fold it into the weights before packing them "
                   "(mega_core.b200.ops.pack_weights_split16(w, scale))");
  } else {
    MEGA_ARG_CHECK(d->res_split == 0, "conv_gemm: res_split needs precision 3");
  }
  if (d->group_width != 0) {
    const int gw = d->group_width;
    MEGA_ARG_CHECK(gw == 8 || gw == 16 || gw == 32 || gw == 64, "conv_gemm: group_width must be 8, 16, 32 or 64 (got %d)", gw);
    MEGA_ARG_CHECK(d->block_n == 64 && d->cout == 64 && d->k_per_tap == 64 && d->b_k == 64 && d->a_c_off == 64 &&
                       d->b_n_off == 64 && d->out_c_off == 64 && d->b_k_off == 0 && (d->residual == nullptr || d->res_c_off == 64),
                   "conv_gemm: group_width needs the 64-channel batched layout (block_n = cout = k_per_tap = b_k = 64, "
                   "a_c_off = b_n_off = out_c_off = res_c_off = 64, b_k_off = 0; got block_n %d cout %d k %d b_k %d offsets "
                   "%d %d %d %d %d)", d->block_n, d->cout, d->k_per_tap, d->b_k, d->a_c_off, d->b_n_off, d->out_c_off,
                   d->res_c_off, d->b_k_off);
    MEGA_ARG_CHECK(d->b_lo_tap_off == 0, "conv_gemm: group_width does not take pre-split weights (b_lo_tap_off)");
  }
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                     : (g_tf32_round && !strict && !pk) ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32
                                                                 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const CUtensorMapDataType odt = out16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;

  CUtensorMap& tmA = *tmA_p;
  CUtensorMap& tmB = *tmB_p;
  {
    cuuint64_t gdim[4] = {static_cast<cuuint64_t>(d->a_c), static_cast<cuuint64_t>(d->a_w),
                          static_cast<cuuint64_t>(d->a_h), static_cast<cuuint64_t>(d->a_n)};
    cuuint64_t gstr[3] = {static_cast<cuuint64_t>(d->a_stride_w) * esz, static_cast<cuuint64_t>(d->a_stride_h) * esz,
                          static_cast<cuuint64_t>(d->a_stride_n) * esz};
    // a strided convolution samples every stride-th pixel of the rectangle: TMA element strides (the box is the
    // bounding rectangle, the copy delivers tile_w x tile_h pixels)
    cuuint32_t box[4] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>((d->tile_w - 1) * stride_w + 1),
                         static_cast<cuuint32_t>((d->tile_h - 1) * stride_h + 1), 1};
    cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride_w), static_cast<cuuint32_t>(stride_h), 1};
    CUresult r = enc(&tmA, dt, 4, const_cast<void*>(d->a), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      mega_set_error("conv_gemm: encode A tensor map failed (CUresult %d) dims %d %d %d %d strides %lld %lld %lld",
                     static_cast<int>(r), d->a_c, d->a_w, d->a_h, d->a_n, d->a_stride_w, d->a_stride_h,
                     d->a_stride_n);
      return MEGA_ERR_CUDA;
    }
  }
  {
    const int taps = d->taps_r * d->taps_s;
    MEGA_ARG_CHECK(d->b_lo_tap_off == 0 || (strict && d->b_lo_tap_off == taps && d->batch == 1),
                   "conv_gemm: b_lo_tap_off (%d) needs precision 1, batch 1 and must equal taps_r * taps_s (%d)",
                   d->b_lo_tap_off, taps);
    cuuint64_t gdim[3] = {static_cast<cuuint64_t>(d->b_k), static_cast<cuuint64_t>(d->b_n),
                          static_cast<cuuint64_t>(taps + d->b_lo_tap_off)};
    cuuint64_t gstr[2] = {static_cast<cuuint64_t>(d->b_stride_n) * esz,
                          static_cast<cuuint64_t>((taps > 1 || d->b_lo_tap_off) && d->b_stride_tap > 0
                                                      ? d->b_stride_tap : d->b_stride_n * d->b_n) * esz};
    cuuint32_t box[3] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(pass_n(d->block_n)), 1};   // one pass
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&tmB, dt, 3, const_cast<void*>(d->b), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      mega_set_error("conv_gemm: encode B tensor map failed (CUresult %d) dims %d %d %d strides %lld %lld",
                     static_cast<int>(r), d->b_k, d->b_n, taps, d->b_stride_n, d->b_stride_tap);
      return MEGA_ERR_CUDA;
    }
  }

  // per-warp store / residual boxes: one 128-byte row segment (32 floats / 64 halves) x (box_h x box_w = 32 output
  // pixels), 128B swizzle
  CUtensorMap& tmOut = *tmOut_p;
  CUtensorMap& tmRes = *tmRes_p;
  int out_cext = 0, out_tail0 = 0;
  long long out_str_h = 0, out_str_n = 0;
  {
    const int box_w = d->tile_w < 32 ? d->tile_w : 32;
    const int box_h = 32 / box_w;
    const int cw = out16 ? 64 : 32;
    for (int which = 0; which < 2; ++which) {
      const void* base = which == 0 ? d->out : d->residual;
      CUtensorMap* tm = which == 0 ? &tmOut : &tmRes;
      if (base == nullptr) {
        *tm = tmOut;
        continue;
      }
      const long long ld = which == 0 ? d->out_ld : d->res_ld;
      const int c_off = which == 0 ? d->out_c_off : d->res_c_off;
      const int n_off = which == 0 ? d->out_n_off : d->res_n_off;
      const bool split_fmt = pk && (which == 0 ? d->out_f16 != 0 : d->res_split != 0);
      const int c_extent = (split_fmt ? ((d->cout + 31) & ~31) : d->cout) + (d->batch - 1) * c_off;
      // the store's channel extent ends at the last 16-byte boundary (the TMA unit clips stores at 16-byte granularity);
      // the epilogue writes the rest of the row with plain stores (ConvGemmParams::out_tail0)
      const int c_tail0 = (c_extent * osz / 16) * 16 / osz;
      if (which == 0) {
        out_cext = c_extent;
        out_tail0 = c_tail0;
      }
      const int c_map = (which == 0 && c_tail0 > 0) ? c_tail0 : c_extent;
      cuuint64_t gdim[4] = {static_cast<cuuint64_t>(c_map), static_cast<cuuint64_t>(d->out_w),
                            static_cast<cuuint64_t>(d->out_h),
                            static_cast<cuuint64_t>(d->n_img + (d->batch - 1) * n_off)};
      const long long sh = which == 0 ? d->out_stride_h : d->res_stride_h;
      const long long sn = which == 0 ? d->out_stride_n : d->res_stride_n;
      const long long str_h = sh > 0 ? sh : ld * d->out_w;
      const long long str_n = sn > 0 ? sn : str_h * d->out_h;
      MEGA_ARG_CHECK((str_h % oalign) == 0 && (str_n % oalign) == 0, "conv_gemm: output strides must be multiples of 16 bytes");
      if (which == 0) {
        out_str_h = str_h;
        out_str_n = str_n;
      }
      cuuint64_t gstr[3] = {static_cast<cuuint64_t>(ld) * osz, static_cast<cuuint64_t>(str_h) * osz,
                            static_cast<cuuint64_t>(str_n) * osz};
      cuuint32_t box[4] = {static_cast<cuuint32_t>(cw), static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(box_h), 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(tm, odt, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) {
        mega_set_error("conv_gemm: encode %s tensor map failed (CUresult %d): C %d W %d H %d N %d ld %lld",
                       which == 0 ? "output" : "residual", static_cast<int>(r), static_cast<int>(gdim[0]), d->out_w,
                       d->out_h, static_cast<int>(gdim[3]), ld);
        return MEGA_ERR_CUDA;
      }
    }
  }

  ConvGemmParams& p = *p_out;
  p.tile_w = d->tile_w;
  p.tile_h = d->tile_h;
  p.tiles_w = mega_ceil_div(d->out_w, d->tile_w);
  p.tiles_h = mega_ceil_div(d->out_h, d->tile_h);
  p.out_h = d->out_h;
  p.out_w = d->out_w;
  p.n_img = d->n_img;
  p.taps_r = d->taps_r;
  p.taps_s = d->taps_s;
  p.dil = d->dil;
  p.pad = d->pad;
  p.pad_w = d->pad_w_set ? d->pad_w : d->pad;
  p.stride_h = stride_h;
  p.stride_w = stride_w;
  p.k_chunks = mega_ceil_div(d->k_per_tap, bk);
  p.cout = d->cout;
  p.scale = d->scale;
  p.bias = d->bias;
  p.has_residual = d->residual != nullptr;
  p.relu = d->relu;
  p.a_c_off = d->a_c_off;
  p.a_n_off = d->a_n_off;
  p.b_k_off = d->b_k_off;
  p.b_n_off = d->b_n_off;
  p.out_c_off = d->out_c_off;
  p.out_n_off = d->out_n_off;
  p.res_c_off = d->res_c_off;
  p.res_n_off = d->res_n_off;
  p.bias_z_off = d->bias_z_off;
  p.box_w = d->tile_w < 32 ? d->tile_w : 32;
  p.box_h = 32 / p.box_w;
  p.m_tiles = p.tiles_w * p.tiles_h * p.n_img;
  p.n_tiles = mega_ceil_div(d->cout, d->block_n);
  p.kb_per_tile = d->taps_r * d->taps_s * p.k_chunks;
  const long long tiles = static_cast<long long>(d->batch) * p.m_tiles * p.n_tiles;
  p.total_units = tiles * p.kb_per_tile;
  p.total_tiles = tiles;
  p.stream_k = d->stream_k ? 1 : 0;
  p.n_fast = 0;
  p.seg_len = g_seg_len;
  p.b_lo_tap_off = d->b_lo_tap_off;
  p.res_split = d->res_split ? 1 : 0;
  p.acc_scale = (pk && d->acc_scale != 0.f) ? d->acc_scale : 1.f;
  p.out_ptr = d->out;
  p.out_ld = d->out_ld;
  p.out_str_h = out_str_h;
  p.out_str_n = out_str_n;
  p.out_tail0 = out_tail0;
  p.out_cext = out_cext;
  MEGA_ARG_CHECK(tiles <= kCounterSlots, "conv_gemm: %lld output tiles exceed the %d counter slots", tiles, kCounterSlots);
  MEGA_ARG_CHECK(p.total_units > 0, "conv_gemm: empty problem");
  MEGA_ARG_CHECK(p.total_units * kMaxCtas < (1LL << 31), "conv_gemm: %lld work units exceed the 32-bit work-list range",
                 p.total_units);
  p.counters = static_cast<int*>(d->workspace);
  p.part_ws = reinterpret_cast<float*>(static_cast<char*>(d->workspace) + kCounterSlots * sizeof(int));
  if (g_num_sms == 0) {
    int dev = 0;
    MEGA_CUDA_CHECK(cudaGetDevice(&dev));
    MEGA_CUDA_CHECK(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
    if (g_num_sms > kMaxCtas) g_num_sms = kMaxCtas;
  }
  // persistent grid: one CTA per SM, but never fewer than kMinUnits k-blocks of work per CTA
  long long ctas = p.stream_k ? p.total_units / kMinUnits : tiles;
  if (ctas < 1) ctas = 1;
  if (ctas > g_num_sms) ctas = g_num_sms;
  if (d->max_ctas > 0 && ctas > d->max_ctas) ctas = d->max_ctas;
  // Very deep reductions (the 100352-deep l_fcs[0]) stream operands larger than L2. With a grid that is a multiple of
  // the tile count every tile is cut at the same k offsets, so the CTAs that share an A row block or a B column block
  // read the same k-blocks at the same time and each operand byte comes from DRAM once (3.08 CTAs per tile let the
  // m-tiles of one weight slab drift > L2 apart: 571 MB of DRAM reads for 280 MB of operands).
  if (p.stream_k && p.kb_per_tile >= 256 && tiles <= ctas) {
    const long long aligned = (ctas / tiles) * tiles;
    if (aligned * 100 >= ctas * 85) ctas = aligned;
  }
  *ctas_out = static_cast<int>(ctas);
  return MEGA_OK;
}

}  // namespace mega

extern "C" int mega_conv_gemm(const mega_conv_gemm_desc* d, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  CUtensorMap tmA, tmB, tmOut, tmRes;
  ConvGemmParams p;
  int ctas = 0;
  const int erc = encode_conv_gemm_problem(d, &tmA, &tmB, &tmOut, &tmRes, &p, &ctas);
  if (erc != MEGA_OK) return erc;
  // 3xFP16 whole tiles run n-fastest: the CTAs of one wave then cover a few M tiles with all their N tiles, so each
  // activation tile comes from HBM once and its other N tiles read it from L2. In m-fastest order, the next N tile reads
  // the same A tile a wave later, and an A larger than L2 (res4 conv1, the res5 1x1 convs: 78 MB) comes from HBM once
  // per N tile. Stream-K launches keep the m-fastest order, and with it their split points.
  if (d->precision == kModeF16x3 && !p.stream_k && p.n_tiles > 1) p.n_fast = 1;
  const bool out16 = d->out_f16 != 0;
  dim3 grid(static_cast<unsigned>(ctas), 1, 1);
  const int pdl = d->pdl ? 1 : 0;
  // grouped launches (block_n 64, checked by the encoder) issue only the diagonal blocks; with one group per 64 channels
  // (gw 64) that is the dense k-block. The layer chain runs grouped layers with the dense issue (same result).
  const int gw = d->group_width == 64 ? 0 : d->group_width;
  switch (d->precision) {
    case kModeTf32: return launch_mode<kModeTf32>(d->block_n, out16, gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
    case kModeSplit3: return launch_mode<kModeSplit3>(d->block_n, out16, gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
    case kModeF16: return launch_mode<kModeF16>(d->block_n, out16, gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
    default: return launch_mode<kModeF16x3>(d->block_n, out16, gw, tmA, tmB, tmOut, tmRes, p, grid, stream, pdl);
  }
}

/* the name under which ABI version 1 exported the same entry point */
extern "C" int mega_conv_gemm_tf32(const mega_conv_gemm_desc* d, void* stream) { return mega_conv_gemm(d, stream); }
