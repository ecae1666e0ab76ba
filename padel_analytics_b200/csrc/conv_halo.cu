// 3x3 / stride-1 conv + bias + activation as an implicit GEMM whose nine filter taps are all served from ONE
// shared-memory halo tile per 64(32/16)-channel block.
//
// Why: with one TMA box per tap (conv_tc_kernel) every K-block of a small-N layer moves 16 KB of activations for
// four k-steps of MMAs, and the kernel is bound by L2->SM / TMA delivery on TrackNet's N=64 layers.  Here the CTA tile is 16 rows x (8*S) columns of output pixels = S sub-tiles of M=128; its
// (16+2) x (8*S+2) pixel halo is fetched by a single TMA box, and tap (r,s) of sub-tile j is just a different
// wgmma descriptor over the same bytes:
//     start = halo + ((r*P + 8*j + s) * row_bytes),   SBO (8-row group stride) = P * row_bytes,   P = 8*S + 2
// (one 8-row group = 8 horizontally adjacent pixels, consecutive groups = consecutive image rows).  This relies on
// the tensor core applying the 128/64/32-byte swizzle XOR on absolute shared-memory address bits (descriptor base
// offset 0 for any row shift / any SBO); tests/test_conv_gpu.py checks every halo variant against torch.
// Weights are fetched per (channel block, tap group) by a second producer warp and shared by the S sub-tile MMAs.
//
// Replaces the same reference layers as conv_tc.cu (TrackNet Conv2DBlock models.py:5-17; ultralytics 3x3 convs).
#include <cstdlib>
#include <mutex>
#include <vector>

#include "conv_halo_kernel.cuh"

namespace pb {

// ------------------------------------------------------------------------------------------------------------
// host: geometry + tensor maps for the halo variant. Returns 0 and sets plan->variant = 1 when applicable,
// returns -1 (no error) when the layer should use the per-tap kernel.
// ------------------------------------------------------------------------------------------------------------

// shared memory for the rings and the staging tile (the tail and the alignment slack come on top, <= 227 KB)
constexpr size_t kHaloSmemBudget = 196 * 1024;

// TMA-store epilogue (conv_halo_kernel.cuh::halo_epilogue_tma) for an fp16 output without residual whose N tile is
// stored whole: the staging tile (S * BN * 256 bytes) joins the rings inside the budget -- the weight ring down to four,
// then the halo ring down to two, then the weight ring down to three stages; S and G stay as chosen.  Layers where it
// does not fit, or does not apply, keep the per-lane store epilogue.  PADEL_B200_CONV_TMA_STORE=0 disables it (A/B).
static int halo_plan_store(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode) {
  const size_t budget = kHaloSmemBudget;
  static const int enabled = [] {
    const char* e = getenv("PADEL_B200_CONV_TMA_STORE");
    return e ? atoi(e) : 1;
  }();
  ConvKParams& kp = plan->kp;
  kp.st_bytes = 0;
  kp.st_maps = 0;
  kp.st_pool = 0;
  const bool f16 = d->out_mode == PB_OUT_F16_NHWC || d->out_mode == PB_OUT_F16_NHWC_UP2;
  if (!enabled || kp.dbg_flags != 0 || d->res || d->head_n != 0 || !f16 || plan->epi == PB_EPI_SILU_RES ||
      d->cout_store != kp.n_ntiles * kp.BN || ((d->out_C | d->out_coff) & 7) != 0)
    return 0;
  // Deep-K streamed layers (more than two channel blocks) are mainloop-bound and need their third halo stage and
  // deep weight ring more than an asynchronous epilogue (H100: up_block_2.conv_1 of TrackNet ran 5 % slower with it).
  if (!kp.b_resident && kp.kblocks > 2) return 0;
  const uint32_t st = (uint32_t)kp.hs_S * (uint32_t)kp.BN * 256u;
  int as = kp.a_stages, bs = kp.b_stages;
  auto total = [&] { return (size_t)as * kp.a_bytes + (size_t)bs * kp.b_bytes + st; };
  while (total() > budget) {
    if (!kp.b_resident && bs > 4) --bs;
    else if (as > 2) --as;
    else if (!kp.b_resident && bs > 3) --bs;
    else return 0;
  }
  // one map per destination of the staging box (channels, 8S columns, 8 rows, image); base = channel 0 of the slice,
  // which spans the N tiles' cout_store channels
  const int S = kp.hs_S, bc = halo_store_box_channels(kp.BN);
  const CUtensorMapSwizzle swz = bc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : bc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                            : CU_TENSOR_MAP_SWIZZLE_32B;
  int nm = 0;
  auto add = [&](void* out, int C, int coff, int W, int H, int up, int dy, int dx, int bw, int bh) {
    const size_t pxb = (size_t)C * 2;
    char* base = reinterpret_cast<char*>(out) + ((size_t)(dy * up * W + dx) * C + coff) * 2;
    cuuint64_t dims[4] = {(cuuint64_t)d->cout_store, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)kp.N};
    cuuint64_t strides[3] = {up * pxb, (cuuint64_t)up * up * W * pxb, (cuuint64_t)up * up * W * H * pxb};
    cuuint32_t box[4] = {(cuuint32_t)bc, (cuuint32_t)bw, (cuuint32_t)bh, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return encode(&plan->tmap_o.m[nm++], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUresult r = CUDA_SUCCESS;
  const int up = d->out_mode == PB_OUT_F16_NHWC_UP2 ? 2 : 1;
  for (int dy = 0; dy < up; ++dy)
    for (int dx = 0; dx < up; ++dx)
      if (r == CUDA_SUCCESS) r = add(d->out, d->out_C, d->out_coff, kp.Wo, kp.Ho, up, dy, dx, 8 * S, 8);
  if (d->out2_mode == PB_OUT2_UP2) {
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx)
        if (r == CUDA_SUCCESS) r = add(d->out2, d->out2_C, d->out2_coff, kp.Wo, kp.Ho, 2, dy, dx, 8 * S, 8);
  }
  kp.st_maps = nm;
  if (d->out2_mode == PB_OUT2_POOL2 && r == CUDA_SUCCESS) {
    r = add(d->out2, d->out2_C, d->out2_coff, kp.Wo / 2, kp.Ho / 2, 1, 0, 0, 4 * S, 4);
    kp.st_pool = 1;
  }
  PB_CHECK(r == CUDA_SUCCESS, "conv(halo): cuTensorMapEncodeTiled(store) failed with %d", (int)r);
  kp.st_bytes = st;
  kp.a_stages = as;
  kp.b_stages = bs;
  return 0;
}

// Launch configuration shared by the halo set-ups: one persistent CTA per SM.
static void halo_finish_config(ConvPlan* plan) {
  const ConvKParams& kp = plan->kp;
  plan->smem_bytes = (size_t)kp.a_stages * kp.a_bytes + (size_t)kp.b_stages * kp.b_bytes + kp.st_bytes +
                     sizeof(HaloSmemTail) + 1024;
  plan->threads = kConvThreads;
  plan->grid = kp.total_tiles < num_sms() ? kp.total_tiles : num_sms();
}

// Stem (PB_IN_STEM4): 3x3 stride-2 conv over the padded 4-channel input. One TMA box of overlapping 16-element rows
// (4 pixels x 4 channels, consecutive rows 2 pixels apart) holds, for a tile of 16 x 8S outputs, the three filter
// rows r = 0..2 as [oh][r][ow] rows of 32 bytes; filter row r of sub-tile j starts at row (r*8S + 8j), 8-row groups
// (consecutive oh) are 3*8S rows apart.  K = 16 per filter row (12 real), 3 wgmmas per sub-tile.
int conv_stem_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode) {
  PB_CHECK(d->ksize == 3 && d->stride == 2 && d->C == 4 && d->cin == 16 && d->c_in_off == 0,
           "conv(stem): needs ksize 3, stride 2, C = 4, cin = 16");
  PB_CHECK(d->cout_pad <= 128, "conv(stem): cout_pad %d > 128", d->cout_pad);
  ConvKParams& kp = plan->kp;
  const int BN = d->cout_pad;
  const int acc_cols = (BN + 31) / 32 * 32;
  int S = 4;
  while (S > 1 && S * acc_cols > 2 * kConvAccRegs) S >>= 1;  // accumulators of S sub-tiles fit the registers
  kp.KB = 16;
  kp.kblocks = 1;
  kp.taps = 3;
  kp.hs_S = S;
  kp.hs_P = 8 * S;
  kp.hs_G = 3;
  kp.hs_ntaps = 3;
  kp.hs_sbo_rows = 3 * 8 * S;
  kp.hs_x0 = 0;
  kp.hs_y0 = 0;
  for (int r = 0; r < 3; ++r) kp.hs_tap_off[r] = r * 8 * S;
  for (int r = 0; r < 3; ++r) kp.hs_tap_desc[r] = (kp.hs_tap_off[r] * 32) >> 4;
  kp.BN = BN;
  kp.n_ntiles = 1;
  kp.halo_bytes = 16u * 3u * (uint32_t)(8 * S) * 32u;
  kp.hs_a_row_bytes = 32u;
  // Raw-pixel operand (default; PADEL_B200_STEM_RAW=0 selects the overlapping-row box above): the tile's input region --
  // 34 rows x (16 S + 2) pixels of 8 bytes, every byte once -- is one dense TMA box, and the wgmma descriptor reads the
  // im2col rows out of it: output pixel ow's K = 16 row (pixels 2ow .. 2ow+3) starts 16 bytes after its neighbour's, so
  // in the un-swizzled K-major layout (16-byte rows at a 16-byte pitch, second half of a row LBO = 16 bytes on) the
  // overlapping rows ARE the canonical core matrix; the next output row is two image rows further (SBO), filter row r
  // one image row (descriptor offset).  A third of the L2->SM traffic and of the shared memory of the box-per-row form.
  const uint32_t pairs = (uint32_t)(8 * S) + 1;  // pixel pairs (16 bytes) per image row of the region
  const uint32_t pitch = pairs * 16u;
  static const int raw = [] {
    const char* e = getenv("PADEL_B200_STEM_RAW");
    return e ? atoi(e) : 1;
  }();
  if (raw) {
    kp.halo_bytes = 17u * 2u * pitch;  // 17 row pairs (2 * 16 + 1 rows are read, the 34th is never addressed)
    kp.hs_a_row_bytes = 16u;
    kp.hs_sbo_rows = (int)(2u * pitch / 16u);  // x hs_a_row_bytes = 2 image rows
    for (int r = 0; r < 3; ++r) kp.hs_tap_desc[r] = (int)(((uint32_t)r * pitch) >> 4);
  }
  kp.a_bytes = (kp.halo_bytes + 1023u) & ~1023u;
  kp.b_tx_bytes = 3u * (uint32_t)BN * 32u;
  kp.b_bytes = (kp.b_tx_bytes + 1023u) & ~1023u;
  kp.a_stages = 4;
  kp.b_stages = 1;  // the three filter rows are one small box: resident
  kp.b_resident = 1;
  kp.tiles_w = (kp.Wo + 8 * S - 1) / (8 * S);
  kp.tiles_h = (kp.Ho + 15) / 16;
  kp.tiles_n = kp.N;
  kp.total_tiles = kp.tiles_w * kp.tiles_h * kp.tiles_n;
  if (halo_plan_store(d, plan, encode) != 0) return 1;
  halo_finish_config(plan);
  plan->variant = 1;
  {
    // overlapping-row view of the padded (N, H+2, W+2, 4) tensor: element (k, ow, r, oh, n) =
    //   base + n*(H+2)*(W+2)*8 + (2*oh + r)*(W+2)*8 + (2*ow)*8 + 2*k  -> pixels 2ow-1 .. 2ow+2 of image row 2oh+r-1
    const cuuint64_t Wp = (cuuint64_t)d->W + 2, Hp = (cuuint64_t)d->H + 2;
    cuuint64_t dims[5] = {16, (cuuint64_t)d->W / 2, 3, (cuuint64_t)d->H / 2, (cuuint64_t)d->N};
    cuuint64_t strides[4] = {16, Wp * 8, 2 * Wp * 8, Hp * Wp * 8};
    cuuint32_t box[5] = {16, (cuuint32_t)(8 * S), 3, 16, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_32B;
    if (raw) {
      // dense view (pixel pair, image-row parity, image-row pair): element (k, p, q, y, n) =
      //   base + n*Hp*Wp*8 + (2*y + q)*Wp*8 + p*16 + 2*k; the producer's coordinates (0, ow0, 0, oh0, n) address
      //   pixel pair ow0 = pixel 2*ow0 and image row 2*oh0 of the padded tensor, i.e. the tile's top-left tap
      dims[0] = 8, dims[1] = Wp / 2, dims[2] = 2, dims[3] = Hp / 2;
      strides[0] = 16, strides[1] = Wp * 8, strides[2] = 2 * Wp * 8;
      box[0] = 8, box[1] = pairs, box[2] = 2, box[3] = 17;
      swz = CU_TENSOR_MAP_SWIZZLE_NONE;
    }
    CUresult r = encode(&plan->tmap_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(d->in), dims, strides,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(stem): cuTensorMapEncodeTiled(A, overlapping rows) failed with %d", (int)r);
  }
  {
    cuuint64_t dims[3] = {16, (cuuint64_t)d->cout_pad, 3};
    cuuint64_t strides[2] = {32, (cuuint64_t)d->cout_pad * 32};
    cuuint32_t box[3] = {16, (cuuint32_t)BN, 3};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&plan->tmap_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(d->weight), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(stem): cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  return 0;
}

// cout > 192 runs in N tiles of BN = 128 with streamed weights.  At S = 2 a CTA fetches one 18 x 18-pixel halo and
// 9 x 128 weight rows per channel block: ~0.010 bytes from L2 per MAC, against 0.023 for the per-tap kernel's
// 128 x 256 tiles and 0.017 for one S = 1, BN = 256 tile here.  S = 4 / BN = 64 would move fewer bytes still, but an
// m64n64k16 wgmma reads 4 KB of shared memory per 32 tensor clocks, the SM's whole 128 B/clk, which is why the
// 64-channel layers trail; BN stays at 128.  Without `force` such a layer is taken only when the 16 x 8S tiles compute
// at most 1.15x its output pixels (after the rows a warpgroup skips below the image): the per-tap kernel's flattened
// 128-pixel tiles waste nothing at the edges.  `force`: wherever the kernel can run the layer.
int conv_halo_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode, bool force) {
  if (d->ksize != 3 || d->stride != 1) return -1;
  const bool ntiled = d->cout_pad > 192 && d->cout_pad % kHaloNTileBN == 0 && d->head_n == 0;
  if (!ntiled && d->cout_pad > (force ? 256 : 192)) return -1;
  ConvKParams& kp = plan->kp;  // common fields (epilogue, KB, kblocks, ...) already filled by the caller
  const int BN = ntiled ? kHaloNTileBN : d->cout_pad;
  const uint32_t row_bytes = (uint32_t)kp.KB * 2u;
  const int acc_cols = (BN + 31) / 32 * 32;
  const size_t budget = kHaloSmemBudget;
  // Choose S (sub-tiles per CTA tile: fewer halo + weight bytes per pixel) first, then G (taps per weight box:
  // fewer TMA operations) as large as shared memory allows.
  const uint32_t tap_bytes = (uint32_t)BN * row_bytes;
  // Resident filter bank: all nine taps of every channel block (one box per block) stay in shared memory for the
  // whole kernel when they fit next to two halo buffers; otherwise weight boxes are streamed through a ring.
  // PADEL_B200_CONV_BRES=0 disables (A/B testing).
  const uint32_t res_box = (9u * tap_bytes + 1023u) & ~1023u;
  const size_t res_total = (size_t)kp.kblocks * res_box;
  bool resident = false;
  {
    const char* er = getenv("PADEL_B200_CONV_BRES");
    resident = (!er || atoi(er) != 0) && !ntiled && kp.kblocks <= kHaloMaxB && res_total <= 120 * 1024;
  }
  int bestS = 0, best_cols = 0, G = 1;
  for (int pass = resident ? 0 : 1; pass < 2 && bestS == 0; ++pass) {
    resident = resident && pass == 0;
    for (int S = 4; S >= 1; S >>= 1) {
      if (S * acc_cols > 2 * kConvAccRegs) continue;  // accumulators of S sub-tiles fit the registers
      const uint32_t halo = 18u * (uint32_t)(8 * S + 2) * row_bytes;
      const uint32_t a_alloc = (halo + 1023u) & ~1023u;
      int g_fit = 0;
      if (resident) {
        if ((size_t)2 * a_alloc + res_total <= budget) g_fit = 9;
      } else {
        for (int g = 9; g >= 1; g = (g == 9 ? 3 : (g == 3 ? 1 : 0))) {
          const uint32_t ba = ((uint32_t)g * tap_bytes + 1023u) & ~1023u;
          const int min_b = g == 9 ? 2 : (g == 3 ? 3 : 4);
          if ((size_t)2 * a_alloc + (size_t)min_b * ba <= budget) {
            g_fit = g;
            break;
          }
        }
      }
      if (!g_fit) continue;
      const int cols = (d->W + 8 * S - 1) / (8 * S) * 8 * S;  // padded width actually computed
      // resident: prefer the largest S that fits (less halo overlap); streaming: the least padding
      if (bestS == 0 || (!resident && cols < best_cols)) {
        bestS = S;
        best_cols = cols;
        G = g_fit;
      }
    }
  }
  const uint32_t b_alloc = ((uint32_t)G * tap_bytes + 1023u) & ~1023u;
  if (bestS == 0) return -1;
  const int S = bestS, P = 8 * S + 2;
  if (ntiled && !force) {
    const long computed = (long)best_cols * ((kp.Ho + 7) / 8 * 8);
    if (20 * computed > 23 * (long)kp.Wo * kp.Ho) return -1;
  }
  kp.b_resident = resident ? 1 : 0;
  kp.hs_S = S;
  kp.hs_P = P;
  kp.hs_G = G;
  kp.hs_ntaps = 9;
  kp.hs_sbo_rows = P;
  kp.hs_x0 = -1;
  kp.hs_y0 = -1;
  for (int r = 0; r < 3; ++r)
    for (int q = 0; q < 3; ++q) {
      kp.hs_tap_off[r * 3 + q] = r * P + q;
      kp.hs_tap_desc[r * 3 + q] = (int)(((uint32_t)(r * P + q) * row_bytes) >> 4);
    }
  kp.BN = BN;
  kp.n_ntiles = d->cout_pad / BN;
  kp.halo_bytes = 18u * (uint32_t)P * row_bytes;
  kp.hs_a_row_bytes = row_bytes;
  kp.a_bytes = (kp.halo_bytes + 1023u) & ~1023u;
  kp.b_tx_bytes = (uint32_t)G * tap_bytes;
  kp.b_bytes = b_alloc;
  kp.a_stages = 2;
  if (resident) {
    // the filter bank occupies kblocks fixed slots; whatever is left goes to halo buffers (up to kHaloMaxA)
    kp.b_stages = kp.kblocks;
    int as = (int)((budget - res_total) / kp.a_bytes);
    if (as > kHaloMaxA) as = kHaloMaxA;
    if (as > 2 * kp.kblocks + 1) as = 2 * kp.kblocks + 1;
    kp.a_stages = as < 2 ? 2 : as;
  } else {
    size_t rest = budget - (size_t)2 * kp.a_bytes;
    if (kp.kblocks > 2 && rest > (size_t)kp.a_bytes + 4 * (size_t)b_alloc) {  // a third halo buffer when K is deep
      kp.a_stages = 3;
      rest -= kp.a_bytes;
    }
    int bs = (int)(rest / b_alloc);
    if (bs > kHaloMaxB) bs = kHaloMaxB;
    if (bs > 9 * kp.kblocks / G * 2) bs = 9 * kp.kblocks / G * 2;
    if (bs < 2) bs = 2;
    kp.b_stages = bs;
  }
  kp.tiles_w = (kp.Wo + 8 * S - 1) / (8 * S);
  kp.tiles_h = (kp.Ho + 15) / 16;
  kp.tiles_n = kp.N;
  kp.total_tiles = kp.tiles_w * kp.tiles_h * kp.tiles_n * kp.n_ntiles;
  if (halo_plan_store(d, plan, encode) != 0) return 1;
  halo_finish_config(plan);
  plan->variant = 1;

  const CUtensorMapSwizzle swz = kp.KB == 64   ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : kp.KB == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                               : CU_TENSOR_MAP_SWIZZLE_32B;
  {
    const cuuint64_t C = (cuuint64_t)d->C, W = (cuuint64_t)d->W, H = (cuuint64_t)d->H;
    cuuint64_t dims[5] = {C, W, 1, H, (cuuint64_t)d->N};
    cuuint64_t strides[4] = {C * 2, W * C * 2, W * C * 2, H * W * C * 2};
    cuuint32_t box[5] = {(cuuint32_t)kp.KB, (cuuint32_t)P, 1, 18, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = encode(&plan->tmap_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(d->in), dims, strides,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(halo): cuTensorMapEncodeTiled(A) failed with %d", (int)r);
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)d->cin, (cuuint64_t)d->cout_pad, 9};
    cuuint64_t strides[2] = {(cuuint64_t)d->cin * 2, (cuuint64_t)d->cin * d->cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)kp.KB, (cuuint32_t)BN, (cuuint32_t)G};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&plan->tmap_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(d->weight), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(halo): cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  return 0;
}

// 1x1 / stride-1 layers through the same kernel (one tap, no halo): a CTA tile is 16 rows x 8S columns (up to 512
// pixels, S accumulator sets) instead of the per-tap kernel's 128, and the whole filter bank (cin x cout, one box per
// channel block) is fetched ONCE per CTA and stays in shared memory -- the per-tap kernel re-reads it from L2 for every
// 128-pixel tile, as many bytes as the activations when cin ~ cout, and pays its fixed per-tile costs four times as
// often.  That pays off for the narrow layers of the pose program (cin 32 -> 32 @320^2); wider layers stay on the
// per-tap kernel, whose flattened 128-pixel tiles waste nothing at the image edges and whose K loop is deeper.  Default rule therefore: cin <= 32; PADEL_B200_CONV_HALO1=0 disables it, =2
// takes every 1x1 layer whose bank fits next to two activation buffers.
int conv_halo_1x1_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode) {
  static const int enabled = [] {
    const char* e = getenv("PADEL_B200_CONV_HALO1");
    return e ? atoi(e) : 1;
  }();
  if (!enabled || d->ksize != 1 || d->stride != 1 || d->cout_pad > 256 || d->head_n != 0) return -1;
  if (enabled == 1 && d->cin > 32) return -1;
  // fp32 outputs (YOLO head maps, the TrackNet predictor) keep the per-tap kernel and its fp32 epilogue class
  if (d->out_mode != PB_OUT_F16_NHWC && d->out_mode != PB_OUT_F16_NHWC_UP2) return -1;
  ConvKParams& kp = plan->kp;  // common fields already filled by the caller
  const int BN = d->cout_pad;
  const uint32_t row_bytes = (uint32_t)kp.KB * 2u;
  const int acc_cols = (BN + 31) / 32 * 32;
  const size_t budget = kHaloSmemBudget;
  const uint32_t tap_bytes = (uint32_t)BN * row_bytes;
  const uint32_t res_box = (tap_bytes + 1023u) & ~1023u;
  const size_t res_total = (size_t)kp.kblocks * res_box;
  if (kp.kblocks > kHaloMaxB || res_total > 120 * 1024) return -1;
  int S = 0;
  for (int s = 4; s >= 1; s >>= 1) {
    if (s * acc_cols > 2 * kConvAccRegs) continue;  // accumulators of S sub-tiles fit the registers
    const uint32_t a_alloc = (16u * (uint32_t)(8 * s) * row_bytes + 1023u) & ~1023u;
    if ((size_t)2 * a_alloc + res_total > budget) continue;
    if (s > 1 && d->W <= 8 * (s / 2)) continue;  // a narrower tile already covers the row
    S = s;
    break;
  }
  if (S == 0) return -1;
  const int P = 8 * S;
  kp.b_resident = 1;
  kp.hs_S = S;
  kp.hs_P = P;
  kp.hs_G = 1;
  kp.hs_ntaps = 1;
  kp.hs_sbo_rows = P;
  kp.hs_x0 = 0;
  kp.hs_y0 = 0;
  kp.hs_tap_off[0] = 0;
  kp.hs_tap_desc[0] = 0;
  kp.BN = BN;
  kp.n_ntiles = 1;
  kp.halo_bytes = 16u * (uint32_t)P * row_bytes;
  kp.hs_a_row_bytes = row_bytes;
  kp.a_bytes = (kp.halo_bytes + 1023u) & ~1023u;
  kp.b_tx_bytes = tap_bytes;
  kp.b_bytes = res_box;
  kp.b_stages = kp.kblocks;
  {
    int as = (int)((budget - res_total) / kp.a_bytes);
    if (as > kHaloMaxA) as = kHaloMaxA;
    if (as > 2 * kp.kblocks + 1) as = 2 * kp.kblocks + 1;
    kp.a_stages = as < 2 ? 2 : as;
  }
  kp.tiles_w = (kp.Wo + 8 * S - 1) / (8 * S);
  kp.tiles_h = (kp.Ho + 15) / 16;
  kp.tiles_n = kp.N;
  kp.total_tiles = kp.tiles_w * kp.tiles_h * kp.tiles_n;
  if (halo_plan_store(d, plan, encode) != 0) return 1;
  halo_finish_config(plan);
  plan->variant = 1;
  const CUtensorMapSwizzle swz = kp.KB == 64   ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : kp.KB == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                               : CU_TENSOR_MAP_SWIZZLE_32B;
  {
    const cuuint64_t C = (cuuint64_t)d->C, W = (cuuint64_t)d->W, H = (cuuint64_t)d->H;
    cuuint64_t dims[5] = {C, W, 1, H, (cuuint64_t)d->N};
    cuuint64_t strides[4] = {C * 2, W * C * 2, W * C * 2, H * W * C * 2};
    cuuint32_t box[5] = {(cuuint32_t)kp.KB, (cuuint32_t)P, 1, 16, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = encode(&plan->tmap_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(d->in), dims, strides,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(halo 1x1): cuTensorMapEncodeTiled(A) failed with %d", (int)r);
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)d->cin, (cuuint64_t)d->cout_pad, 1};
    cuuint64_t strides[2] = {(cuuint64_t)d->cin * 2, (cuuint64_t)d->cin * d->cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)kp.KB, (cuuint32_t)BN, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&plan->tmap_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(d->weight), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(halo 1x1): cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  return 0;
}

// 3x3 / stride-2 conv over a whole C = 16 / 32 channel tensor.  The input is read through the pixel-pair view
// (2C, W/2, 2, H/2, N) -- element (k, w2, ph, h2, n) = channel k % C of pixel (2*h2 + ph, 2*w2 + k / C) -- so one TMA
// box (2C, 8S+1, 2, 17, 1) holds everything a 16 x 8S output tile needs, as rows of one PIXEL PAIR (4C bytes):
//   smem row = ((h2i * 2 + ph) * P + w2i),  P = 8S + 1,  box origin (w2, h2) = (ow0 - 1, oh0 - 1).
// Tap (r, s) of output (ohi, owi) reads input (2*oh + r - 1, 2*ow + s - 1):
//   r = 0 -> (h2i, ph) = (ohi, 1)      r = 1 -> (ohi + 1, 0)      r = 2 -> (ohi + 1, 1)
//   s = 0 -> (w2i, half) = (owi, 1)    s = 1 -> (owi + 1, 0)      s = 2 -> (owi + 1, 1)
// i.e. again only a descriptor start offset (row offset * 4C + half * 2C bytes) with SBO = 2P rows, and K = C per tap
// (the 32-byte k-step advance inside the swizzle row is the usual one).  Versus nine per-tap boxes of 2C-byte rows
// this issues one TMA per tile with rows twice as long (TMA delivery of 32-byte rows is what bounds the per-tap path).
int conv_halo_s2_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode) {
  if (d->ksize != 3 || d->stride != 2 || d->cout_pad > 256 || d->c_in_off != 0 || d->C != d->cin ||
      (d->cin != 16 && d->cin != 32))
    return -1;
  ConvKParams& kp = plan->kp;  // common fields already filled by the caller (KB = cin, kblocks = 1)
  const int BN = d->cout_pad;
  const uint32_t row_bytes = (uint32_t)d->cin * 2u;  // weight rows
  const uint32_t a_row = 2u * row_bytes;             // pixel-pair rows
  const int acc_cols = (BN + 31) / 32 * 32;
  const uint32_t tap_bytes = (uint32_t)BN * row_bytes;
  const uint32_t b_alloc = (9u * tap_bytes + 1023u) & ~1023u;  // all nine taps in one weight box
  const size_t budget = kHaloSmemBudget;
  int S = 0;
  for (int s = 4; s >= 1; s >>= 1) {
    if (s * acc_cols > 2 * kConvAccRegs) continue;
    const uint32_t halo = 34u * (uint32_t)(8 * s + 1) * a_row;
    if ((size_t)2 * ((halo + 1023u) & ~1023u) + (size_t)2 * b_alloc <= budget) {
      S = s;
      break;
    }
  }
  if (S == 0) return -1;
  const int P = 8 * S + 1;
  kp.KB = d->cin;
  kp.kblocks = 1;
  kp.hs_S = S;
  kp.hs_P = P;
  kp.hs_G = 9;
  kp.hs_ntaps = 9;
  kp.hs_sbo_rows = 2 * P;
  kp.hs_x0 = -1;
  kp.hs_y0 = -1;
  kp.hs_a_row_bytes = a_row;
  for (int r = 0; r < 3; ++r)
    for (int q = 0; q < 3; ++q) {
      const int row = ((r == 0 ? 0 : 1) * 2 + (r == 1 ? 0 : 1)) * P + (q == 0 ? 0 : 1);
      const int half = q == 1 ? 0 : 1;
      kp.hs_tap_off[r * 3 + q] = row;
      kp.hs_tap_desc[r * 3 + q] = (int)(((uint32_t)row * a_row + (uint32_t)half * row_bytes) >> 4);
    }
  kp.BN = BN;
  kp.n_ntiles = 1;
  kp.halo_bytes = 34u * (uint32_t)P * a_row;
  kp.a_bytes = (kp.halo_bytes + 1023u) & ~1023u;
  kp.b_tx_bytes = 9u * tap_bytes;
  kp.b_bytes = b_alloc;
  kp.a_stages = 2;
  kp.b_stages = 1;  // all nine taps are one box: resident
  kp.b_resident = 1;
  kp.tiles_w = (kp.Wo + 8 * S - 1) / (8 * S);
  kp.tiles_h = (kp.Ho + 15) / 16;
  kp.tiles_n = kp.N;
  kp.total_tiles = kp.tiles_w * kp.tiles_h * kp.tiles_n;
  if (halo_plan_store(d, plan, encode) != 0) return 1;
  halo_finish_config(plan);
  plan->variant = 1;
  {
    const cuuint64_t C = (cuuint64_t)d->C, W = (cuuint64_t)d->W, H = (cuuint64_t)d->H;
    cuuint64_t dims[5] = {2 * C, W / 2, 2, H / 2, (cuuint64_t)d->N};
    cuuint64_t strides[4] = {2 * C * 2, W * C * 2, 2 * W * C * 2, H * W * C * 2};
    cuuint32_t box[5] = {(cuuint32_t)(2 * d->C), (cuuint32_t)P, 2, 17, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = encode(&plan->tmap_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(d->in), dims, strides,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        a_row == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(halo s2): cuTensorMapEncodeTiled(A) failed with %d", (int)r);
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)d->cin, (cuuint64_t)d->cout_pad, 9};
    cuuint64_t strides[2] = {(cuuint64_t)d->cin * 2, (cuuint64_t)d->cin * d->cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)d->cin, (cuuint32_t)BN, 9};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&plan->tmap_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(d->weight), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv(halo s2): cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  return 0;
}

static HaloKernelFn halo_kernel_pick(const ConvPlan* plan) {
  const ConvKParams& kp = plan->kp;
  const int S = kp.hs_S, steps = kp.KB / 16, BN = kp.BN;
  if (plan->epi == PB_EPI_SILU) return halo_kernel_lookup<PB_EPI_SILU>(S, steps, BN);
  if (plan->epi == PB_EPI_RELU) return halo_kernel_lookup<PB_EPI_RELU>(S, steps, BN);
  if (plan->epi == PB_EPI_SILU_RES) return halo_kernel_lookup<PB_EPI_SILU_RES>(S, steps, BN);
  return halo_kernel_lookup<PB_EPI_GENERIC>(S, steps, BN);
}

int conv_halo_launch(const ConvPlan* plan, cudaStream_t stream) {
  const ConvKParams& kp = plan->kp;
  const int tma_store = kp.st_bytes != 0;
  HaloKernelFn fn = halo_kernel_pick(plan);
  PB_CHECK(fn != nullptr,
           "conv(halo): no kernel instantiation for S=%d, k-steps=%d, N=%d, epilogue class %d (TMA store %d)", kp.hs_S,
           kp.KB / 16, kp.BN, plan->epi, tma_store);
  PB_CUDA((cudaError_t)ensure_dynamic_smem(reinterpret_cast<const void*>(fn), 227 * 1024));
  cudaError_t le = launch_ex(fn, dim3(plan->grid), dim3(plan->threads), plan->smem_bytes, stream, 1, plan->pdl != 0,
                             plan->tmap_a, plan->tmap_w, plan->kp, plan->tmap_o);
  PB_CHECK(le == cudaSuccess,
           "conv(halo): launch failed: %s (grid %d, threads %d, smem %zu, tiles %d, S %d, k-steps %d, N %d, epilogue "
           "class %d, TMA store %d)",
           cudaGetErrorString(le), plan->grid, plan->threads, plan->smem_bytes, kp.total_tiles, kp.hs_S, kp.KB / 16,
           kp.BN, plan->epi, tma_store);
  count_launch();
  return 0;
}

}  // namespace pb
