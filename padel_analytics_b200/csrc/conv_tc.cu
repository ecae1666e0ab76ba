// Fused conv(k1|k3, s1|s2) + bias + activation (+ residual) as an implicit GEMM on Hopper tensor cores (wgmma).
//
//   D[M = 128 output pixels, N = BN out-channels] += A[M, K] * B[N, K]^T,   K = taps x input channels
//
// * A (activations, NHWC fp16) is fetched by TMA in tiled mode: one box = a (TN x TH x TW) patch of pixels x KB
//   channels, shifted by the filter tap; out-of-bounds coordinates are zero-filled by TMA, which implements the
//   conv zero padding for free.  Stride-2 convs read a 5-D view (N, H/2, 2, W/2, 2C) of the same tensor so every
//   tap is again a dense box.  The box lands in shared memory directly in the wgmma K-major swizzled layout
//   (one pixel = one KB*2-byte row; swizzle 32/64/128B == row size).
// * B (weights, fp16 [tap][cout][cin]) is fetched by TMA the same way.
// * warps 0 / 1 = TMA producers (activations / weights); warpgroups 1-2 = consumers, each issuing the wgmmas of 64
//   rows (register accumulators) and then storing them.  Persistent CTAs, static tile striding, fast-division decode.
//
// Replaces: ultralytics Conv/C2f/Bottleneck/Detect convs (3P, SURVEY App. A.2) and TrackNet Conv2DBlock
// (reference trackers/ball_tracker/models.py:5-17) with BN folded into weight/bias.
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "internal.h"
#include "ptx.cuh"
#include "conv_common.cuh"

namespace pb {

// shared memory for the operand rings: what the 227 KB of an SM leaves beside the tail (bias, barriers, epilogue
// scratch) and the alignment slack
constexpr size_t kConvStageBudget = 196 * 1024;

struct ConvSmemTail {
  uint64_t full[kConvMaxStages];
  uint64_t empty[kConvMaxStages];
  float bias[kConvMaxCout];  // staged once per CTA
  float scratch[kConvConsumerWarps * kEpiScratchFloats];  // epilogue transposition, one slice per consumer warp
};

struct TileCoord {
  int nt, tw, th, tn;
};
__device__ __forceinline__ TileCoord decode_tile(const ConvKParams& kp, int tile) {
  TileCoord c;
  int t;
  fast_divmod(t, c.nt, tile, kp.fd_nt);
  fast_divmod(t, c.tw, t, kp.fd_w);
  fast_divmod(c.tn, c.th, t, kp.fd_h);
  return c;
}

template <int kEpi>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
               const __grid_constant__ ConvKParams kp) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024B alignment is required by the 128B swizzle pattern; align explicitly (the launch adds 1 KB of slack).
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t stage_bytes = kp.a_bytes + kp.b_bytes;
  ConvSmemTail* tail = reinterpret_cast<ConvSmemTail*>(smem + (size_t)kp.stages * stage_bytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int k_iters = kp.taps * kp.kblocks;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    for (int i = 0; i < kp.stages; ++i) {
      mbar_init(&tail->full[i], 2);  // A producer + B producer (each arrives with its expected bytes)
      mbar_init(&tail->empty[i], kConvConsumerWarps);
    }
    fence_mbar_init();
  }
  if (warp == 1 && lane == 0) tma_prefetch_desc(&tmap_w);
  for (int i = threadIdx.x; i < kp.cout_pad; i += blockDim.x) tail->bias[i] = kp.bias[i];
  __syncthreads();
  // PDL: the prologue above touched constant data only; from here on activations are read and written.  The weight
  // producer (warp 1) reads constants only and starts fetching while the previous kernel is still running.
  griddep_launch_dependents();
  if (warp != 1) griddep_wait();

  if (warp < 4) {
    warpgroup_reg_dealloc<kConvProducerRegs>();
    if (warp == 0 && lane == 0) {
      // ============================== TMA producer: activations ==============================
      int stage = 0;
      uint32_t phase = 0;
      const int TW = 1 << kp.tw_log2, TH = 1 << kp.th_log2;
      const int TN = 128 >> (kp.tw_log2 + kp.th_log2);
      for (int tile = blockIdx.x; tile < kp.total_tiles; tile += gridDim.x) {
        const TileCoord tc = decode_tile(kp, tile);
        for (int tap = 0; tap < kp.taps; ++tap) {
          const int cw = tc.tw * TW + kp.tap_dw[tap];
          const int ch = tc.th * TH + kp.tap_dh[tap];
          const int cc = kp.c_in_off + kp.tap_dc[tap];
          for (int kb = 0; kb < kp.kblocks; ++kb) {
            mbar_wait(&tail->empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&tail->full[stage], kp.a_bytes);
            tma_load_5d(smem + (size_t)stage * stage_bytes, &tmap_a, &tail->full[stage], cc + kb * kp.KB, cw,
                        kp.tap_d2[tap], ch, tc.tn * TN);
            if (++stage == kp.stages) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    } else if (warp == 1 && lane == 0) {
      // ============================== TMA producer: weights (issued in parallel with warp 0) =================
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < kp.total_tiles; tile += gridDim.x) {
        int nt, tq;
        fast_divmod(tq, nt, tile, kp.fd_nt);
        for (int tap = 0; tap < kp.taps; ++tap) {
          for (int kb = 0; kb < kp.kblocks; ++kb) {
            mbar_wait(&tail->empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&tail->full[stage], kp.b_tx_bytes);
            tma_load_3d(smem + (size_t)stage * stage_bytes + kp.a_bytes, &tmap_w, &tail->full[stage], kb * kp.KB,
                        nt * kp.BN, tap);
            if (++stage == kp.stages) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
    return;
  }

  // ============================== consumers: wgmma + epilogue ==============================
  // warpgroup g computes rows 64g .. 64g + 63 of every 128-pixel tile; its warp wq holds rows 64g + 16wq .. +15.
  warpgroup_reg_alloc<kConvConsumerRegs>();
  const int cw = warp - 4, g = cw >> 2, wq = cw & 3;
  float* scr = tail->scratch + cw * kEpiScratchFloats;
  const uint32_t row_bytes = (uint32_t)kp.KB * 2u;
  const int ksteps = kp.KB / 16;
  const int p = 64 * g + 16 * wq + (lane & 15);  // this lane's row of the M = 128 tile in the epilogue
  const int TWm = (1 << kp.tw_log2) - 1, THm = (1 << kp.th_log2) - 1;
  const int tw_i = p & TWm;
  const int th_i = (p >> kp.tw_log2) & THm;
  const int tn_i = p >> (kp.tw_log2 + kp.th_log2);
  float acc[kConvAccRegs];
#pragma unroll
  for (int i = 0; i < kConvAccRegs; ++i) acc[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < kp.total_tiles; tile += gridDim.x) {
    const TileCoord tc = decode_tile(kp, tile);
    int prev = -1;
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait(&tail->full[stage], phase);
      const uint32_t a_addr = smem_u32(smem + (size_t)stage * stage_bytes) + 64u * (uint32_t)g * row_bytes;
      const uint64_t adesc = wgmma_desc_kmajor(a_addr, row_bytes);
      const uint64_t bdesc = wgmma_desc_kmajor(smem_u32(smem + (size_t)stage * stage_bytes + kp.a_bytes), row_bytes);
      wgmma_fence();
      for (int k = 0; k < ksteps; ++k)  // advance 16 K-elements = 32 bytes inside the swizzle row: +2 in (addr >> 4)
        mma_group<1, 1>(kp.BN, acc, adesc + (uint64_t)(2 * k), 0, bdesc + (uint64_t)(2 * k), (uint32_t)((it | k) != 0));
      wgmma_commit();
      if (prev >= 0) {  // keep one stage of wgmmas in flight; the one before it has retired
        wgmma_wait<1>();
        consumer_release(&tail->empty[prev], lane);
      }
      prev = stage;
      if (++stage == kp.stages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    consumer_release(&tail->empty[prev], lane);

    EpiPix px;
    px.ow = (tc.tw << kp.tw_log2) + tw_i;
    px.oh = (tc.th << kp.th_log2) + th_i;
    px.n = tc.tn * (128 >> (kp.tw_log2 + kp.th_log2)) + tn_i;
    px.valid = (px.ow < kp.Wo) && (px.oh < kp.Ho) && (px.n < kp.N);
    px.pix = ((size_t)px.n * kp.Ho + px.oh) * kp.Wo + px.ow;
    epilogue_tile<kEpi>(kp, acc, 1, tc.nt, tail->bias + tc.nt * kp.BN, scr, lane, [&](int, bool& pool_writer) {
      pool_writer = false;  // pool windows do not map onto this tiling (halo kernel only)
      return px;
    });
  }
}

// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

// Which epilogue instantiation a layer runs: a plain class when the vectorised epilogue applies (the conditions of
// epilogue_fast_ok) and the layer is activation-only -- no residual, fp16 NHWC store, no secondary output, no fused head.
// PADEL_B200_CONV_EPI=0 keeps every layer on the run-time epilogue (A/B).
int conv_epi_class(const pb_conv_desc* d, const ConvKParams& kp) {
  static const int enabled = [] {
    const char* e = getenv("PADEL_B200_CONV_EPI");
    return e ? atoi(e) : 1;
  }();
  if (!enabled || kp.dbg_flags != 0) return PB_EPI_GENERIC;
  if (d->head_n != 0 || d->out2_mode != PB_OUT2_NONE || (reinterpret_cast<uintptr_t>(d->out) & 31) != 0)
    return PB_EPI_GENERIC;
  if (d->out_mode == PB_OUT_F32_NHWC) {  // 32-byte aligned 8-float groups
    return (!d->res && d->act == PB_ACT_NONE && ((d->out_C | d->out_coff) & 7) == 0 && d->ksize == 1) ? PB_EPI_F32
                                                                                                       : PB_EPI_GENERIC;
  }
  if (d->out_mode != PB_OUT_F16_NHWC || ((d->out_C | d->out_coff | d->cout_store) & 15) != 0) return PB_EPI_GENERIC;
  if (d->res) {
    const bool ok = !d->res_before_act && d->act == PB_ACT_SILU && ((d->res_C | d->res_coff) & 7) == 0;
    return ok ? PB_EPI_SILU_RES : PB_EPI_GENERIC;
  }
  return d->act == PB_ACT_SILU ? PB_EPI_SILU : (d->act == PB_ACT_RELU ? PB_EPI_RELU : PB_EPI_GENERIC);
}

static int conv_plan_build_impl(const pb_conv_desc* d, ConvPlan* plan) {
  PB_CHECK(d && plan, "conv: null argument");
  PB_CHECK(d->in_layout == PB_IN_NHWC || d->in_layout == PB_IN_STEM4, "conv: bad in_layout");
  const bool stem = d->in_layout == PB_IN_STEM4;
  PB_CHECK(d->ksize == 1 || d->ksize == 3, "conv: ksize %d unsupported", d->ksize);
  PB_CHECK(d->stride == 1 || d->stride == 2, "conv: stride %d unsupported", d->stride);
  PB_CHECK(d->cin > 0 && d->cin % 16 == 0, "conv: cin %d must be a positive multiple of 16", d->cin);
  PB_CHECK(d->cout_pad <= kConvMaxCout, "conv: cout_pad %d > %d", d->cout_pad, kConvMaxCout);
  PB_CHECK(d->cout_pad > 0 && d->cout_pad % 16 == 0, "conv: cout_pad %d must be a multiple of 16", d->cout_pad);
  PB_CHECK(stem || (d->C % 8 == 0 && d->c_in_off >= 0 && d->c_in_off + d->cin <= d->C),
           "conv: bad input channel slice");
  PB_CHECK(d->c_in_off % 8 == 0, "conv: c_in_off must be a multiple of 8");
  PB_CHECK((reinterpret_cast<uintptr_t>(d->in) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->weight) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(d->bias) & 15) == 0 &&
               (d->out_mode == PB_OUT_NONE || (reinterpret_cast<uintptr_t>(d->out) & 15) == 0),
           "conv: pointers must be 16-byte aligned");
  PB_CHECK(d->stride == 1 || (d->H % 2 == 0 && d->W % 2 == 0), "conv: stride 2 needs even H and W");
  PB_CHECK(d->cout_store > 0 && d->cout_store <= d->cout_pad, "conv: bad cout_store");
  PB_CHECK(d->out_mode >= PB_OUT_F16_NHWC && d->out_mode <= PB_OUT_NONE, "conv: bad out_mode");
  PB_CHECK(d->out_mode != PB_OUT_NONE || d->head_n > 0, "conv: PB_OUT_NONE needs a fused head");
  if (d->head_n > 0) {
    PB_CHECK(d->head_n <= 8 && d->head_weight && d->head_bias && d->head_out, "conv: bad fused head");
    PB_CHECK(d->cout_pad <= 256 && d->cout_store == d->cout_pad, "conv: fused head needs a single full N tile");
    PB_CHECK((reinterpret_cast<uintptr_t>(d->head_weight) & 15) == 0, "conv: head_weight must be 16-byte aligned");
  }
  const bool f16out = d->out_mode == PB_OUT_F16_NHWC || d->out_mode == PB_OUT_F16_NHWC_UP2;
  if (f16out) {
    PB_CHECK(d->cout_store % 8 == 0 && d->out_coff % 8 == 0 && d->out_C % 8 == 0,
             "conv: f16 output needs cout_store/out_coff/out_C multiples of 8");
    PB_CHECK(d->out_coff + d->cout_store <= d->out_C, "conv: output slice exceeds out_C");
  }
  if (d->res) {
    PB_CHECK(d->res_C % 8 == 0 && d->res_coff % 8 == 0 && (reinterpret_cast<uintptr_t>(d->res) & 15) == 0,
             "conv: residual must be 16-byte aligned slices");
  }
  PB_CHECK(d->out2_mode >= PB_OUT2_NONE && d->out2_mode <= PB_OUT2_POOL2, "conv: bad out2_mode");
  if (d->out2_mode != PB_OUT2_NONE) {
    // the secondary store lives in the vectorised epilogue only: 32-byte channel groups on both outputs
    PB_CHECK(d->out_mode == PB_OUT_F16_NHWC && d->head_n == 0 && !stem, "conv: out2 needs a plain f16 NHWC primary output");
    PB_CHECK(d->out2 && (reinterpret_cast<uintptr_t>(d->out2) & 31) == 0 && (reinterpret_cast<uintptr_t>(d->out) & 31) == 0,
             "conv: out2 pointers must be 32-byte aligned");
    PB_CHECK(d->cout_store % 16 == 0 && d->out_C % 16 == 0 && d->out_coff % 16 == 0 && d->out2_C % 16 == 0 &&
                 d->out2_coff % 16 == 0 && d->out2_coff >= 0 && d->out2_coff + d->cout_store <= d->out2_C,
             "conv: out2 needs 16-channel aligned slices");
    if (d->out2_mode == PB_OUT2_POOL2)
      PB_CHECK(d->ksize == 3 && d->stride == 1 && d->H % 2 == 0 && d->W % 2 == 0,
               "conv: PB_OUT2_POOL2 needs a 3x3 stride-1 conv on even H, W");
  }
  EncodeTiledFn encode = get_encode_fn();
  PB_CHECK(encode != nullptr, "conv: cuTensorMapEncodeTiled not available (no CUDA driver?)");

  plan->desc = *d;
  ConvKParams& kp = plan->kp;
  memset(&kp, 0, sizeof(kp));
  kp.cout_pad = d->cout_pad;
  const int s = d->stride;
  kp.N = d->N;
  kp.Ho = d->H / s;
  kp.Wo = d->W / s;
  kp.taps = d->ksize * d->ksize;
  kp.KB = (d->cin % 64 == 0) ? 64 : (d->cin % 32 == 0 ? 32 : 16);
  kp.kblocks = d->cin / kp.KB;
  kp.c_in_off = d->c_in_off;
  kp.bias = d->bias;
  kp.act = d->act;
  kp.res = reinterpret_cast<const __half*>(d->res);
  kp.res_C = d->res_C;
  kp.res_coff = d->res_coff;
  kp.res_first = d->res_before_act ? 1 : 0;
  kp.out = d->out;
  kp.out_C = d->out_C;
  kp.out_coff = d->out_coff;
  kp.out_mode = d->out_mode;
  kp.cout_store = d->cout_store;
  kp.out2 = d->out2;
  kp.out2_C = d->out2_C;
  kp.out2_coff = d->out2_coff;
  kp.out2_mode = d->out2_mode;
  kp.head_w = d->head_weight;
  kp.head_b = d->head_bias;
  kp.head_n = d->head_n;
  kp.head_out = d->head_out;
  {
    const char* df = getenv("PADEL_B200_CONV_DEBUG");
    kp.dbg_flags = df ? atoi(df) : 0;
  }
  plan->variant = 0;
  plan->pdl = plan_pdl();
  plan->epi = conv_epi_class(d, kp);
  if (stem) return conv_stem_setup(d, plan, encode);
  {
    // halo variant: default on for cout <= 192 (the layers the per-tap kernel leaves L2/TMA-bound) and for the 3x3 / s1
    // layers conv_halo_setup runs in N tiles with little edge waste; PADEL_B200_CONV_HALO=0 disables it, =1 forces it
    // wherever it applies.  PB_OUT2_POOL2 exists in the halo kernel only, so such a layer takes it wherever it can.
    const char* e = getenv("PADEL_B200_CONV_HALO");
    const int mode = e ? atoi(e) : 2;
    const bool s1_3x3 = d->ksize == 3 && d->stride == 1;
    if (mode == 1 || (mode == 2 && (d->cout_pad <= 192 || s1_3x3))) {
      const int rc = d->ksize == 1    ? conv_halo_1x1_setup(d, plan, encode)
                     : d->stride == 2 ? conv_halo_s2_setup(d, plan, encode)
                                      : conv_halo_setup(d, plan, encode, mode == 1 || d->out2_mode == PB_OUT2_POOL2);
      if (rc >= 0) return rc;
    }
  }
  PB_CHECK(d->out2_mode != PB_OUT2_POOL2,
           "conv: PB_OUT2_POOL2 is only implemented by the halo kernel (3x3 stride 1, cout <= 256 or a multiple of 128)");
  // N tile: largest multiple-of-16 divisor of cout_pad that is <= 256
  int nn = (d->cout_pad + 255) / 256;
  while (d->cout_pad % nn != 0 || (d->cout_pad / nn) % 16 != 0) ++nn;
  kp.n_ntiles = nn;
  kp.BN = d->cout_pad / nn;
  PB_CHECK(kp.BN >= 16 && kp.BN <= 256, "conv: cannot tile cout_pad %d", d->cout_pad);

  // pixel tile shape (TN x TH x TW = 128): minimise the number of tiles, prefer wide tiles
  long best_cost = -1;
  int best_tw = 0, best_th = 0;
  for (int twl = 7; twl >= 2; --twl) {
    for (int thl = 7 - twl; thl >= 0; --thl) {
      const int TW = 1 << twl, TH = 1 << thl, TN = 128 >> (twl + thl);
      const long cost = (long)((kp.Wo + TW - 1) / TW) * ((kp.Ho + TH - 1) / TH) * ((kp.N + TN - 1) / TN);
      if (best_cost < 0 || cost < best_cost) {
        best_cost = cost;
        best_tw = twl;
        best_th = thl;
      }
    }
  }
  kp.tw_log2 = best_tw;
  kp.th_log2 = best_th;
  const int TW = 1 << best_tw, TH = 1 << best_th, TN = 128 >> (best_tw + best_th);
  kp.tiles_w = (kp.Wo + TW - 1) / TW;
  kp.tiles_h = (kp.Ho + TH - 1) / TH;
  kp.tiles_n = (kp.N + TN - 1) / TN;
  kp.total_tiles = kp.tiles_w * kp.tiles_h * kp.tiles_n * kp.n_ntiles;
  (void)ilog2;

  for (int r = 0; r < d->ksize; ++r)
    for (int q = 0; q < d->ksize; ++q) {
      const int t = r * d->ksize + q;
      const int dy = r - d->ksize / 2, dx = q - d->ksize / 2;  // input offset relative to s*o
      if (s == 1) {
        kp.tap_dc[t] = 0;
        kp.tap_dw[t] = dx;
        kp.tap_d2[t] = 0;
        kp.tap_dh[t] = dy;
      } else {
        // input col = 2*ow + dx  ->  (w/2 coord, parity): dx=-1 -> (ow-1, 1); 0 -> (ow, 0); 1 -> (ow, 1)
        kp.tap_dw[t] = (dx < 0) ? -1 : 0;
        kp.tap_dc[t] = (dx != 0) ? d->C : 0;
        kp.tap_dh[t] = (dy < 0) ? -1 : 0;
        kp.tap_d2[t] = (dy != 0) ? 1 : 0;
      }
    }
  kp.a_bytes = 128u * kp.KB * 2u;
  kp.b_tx_bytes = (uint32_t)kp.BN * kp.KB * 2u;
  kp.b_bytes = (kp.b_tx_bytes + 1023u) & ~1023u;
  const uint32_t stage_bytes = kp.a_bytes + kp.b_bytes;
  int stages = (int)(kConvStageBudget / stage_bytes);
  if (stages > kConvMaxStages) stages = kConvMaxStages;
  PB_CHECK(stages >= 2, "conv: stage too large (%u bytes)", stage_bytes);
  kp.stages = stages;
  plan->smem_bytes = (size_t)stages * stage_bytes + sizeof(ConvSmemTail) + 1024;
  plan->threads = kConvThreads;
  plan->grid = kp.total_tiles < num_sms() ? kp.total_tiles : num_sms();
  const CUtensorMapSwizzle swz = kp.KB == 64   ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : kp.KB == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                               : CU_TENSOR_MAP_SWIZZLE_32B;
  {
    // activations: stride 1 -> (C, W, 1, H, N); stride 2 -> (2C, W/2, 2, H/2, N)
    const cuuint64_t C = (cuuint64_t)d->C, W = (cuuint64_t)d->W, H = (cuuint64_t)d->H;
    cuuint64_t dims[5];
    cuuint64_t strides[4];
    if (s == 1) {
      dims[0] = C; dims[1] = W; dims[2] = 1; dims[3] = H; dims[4] = (cuuint64_t)d->N;
      strides[0] = C * 2; strides[1] = W * C * 2; strides[2] = W * C * 2; strides[3] = H * W * C * 2;
    } else {
      dims[0] = 2 * C; dims[1] = W / 2; dims[2] = 2; dims[3] = H / 2; dims[4] = (cuuint64_t)d->N;
      strides[0] = 2 * C * 2; strides[1] = W * C * 2; strides[2] = 2 * W * C * 2; strides[3] = H * W * C * 2;
    }
    cuuint32_t box[5] = {(cuuint32_t)kp.KB, (cuuint32_t)TW, 1, (cuuint32_t)TH, (cuuint32_t)TN};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = encode(&plan->tmap_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(d->in), dims, strides,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(A) failed with %d (N=%d H=%d W=%d C=%d s=%d)", (int)r,
             d->N, d->H, d->W, d->C, s);
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)d->cin, (cuuint64_t)d->cout_pad, (cuuint64_t)kp.taps};
    cuuint64_t strides[2] = {(cuuint64_t)d->cin * 2, (cuuint64_t)d->cin * d->cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)kp.KB, (cuuint32_t)kp.BN, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&plan->tmap_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(d->weight), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  return 0;
}

int conv_plan_build(const pb_conv_desc* d, ConvPlan* plan) {
  const int rc = conv_plan_build_impl(d, plan);
  if (rc == 0) {
    plan->kp.fd_w = make_fastdiv(plan->kp.tiles_w);
    plan->kp.fd_h = make_fastdiv(plan->kp.tiles_h);
    plan->kp.fd_nt = make_fastdiv(plan->kp.n_ntiles);
  }
  return rc;
}

int conv_plan_launch(const ConvPlan* plan, cudaStream_t stream) {
  if (plan->variant == 1) return conv_halo_launch(plan, stream);
  typedef void (*TcKernelFn)(CUtensorMap, CUtensorMap, ConvKParams);
  const TcKernelFn fn = plan->epi == PB_EPI_SILU       ? conv_tc_kernel<PB_EPI_SILU>
                        : plan->epi == PB_EPI_RELU     ? conv_tc_kernel<PB_EPI_RELU>
                        : plan->epi == PB_EPI_SILU_RES ? conv_tc_kernel<PB_EPI_SILU_RES>
                        : plan->epi == PB_EPI_F32      ? conv_tc_kernel<PB_EPI_F32>
                                                       : conv_tc_kernel<PB_EPI_GENERIC>;
  PB_CUDA((cudaError_t)ensure_dynamic_smem(reinterpret_cast<const void*>(fn), 227 * 1024));
  PB_CUDA(launch_ex(fn, dim3(plan->grid), dim3(plan->threads), plan->smem_bytes, stream, 1, plan->pdl != 0, plan->tmap_a,
                    plan->tmap_w, plan->kp));
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// CUDA-core reference kernel (tests only): same descriptor, one thread per (pixel, out-channel)
// ------------------------------------------------------------------------------------------------------------
__global__ void conv_reference_kernel(pb_conv_desc d, int Ho, int Wo) {
  const long total = (long)d.N * Ho * Wo * d.cout_pad;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int co = (int)(idx % d.cout_pad);
    long pixl = idx / d.cout_pad;
    const int ow = (int)(pixl % Wo);
    const int oh = (int)((pixl / Wo) % Ho);
    const int n = (int)(pixl / ((long)Wo * Ho));
    if (co >= d.cout_store) continue;
    const __half* in = reinterpret_cast<const __half*>(d.in);
    const __half* w = reinterpret_cast<const __half*>(d.weight);
    float acc = 0.f;
    const int pad = d.ksize / 2;
    for (int r = 0; r < d.ksize; ++r)
      for (int q = 0; q < d.ksize; ++q) {
        const int ih = oh * d.stride + r - pad, iw = ow * d.stride + q - pad;
        if (ih < 0 || ih >= d.H || iw < 0 || iw >= d.W) continue;
        if (d.in_layout == PB_IN_STEM4) {  // padded 4-channel pixels; weight [r][cout][s*4 + c]
          const __half* ip = in + (((size_t)n * (d.H + 2) + ih + 1) * (d.W + 2) + iw + 1) * 4;
          const __half* wp = w + ((size_t)r * d.cout_pad + co) * 16 + q * 4;
          for (int c = 0; c < 3; ++c) acc += __half2float(ip[c]) * __half2float(wp[c]);
          continue;
        }
        const __half* ip = in + (((size_t)n * d.H + ih) * d.W + iw) * d.C + d.c_in_off;
        const __half* wp = w + ((size_t)(r * d.ksize + q) * d.cout_pad + co) * d.cin;
        for (int c = 0; c < d.cin; ++c) acc += __half2float(ip[c]) * __half2float(wp[c]);
      }
    float v = acc + d.bias[co];
    const size_t pix = ((size_t)n * Ho + oh) * Wo + ow;
    const float resv = d.res ? __half2float(reinterpret_cast<const __half*>(d.res)[pix * d.res_C + d.res_coff + co]) : 0.f;
    if (d.res_before_act) v += resv;
    if (d.act == PB_ACT_RELU) v = fmaxf(v, 0.f);
    else if (d.act == PB_ACT_SILU) v = v / (1.f + expf(-v));
    else if (d.act == PB_ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
    if (!d.res_before_act) v += resv;
    if (d.out_mode == PB_OUT_F16_NHWC) {
      reinterpret_cast<__half*>(d.out)[pix * d.out_C + d.out_coff + co] = __float2half_rn(v);
    } else if (d.out_mode == PB_OUT_F16_NHWC_UP2) {
      for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) {
          const size_t pix2 = ((size_t)n * (Ho * 2) + (oh * 2 + dy)) * (Wo * 2) + (ow * 2 + dx);
          reinterpret_cast<__half*>(d.out)[pix2 * d.out_C + d.out_coff + co] = __float2half_rn(v);
        }
    } else if (d.out_mode == PB_OUT_F32_NHWC) {
      reinterpret_cast<float*>(d.out)[pix * d.out_C + d.out_coff + co] = v;
    } else if (d.out_mode == PB_OUT_F32_NCHW) {
      reinterpret_cast<float*>(d.out)[(((size_t)n * d.cout_store + co) * Ho + oh) * Wo + ow] = v;
    }
    if (d.head_n > 0)  // tests only: head_out pre-zeroed by the caller, receives the pre-sigmoid sums (no bias)
      for (int j = 0; j < d.head_n; ++j)
        atomicAdd(d.head_out + (((size_t)n * d.head_n + j) * Ho + oh) * Wo + ow, d.head_weight[j * d.cout_pad + co] * v);
  }
}

int conv_reference_launch(const pb_conv_desc* d, cudaStream_t stream) {
  PB_CHECK(d != nullptr, "conv_reference: null desc");
  const int Ho = d->H / d->stride, Wo = d->W / d->stride;
  const long total = (long)d->N * Ho * Wo * d->cout_pad;
  int blocks = (int)((total + 255) / 256);
  if (blocks > (long)num_sms() * 32) blocks = (int)((long)num_sms() * 32);
  conv_reference_kernel<<<blocks, 256, 0, stream>>>(*d, Ho, Wo);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace pb
