// The halo conv kernel (conv_halo_kernel) and the lookup of its instantiations; the host set-ups live in
// conv_halo.cu.  Each epilogue class is instantiated in a translation unit of its own (conv_halo_inst_*.cu) so that the
// several hundred (S, k-steps, N) variants compile in parallel.
#pragma once
#include "conv_common.cuh"
#include "internal.h"
#include "ptx.cuh"

namespace pb {

constexpr int kHaloMaxA = 4;
constexpr int kHaloMaxB = 12;
// N tile of the layers conv_halo_setup splits into N tiles (cout > 192).  Only the kBN == kHaloNTileBN instantiations
// carry the N-tile index; in all others it is the constant 0, which keeps the widest ones (S = 1, N = 240: 128
// accumulators) free of spills.
constexpr int kHaloNTileBN = 128;

struct HaloSmemTail {
  uint64_t a_full[kHaloMaxA];
  uint64_t a_empty[kHaloMaxA];
  uint64_t b_full[kHaloMaxB];
  uint64_t b_empty[kHaloMaxB];
  float bias[kConvMaxCout];
  float scratch[kConvConsumerWarps * kEpiScratchFloats];  // epilogue transposition, one slice per consumer warp
};

struct HaloTile {
  int nt, tw, th, n;
};
// The N tile is the fastest index: the CTAs computing the N tiles of one spatial tile run at the same time, so all but
// the first read of its halo hit L2.
__device__ __forceinline__ HaloTile halo_decode(const ConvKParams& kp, int tile) {
  HaloTile t;
  int q;
  fast_divmod(q, t.nt, tile, kp.fd_nt);
  fast_divmod(q, t.tw, q, kp.fd_w);
  fast_divmod(t.n, t.th, q, kp.fd_h);
  return t;
}

// Channels per TMA store box of the staging tile: its rows are one swizzle span (128 / 64 / 32 bytes).
__host__ __device__ constexpr int halo_store_box_channels(int bn) { return bn % 64 == 0 ? 64 : (bn % 32 == 0 ? 32 : 16); }

// TMA-store epilogue (kp.st_bytes != 0) of one consumer warpgroup: its 8 image rows x 8S columns x kBN channels.
// Bias, activation and fp16 packing run on the accumulators in the wgmma fragment layout (channel 8i + 2(lane % 4),
// pixel row lane / 4 and + 8 = image rows 2wq, 2wq + 1) with the fp32 operations of epi_compute16, so the values are
// bit-identical to the per-lane store epilogue.  stmatrix writes them into the staging tile, laid out as TMA boxes
// (channels, 8S columns, 8 rows) whose 16-byte chunks carry the store map's swizzle (no bank conflicts at any pixel
// stride); one thread then issues the stores, and the warpgroup goes back to the next tile's wgmmas while the copy
// engine writes.  PB_OUT2_POOL2: the 2x2 maxima are read back from the staged tile and reuse the staging area once
// the primary stores have read it (no registers held across the accumulators).  TMA drops the parts of a box outside the tensor (edge tiles).
template <int kEpi, int kS, int kBN, int kAcc>
__device__ __forceinline__ void halo_epilogue_tma(const ConvKParams& kp, const HaloStoreMaps& maps,
                                                  const float (&acc)[kAcc], const float* __restrict__ sbias,
                                                  uint8_t* stage, const HaloTile& t, int g, int wq, int lane) {
  constexpr int kAS = (kBN + 31) / 32 * 16;  // accumulators per sub-tile
  constexpr int kBC = halo_store_box_channels(kBN);
  constexpr uint32_t kRow = 2u * kBC;               // staging row = one pixel's kBC channels = the swizzle span
  constexpr uint32_t kBox = 64u * kS * kRow;        // 8 rows x 8S columns
  constexpr uint32_t kPoolBox = 16u * kS * kRow;    // 4 x 4S pooled pixels
  constexpr int kCpr = kBC / 8;                     // 16-byte chunks per row
  const int act = kEpi == PB_EPI_SILU ? PB_ACT_SILU : (kEpi == PB_EPI_RELU ? PB_ACT_RELU : kp.act);
  const bool pool = kp.st_pool != 0;
  const bool leader = (threadIdx.x & 127) == 0;
  const int bar = 1 + g;  // named barrier of this warpgroup
  const int q = lane & 3, mi = lane >> 3;
  const uint32_t sbase = smem_u32(stage);
  // stmatrix: lane l addresses row l % 8 (= pixel column) of matrix mi = l / 8 (image row + (mi & 1), channel chunk
  // + (mi >> 1)).  Pixel index = image row * 8S + column, so the swizzle key (the pixel's 128-byte line mod the span)
  // is a per-lane constant.
  const uint32_t key = (((uint32_t)(lane & 7) * kRow) >> 7) & (uint32_t)(kCpr - 1);
  const uint32_t lane_row = sbase + (uint32_t)((2 * wq + (mi & 1)) * 8 * kS + (lane & 7)) * kRow;
  const uint32_t hi = (uint32_t)(mi >> 1);

  if (leader) bulk_wait_group_read0();  // the previous tile's stores have read the staging area
  named_barrier_sync(bar, 128);
#pragma unroll
  for (int j = 0; j < kS; ++j) {
#pragma unroll
    for (int i = 0; i < kBN / 8; i += 2) {  // 16 channels: fragment column blocks i, i + 1
      uint32_t h[4];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float* a4 = acc + j * kAS + 4 * (i + u);
        const float2 b = *reinterpret_cast<const float2*>(sbias + 8 * (i + u) + 2 * q);
        float v0 = a4[0] + b.x, v1 = a4[1] + b.y, v2 = a4[2] + b.x, v3 = a4[3] + b.y;
        if (act == PB_ACT_SILU) {
          silu2_frag(v0, v1);
          silu2_frag(v2, v3);
        } else if (act == PB_ACT_RELU) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
          v2 = fmaxf(v2, 0.f);
          v3 = fmaxf(v3, 0.f);
        } else if (act == PB_ACT_SIGMOID) {
          v0 = __fdividef(1.f, 1.f + __expf(-v0));
          v1 = __fdividef(1.f, 1.f + __expf(-v1));
          v2 = __fdividef(1.f, 1.f + __expf(-v2));
          v3 = __fdividef(1.f, 1.f + __expf(-v3));
        }
        const __half2 top = __floats2half2_rn(v0, v1), bot = __floats2half2_rn(v2, v3);
        h[2 * u] = *reinterpret_cast<const uint32_t*>(&top);
        h[2 * u + 1] = *reinterpret_cast<const uint32_t*>(&bot);
      }
      const uint32_t chunk = ((uint32_t)(i % kCpr) + hi) ^ key;
      stmatrix_x4(lane_row + (uint32_t)(i / kCpr) * kBox + (uint32_t)(8 * j) * kRow + (chunk << 4), h[0], h[1], h[2],
                  h[3]);
    }
  }
  fence_proxy_async_smem();
  named_barrier_sync(bar, 128);
  const int x0 = t.tw * 8 * kS, y0 = t.th * 16 + 8 * g;
  if (leader) {
    for (int m = 0; m < kp.st_maps; ++m)
#pragma unroll
      for (int b = 0; b < kBN / kBC; ++b)
        tma_store_4d(&maps.m[m], stage + b * kBox, t.nt * kBN + b * kBC, x0, y0, t.n);
    bulk_commit_group();
  }
  if (pool) {
    // 16-byte units (8 channels of one pooled pixel) of the 4 x 4S pooled box, read back from the staged tile while
    // the primary stores read it too; written once those have finished reading.
    constexpr int kUnits = 2 * kS * kBN, kPer = (kUnits + 127) / 128;
    auto addr = [&](int pix, int cc, uint32_t box) {
      const uint32_t k = (((uint32_t)pix * kRow) >> 7) & (uint32_t)(kCpr - 1);
      return sbase + (uint32_t)(cc / kCpr) * box + (uint32_t)pix * kRow + ((((uint32_t)(cc % kCpr)) ^ k) << 4);
    };
    const int tid = threadIdx.x & 127;
    uint4 pv[kPer];
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int un = tid + 128 * k, cc = un % (kBN / 8), pp = un / (kBN / 8);
      const int src = (pp / (4 * kS)) * 16 * kS + 2 * (pp % (4 * kS));  // top-left pixel of the 2x2 window
      if (un < kUnits) {
        uint4 w[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(w[e].x), "=r"(w[e].y), "=r"(w[e].z), "=r"(w[e].w)
                       : "r"(addr(src + (e >> 1) * 8 * kS + (e & 1), cc, kBox))
                       : "memory");
        const __half2* h0 = reinterpret_cast<const __half2*>(&w[0]);
        const __half2* h1 = reinterpret_cast<const __half2*>(&w[1]);
        const __half2* h2 = reinterpret_cast<const __half2*>(&w[2]);
        const __half2* h3 = reinterpret_cast<const __half2*>(&w[3]);
        __half2* o = reinterpret_cast<__half2*>(&pv[k]);
#pragma unroll
        for (int c = 0; c < 4; ++c) o[c] = __hmax2(__hmax2(h0[c], h1[c]), __hmax2(h2[c], h3[c]));
      }
    }
    if (leader) bulk_wait_group_read0();
    named_barrier_sync(bar, 128);
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int un = tid + 128 * k;
      if (un < kUnits)
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr(un / (kBN / 8), un % (kBN / 8), kPoolBox)),
                     "r"(pv[k].x), "r"(pv[k].y), "r"(pv[k].z), "r"(pv[k].w)
                     : "memory");
    }
    fence_proxy_async_smem();
    named_barrier_sync(bar, 128);
    if (leader) {
#pragma unroll
      for (int b = 0; b < kBN / kBC; ++b)
        tma_store_4d(&maps.m[kp.st_maps], stage + b * kPoolBox, t.nt * kBN + b * kBC, x0 >> 1, y0 >> 1, t.n);
      bulk_commit_group();
    }
  }
}

// kS (sub-tiles), kSteps (16-element k-steps per channel block) and kBN (the N tile = cout_pad) are compile-time so
// the wgmma issue loop is straight-line code with immediate descriptor offsets, the accumulator array holds exactly
// the kS * ceil(kBN / 32) * 16 registers this layer needs, and the epilogue indexes it with constants.  One
// instantiation per N keeps ptxas from reserving registers for the widest case, which would serialise the wgmmas
// (no group in flight while the next is issued) and spill.
template <int kS, int kSteps, int kBN, int kEpi>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const __grid_constant__ ConvKParams kp, const __grid_constant__ HaloStoreMaps tmap_o) {
  constexpr int kNch = (kBN + 31) / 32;  // 32-column epilogue chunks per sub-tile
  constexpr int kAcc = kS * kNch * 16;   // fp32 accumulators per consumer thread
  static_assert(kAcc <= kConvAccRegs, "accumulators of kS sub-tiles must fit the registers");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_base = smem;
  uint8_t* b_base = smem + (size_t)kp.a_stages * kp.a_bytes;
  uint8_t* st_base = b_base + (size_t)kp.b_stages * kp.b_bytes;  // TMA-store staging, kp.st_bytes / 2 per warpgroup
  HaloSmemTail* tail = reinterpret_cast<HaloSmemTail*>(st_base + kp.st_bytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int S = kS;
  const int G = kp.hs_G;
  const uint32_t row_bytes = (uint32_t)kp.KB * 2u;       // weight rows (and activation rows unless stride 2)
  const uint32_t a_row_bytes = kp.hs_a_row_bytes;        // activation (halo) rows
  const int tap_groups = kp.hs_ntaps / G;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    for (int i = 0; i < kp.a_stages; ++i) {
      mbar_init(&tail->a_full[i], 1);
      mbar_init(&tail->a_empty[i], kConvConsumerWarps);
    }
    for (int i = 0; i < kp.b_stages; ++i) {
      mbar_init(&tail->b_full[i], 1);
      mbar_init(&tail->b_empty[i], kConvConsumerWarps);
    }
    fence_mbar_init();
  }
  if (warp == 1 && lane == 0) tma_prefetch_desc(&tmap_w);
  if (warp == 2 && lane < kp.st_maps + kp.st_pool) tma_prefetch_desc(&tmap_o.m[lane]);
  for (int i = threadIdx.x; i < kp.cout_pad; i += blockDim.x) tail->bias[i] = kp.bias[i];
  __syncthreads();
  // PDL: the prologue above touched constant data only; from here on activations are read and written.  The weight
  // producer (warp 1) reads constants only and starts fetching while the previous kernel is still running.
  griddep_launch_dependents();
  if (warp != 1) griddep_wait();

  if (warp < 4) {
    warpgroup_reg_dealloc<kConvProducerRegs>();
    if (warp == 0 && lane == 0) {
      // ===================== halo producer: one TMA box per (tile, channel block) =====================
      int st = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < kp.total_tiles; tile += gridDim.x) {
        const HaloTile t = halo_decode(kp, tile);
        for (int cb = 0; cb < kp.kblocks; ++cb) {
          mbar_wait(&tail->a_empty[st], ph ^ 1);
          mbar_arrive_expect_tx(&tail->a_full[st], kp.halo_bytes);
          tma_load_5d(a_base + (size_t)st * kp.a_bytes, &tmap_a, &tail->a_full[st], kp.c_in_off + cb * kp.KB,
                      t.tw * 8 * S + kp.hs_x0, 0, t.th * 16 + kp.hs_y0, t.n);
          if (++st == kp.a_stages) {
            st = 0;
            ph ^= 1;
          }
        }
      }
    } else if (warp == 1 && lane == 0) {
      // ===================== weight producer: one TMA box per (channel block, tap group) =====================
      // Resident mode (kp.b_resident: the whole filter bank fits next to the halo ring): every box is fetched ONCE per
      // CTA and reused by all its tiles -- without it a small-channel layer re-reads its weights from L2 for every
      // tile, as many bytes as the activations themselves.
      int st = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < kp.total_tiles; tile += gridDim.x) {
        const int co = kBN == kHaloNTileBN ? halo_decode(kp, tile).nt * kBN : 0;  // first channel of the N tile
        for (int cb = 0; cb < kp.kblocks; ++cb) {
          for (int tg = 0; tg < tap_groups; ++tg) {
            if (!kp.b_resident) mbar_wait(&tail->b_empty[st], ph ^ 1);
            mbar_arrive_expect_tx(&tail->b_full[st], kp.b_tx_bytes);
            tma_load_3d(b_base + (size_t)st * kp.b_bytes, &tmap_w, &tail->b_full[st], cb * kp.KB, co, tg * G);
            if (++st == kp.b_stages) {
              st = 0;
              ph ^= 1;
            }
          }
        }
        if (kp.b_resident) break;
      }
    }
    return;
  }

  // ===================== consumers: wgmma + epilogue =====================
  // A sub-tile is 16 image rows x 8 columns = 128 pixels (row m = 8 * image row + column); warpgroup g computes its
  // image rows 8g .. 8g + 7, i.e. the 8-row groups 8g .. 8g + 7 of every tap's A descriptor.
  warpgroup_reg_alloc<kConvConsumerRegs>();
  const int cw = warp - 4, g = cw >> 2, wq = cw & 3;
  // g broadcast from lane 0: the compiler then knows the warpgroup skip test below, and with it the ring positions
  // after it, are warp-uniform, and keeps the descriptor arithmetic in uniform registers
  const int g_uni = __shfl_sync(0xffffffffu, g, 0);
  float* scr = tail->scratch + cw * kEpiScratchFloats;
  const uint32_t sbo = (uint32_t)kp.hs_sbo_rows * a_row_bytes;
  const uint64_t g_units = (uint64_t)((8u * (uint32_t)g * sbo) >> 4);
  const uint32_t tap_b_units = ((uint32_t)kBN * row_bytes) >> 4;               // 16-byte units
  const uint64_t sub_units = (uint64_t)((8u * a_row_bytes) >> 4);              // next sub-tile: +8 pixels
  const int m = 64 * g + 16 * wq + (lane & 15);  // this lane's pixel of each sub-tile in the epilogue
  const int row = m >> 3, col = m & 7;
  float acc[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
  int ast = 0, bst = 0;
  uint32_t aph = 0, bph = 0;
  for (int tile = blockIdx.x; tile < kp.total_tiles; tile += gridDim.x) {
    HaloTile t = halo_decode(kp, tile);
    if constexpr (kBN != kHaloNTileBN) t.nt = 0;
    if (t.th * 16 + 8 * g_uni >= kp.Ho) {
      // All 8 image rows of this warpgroup lie below the image (last tile row of a height that is not a multiple of
      // 16): no wgmmas and no stores.  It still waits on every stage and releases it -- the empty barriers count its
      // warps' arrivals -- and keeps the ring phases in step with its partner.
      for (int cb = 0; cb < kp.kblocks; ++cb) {
        mbar_wait(&tail->a_full[ast], aph);
        for (int tg = 0; tg < tap_groups; ++tg) {
          mbar_wait(&tail->b_full[bst], kp.b_resident ? 0u : bph);
          if (!kp.b_resident) consumer_release(&tail->b_empty[bst], lane);
          if (++bst == kp.b_stages) {
            bst = 0;
            bph ^= 1;
          }
        }
        consumer_release(&tail->a_empty[ast], lane);
        if (++ast == kp.a_stages) {
          ast = 0;
          aph ^= 1;
        }
      }
      continue;
    }
    // One group of wgmmas (one weight stage) stays in flight while the next is issued: a weight stage is released
    // once the group after it has been issued and wgmma_wait<1> has retired it, a halo stage once the first group
    // of the next channel block has (prev_b / prev_a: the stages still read by the group in flight, -1 = none).
    int prev_b = -1, prev_a = -1;
    for (int cb = 0; cb < kp.kblocks; ++cb) {
      mbar_wait(&tail->a_full[ast], aph);
      // Descriptor arithmetic is hoisted: per (channel block, weight stage) one base descriptor each; taps,
      // sub-tiles and k-steps only add precomputed 16-byte-unit offsets to the low word.
      const uint64_t a_desc0 = wgmma_desc(smem_u32(a_base + (size_t)ast * kp.a_bytes), a_row_bytes, sbo) + g_units;
      for (int tg = 0; tg < tap_groups; ++tg) {
        mbar_wait(&tail->b_full[bst], kp.b_resident ? 0u : bph);  // resident: filled once, phase 0 stays complete
        const uint64_t b_desc0 = wgmma_desc_kmajor(smem_u32(b_base + (size_t)bst * kp.b_bytes), row_bytes);
        wgmma_fence();
        for (int ti = 0; ti < G; ++ti) {
          const int tap = tg * G + ti;
          mma_n<kBN, kS, kSteps>(acc, a_desc0 + (uint64_t)(uint32_t)kp.hs_tap_desc[tap], sub_units,
                                 b_desc0 + (uint64_t)((uint32_t)ti * tap_b_units), (uint32_t)((cb | tap) != 0));
        }
        wgmma_commit();
        if (prev_b >= 0) {
          wgmma_wait<1>();
          if (!kp.b_resident) consumer_release(&tail->b_empty[prev_b], lane);
          if (prev_a >= 0) consumer_release(&tail->a_empty[prev_a], lane);
          prev_a = -1;
        }
        prev_b = bst;
        if (++bst == kp.b_stages) {
          bst = 0;
          bph ^= 1;
        }
      }
      prev_a = ast;
      if (++ast == kp.a_stages) {
        ast = 0;
        aph ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (!kp.b_resident) consumer_release(&tail->b_empty[prev_b], lane);
    consumer_release(&tail->a_empty[prev_a], lane);
    const float* sbias = tail->bias + t.nt * kBN;
    if constexpr (kEpi != PB_EPI_SILU_RES) {  // a residual keeps the per-lane store epilogue
      if (kp.st_bytes != 0) {
        halo_epilogue_tma<kEpi, kS, kBN>(kp, tmap_o, acc, sbias, st_base + (size_t)g * (kp.st_bytes / 2), t, g, wq,
                                         lane);
        continue;
      }
    }
    const int oh = t.th * 16 + row, ow0 = t.tw * 8 * S + col;
    epilogue_tile<kEpi, kS, kNch>(kp, acc, S, t.nt, sbias, scr, lane, [&](int j, bool& pool_writer) {
      EpiPix px;
      px.n = t.n;
      px.oh = oh;
      px.ow = ow0 + 8 * j;
      px.valid = (px.ow < kp.Wo) && (px.oh < kp.Ho);
      px.pix = ((size_t)px.n * kp.Ho + px.oh) * kp.Wo + px.ow;
      pool_writer = ((row | col) & 1) == 0;
      return px;
    });
  }
  if (kp.st_bytes != 0 && (threadIdx.x & 127) == 0) bulk_wait_group0();  // the stores complete before the CTA exits
}

typedef void (*HaloKernelFn)(CUtensorMap, CUtensorMap, ConvKParams, HaloStoreMaps);

// Instantiations: every N tile a halo set-up can produce (cout_pad = 16 .. 256 in steps of 16) with every sub-tile
// count whose accumulators fit (S * ceil(N / 32) * 16 <= kConvAccRegs), for k-steps 1 / 2 / 4 (KB = 16 / 32 / 64).
template <int kS, int kSteps, int kEpi>
static HaloKernelFn halo_kernel_for_bn(int BN) {
  switch (BN) {
#define PB_HALO_BN(n_)                                                                     \
  case n_:                                                                                 \
    if constexpr (kS * ((n_ + 31) / 32) * 16 <= kConvAccRegs) return conv_halo_kernel<kS, kSteps, n_, kEpi>; \
    break;
    PB_HALO_BN(16) PB_HALO_BN(32) PB_HALO_BN(48) PB_HALO_BN(64) PB_HALO_BN(80) PB_HALO_BN(96) PB_HALO_BN(112)
    PB_HALO_BN(128) PB_HALO_BN(144) PB_HALO_BN(160) PB_HALO_BN(176) PB_HALO_BN(192) PB_HALO_BN(208)
    PB_HALO_BN(224) PB_HALO_BN(240) PB_HALO_BN(256)
#undef PB_HALO_BN
    default: break;
  }
  return nullptr;
}

template <int kEpi>
HaloKernelFn halo_kernel_lookup(int S, int steps, int BN) {
#define PB_HALO_CASE(s_, k_) \
  if (S == s_ && steps == k_) return halo_kernel_for_bn<s_, k_, kEpi>(BN);
  PB_HALO_CASE(1, 1) PB_HALO_CASE(1, 2) PB_HALO_CASE(1, 4)
  PB_HALO_CASE(2, 1) PB_HALO_CASE(2, 2) PB_HALO_CASE(2, 4)
  PB_HALO_CASE(4, 1) PB_HALO_CASE(4, 2) PB_HALO_CASE(4, 4)
#undef PB_HALO_CASE
  return nullptr;
}


// instantiated in conv_halo_inst_*.cu
extern template HaloKernelFn halo_kernel_lookup<PB_EPI_GENERIC>(int, int, int);
extern template HaloKernelFn halo_kernel_lookup<PB_EPI_SILU>(int, int, int);
extern template HaloKernelFn halo_kernel_lookup<PB_EPI_RELU>(int, int, int);
extern template HaloKernelFn halo_kernel_lookup<PB_EPI_SILU_RES>(int, int, int);

}  // namespace pb
