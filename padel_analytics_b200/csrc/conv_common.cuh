// Epilogue helpers shared by the conv kernels (per-tap conv_tc_kernel and halo conv_halo_kernel).
#pragma once
#include "internal.h"
#include "ptx.cuh"

namespace pb {

// bias + activation on 16 accumulator columns; `act` is CTA-uniform and each case is a straight unrolled loop so
// the 16 independent MUFU chains interleave
__device__ __forceinline__ void bias_act16(const uint32_t (&r)[16], const float* __restrict__ sbias, int act,
                                           float (&v)[16], const __half* __restrict__ res_first = nullptr) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 b = *reinterpret_cast<const float4*>(sbias + 4 * q);
    v[4 * q + 0] = __uint_as_float(r[4 * q + 0]) + b.x;
    v[4 * q + 1] = __uint_as_float(r[4 * q + 1]) + b.y;
    v[4 * q + 2] = __uint_as_float(r[4 * q + 2]) + b.z;
    v[4 * q + 3] = __uint_as_float(r[4 * q + 3]) + b.w;
  }
  if (res_first != nullptr) {  // ResNet: the identity joins before the activation
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] += __half2float(res_first[j]);
  }
  if (act == PB_ACT_SILU) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = __fdividef(v[i], 1.f + __expf(-v[i]));
  } else if (act == PB_ACT_RELU) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
  } else if (act == PB_ACT_SIGMOID) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = __fdividef(1.f, 1.f + __expf(-v[i]));
  }
}

// one 32-byte run of 16 fp16 channels (a full 32-byte sector) as two 16-byte stores
__device__ __forceinline__ void st_global_256(void* p, const uint4& a, const uint4& b) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = a;
  q[1] = b;
}

struct EpiPix {
  bool valid;
  int n, oh, ow;
  size_t pix;
};

// residual / fused head / store of 16 activated channels starting at output channel ch0 (c = column in the N tile)
__device__ __forceinline__ void epilogue_store16(const ConvKParams& kp, const EpiPix& px, int ch0, int c,
                                                 float (&v)[16], float (&hacc)[8]) {
  if (kp.res != nullptr && !kp.res_first) {
    const uint4* rp = reinterpret_cast<const uint4*>(kp.res + px.pix * kp.res_C + kp.res_coff + ch0);
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      const uint4 rv = __ldg(rp + g);
      const __half2* h2 = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        v[8 * g + 2 * j] += f.x;
        v[8 * g + 2 * j + 1] += f.y;
      }
    }
  }
  if (kp.head_n > 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < kp.head_n) {
        const float4* w4 = reinterpret_cast<const float4*>(kp.head_w + (size_t)j * kp.BN + c);
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int q = 0; q < 4; q += 2) {
          const float4 wa = __ldg(w4 + q), wb = __ldg(w4 + q + 1);
          s0 = fmaf(wa.x, v[4 * q], fmaf(wa.y, v[4 * q + 1], fmaf(wa.z, v[4 * q + 2], fmaf(wa.w, v[4 * q + 3], s0))));
          s1 = fmaf(wb.x, v[4 * q + 4], fmaf(wb.y, v[4 * q + 5], fmaf(wb.z, v[4 * q + 6], fmaf(wb.w, v[4 * q + 7], s1))));
        }
        hacc[j] += s0 + s1;
      }
    }
  }
  if (kp.out_mode == PB_OUT_F16_NHWC || kp.out_mode == PB_OUT_F16_NHWC_UP2) {
    uint4 pk[2];
    __half2* h2 = reinterpret_cast<__half2*>(pk);
#pragma unroll
    for (int j = 0; j < 8; ++j) h2[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
    __half* ob = reinterpret_cast<__half*>(kp.out);
    const bool two = (kp.cout_store - ch0 >= 16);  // cout_store is a multiple of 8
    const bool wide = two && (((kp.out_C | kp.out_coff) & 15) == 0);  // 32-byte aligned 16-channel run
    if (kp.out_mode == PB_OUT_F16_NHWC) {
      uint4* op = reinterpret_cast<uint4*>(ob + px.pix * kp.out_C + kp.out_coff + ch0);
      if (wide) {
        st_global_256(op, pk[0], pk[1]);
      } else {
        op[0] = pk[0];
        if (two) op[1] = pk[1];
      }
    } else {
      const int Wo2 = kp.Wo * 2;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const size_t pix2 = ((size_t)px.n * (kp.Ho * 2) + (px.oh * 2 + dy)) * Wo2 + (px.ow * 2 + dx);
          uint4* op = reinterpret_cast<uint4*>(ob + pix2 * kp.out_C + kp.out_coff + ch0);
          if (wide) {
            st_global_256(op, pk[0], pk[1]);
          } else {
            op[0] = pk[0];
            if (two) op[1] = pk[1];
          }
        }
    }
  } else if (kp.out_mode == PB_OUT_F32_NHWC) {
    float* op = reinterpret_cast<float*>(kp.out) + px.pix * kp.out_C + kp.out_coff + ch0;
    if (((kp.out_C | kp.out_coff) & 3) == 0) {  // 16-byte aligned rows: vector stores for the full groups
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (ch0 + 4 * q + 4 <= kp.cout_store) {
          *reinterpret_cast<float4*>(op + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
        } else {
#pragma unroll
          for (int j = 4 * q; j < 4 * q + 4; ++j)
            if (ch0 + j < kp.cout_store) op[j] = v[j];
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (ch0 + j < kp.cout_store) op[j] = v[j];
    }
  } else if (kp.out_mode == PB_OUT_F32_NCHW) {
    float* ob = reinterpret_cast<float*>(kp.out);
    const size_t plane = (size_t)kp.Ho * kp.Wo;
    const size_t base = (size_t)px.n * kp.cout_store * plane + (size_t)px.oh * kp.Wo + px.ow;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      if (ch0 + j < kp.cout_store) ob[base + (size_t)(ch0 + j) * plane] = v[j];
  }
}

// ------------------------------------------------------------------------------------------------------------
// Fast epilogue for the common case (fp16 NHWC slice out, 32-byte aligned 16-channel runs, no fused head).
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool epilogue_fast_ok(const ConvKParams& kp) {
  if ((kp.dbg_flags & 2) != 0 && kp.out2_mode == PB_OUT2_NONE) return false;
  if (kp.head_n != 0 || (kp.res != nullptr && ((kp.res_C | kp.res_coff) & 7) != 0)) return false;
  if ((reinterpret_cast<uintptr_t>(kp.out) & 31) != 0) return false;  // 32-byte stores
  if (kp.out_mode == PB_OUT_F16_NHWC || kp.out_mode == PB_OUT_F16_NHWC_UP2)
    return ((kp.out_C | kp.out_coff) & 15) == 0 && (kp.cout_store & 15) == 0;
  if (kp.out_mode == PB_OUT_F32_NHWC) return ((kp.out_C | kp.out_coff) & 7) == 0;  // 32-byte aligned 8-float groups
  return false;
}

// SiLU on four values with ONE reciprocal: 1/da = db*dc*dd * r, ... with r = 1/(da*db*dc*dd), d = 1 + 2^(-v*log2 e).
// The plain form v / (1 + exp(-v)) costs two MUFU operations per value (EX2 + RCP), and the MUFU pipe is what bounds
// the epilogue of a wide SiLU layer; this one costs 1.25 plus a few FMULs on the FMA pipe, with the same few-ulp fp32
// accuracy (no approximation of the function itself).
// The exponent is clamped to 2^30 so that the product of four stays finite (< 2^121); silu(v) for v < -20.8 is below
// 2e-8 in magnitude either way, i.e. an fp16 zero / smallest subnormal.
// PADEL_B200_CONV_DEBUG bit 0 selects the plain two-MUFU form for A/B runs.
__device__ __forceinline__ void silu4(float& a, float& b, float& c, float& d) {
  constexpr float kNegLog2e = -1.4426950408889634f;
  const float da = 1.f + ex2_approx(fminf(a * kNegLog2e, 30.f));
  const float db = 1.f + ex2_approx(fminf(b * kNegLog2e, 30.f));
  const float dc = 1.f + ex2_approx(fminf(c * kNegLog2e, 30.f));
  const float dd = 1.f + ex2_approx(fminf(d * kNegLog2e, 30.f));
  const float pab = da * db, pcd = dc * dd;
  const float r = rcp_approx(pab * pcd);
  const float rab = pcd * r, rcd = pab * r;  // 1 / (da db), 1 / (dc dd)
  a *= db * rab;
  b *= da * rab;
  c *= dd * rcd;
  d *= dc * rcd;
}

// silu4 on the wgmma fragment layout, where channels 4k .. 4k+3 of a pixel are split over lane l (two of them) and
// lane l ^ 1 (the other two).  Each lane forms its pair's product of denominators, swaps it with lane l ^ 1 and
// finishes its two values with the operations silu4 applies to them, so the results are bit-identical (the product
// of the two pair products is commutative).  Every lane of the warp must call it.
__device__ __forceinline__ void silu2_frag(float& a, float& b) {
  constexpr float kNegLog2e = -1.4426950408889634f;
  const float da = 1.f + ex2_approx(fminf(a * kNegLog2e, 30.f));
  const float db = 1.f + ex2_approx(fminf(b * kNegLog2e, 30.f));
  const float p = da * db;
  const float po = __shfl_xor_sync(0xffffffffu, p, 1);
  const float r = rcp_approx(p * po);
  const float rp = po * r;  // 1 / (da db)
  a *= db * rp;
  b *= da * rp;
}

// Where one thread's 16-channel chunk goes: byte pointer of the pixel (channel 0 of the N tile), byte strides of the
// 2x2 replication (UP2 only) and the number of channels of this chunk that exist (fp32 heads may end mid-chunk).
struct EpiOut {
  int mode;       // PB_OUT_F16_NHWC | PB_OUT_F16_NHWC_UP2 | PB_OUT_F32_NHWC   (CTA-uniform)
  size_t dx, dy;  // UP2: bytes to the pixel one to the right / one row down in the upsampled tensor
  int mode2;      // PB_OUT2_*: secondary output (CTA-uniform)
  size_t dx2, dy2;  // PB_OUT2_UP2: the same strides in the secondary tensor
  bool pool_writer;  // PB_OUT2_POOL2: this lane owns the top-left pixel of a 2x2 window
};

// bias + activation (+ residual) of one 16-column chunk of this thread's pixel
__device__ __forceinline__ void epi_add_res16(const uint4 (&rv)[2], float (&v)[16]) {
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    const __half2* h2 = reinterpret_cast<const __half2*>(&rv[g]);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h2[j]);
      // __fadd_rn: never contracted with the activation's last multiply into an FMA -- the folded epilogue classes
      // would otherwise round differently from the run-time epilogue, and a frame's result must not depend on which
      // of them its batch size selects (tests/test_full_size_gpu.py)
      v[8 * g + 2 * j] = __fadd_rn(v[8 * g + 2 * j], f.x);
      v[8 * g + 2 * j + 1] = __fadd_rn(v[8 * g + 2 * j + 1], f.y);
    }
  }
}

// has_res: 0 none, 1 residual after the activation, 2 residual before it (CTA-uniform)
__device__ __forceinline__ void epi_compute16(int act, int has_res, bool plain_silu, uint32_t (&r)[16],
                                              const float* __restrict__ sbias, const uint4 (&rv)[2], float (&v)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 b = *reinterpret_cast<const float4*>(sbias + 4 * q);
    v[4 * q + 0] = __uint_as_float(r[4 * q + 0]) + b.x;
    v[4 * q + 1] = __uint_as_float(r[4 * q + 1]) + b.y;
    v[4 * q + 2] = __uint_as_float(r[4 * q + 2]) + b.z;
    v[4 * q + 3] = __uint_as_float(r[4 * q + 3]) + b.w;
  }
  if (has_res == 2) epi_add_res16(rv, v);
  if (act == PB_ACT_SILU) {  // CTA-uniform
    if (plain_silu) {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = __fdividef(v[i], 1.f + __expf(-v[i]));
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) silu4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
  } else if (act == PB_ACT_RELU) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
  } else if (act == PB_ACT_SIGMOID) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = __fdividef(1.f, 1.f + __expf(-v[i]));
  }
  if (has_res == 1) epi_add_res16(rv, v);
}

__device__ __forceinline__ void epi_chunk(int act, int has_res, bool plain_silu, const EpiOut& eo, uint32_t (&r)[16],
                                          const float* __restrict__ sbias, char* op, const uint4 (&rv)[2], bool valid,
                                          int nvalid, char* op2 = nullptr, bool vec_tail = false) {
  float v[16];
  epi_compute16(act, has_res, plain_silu, r, sbias, rv, v);
  if (eo.mode == PB_OUT_F32_NHWC) {
    if (!valid) return;
    if (nvalid >= 16) {
      uint4 w[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        w[q] = make_uint4(__float_as_uint(v[4 * q]), __float_as_uint(v[4 * q + 1]), __float_as_uint(v[4 * q + 2]),
                          __float_as_uint(v[4 * q + 3]));
      st_global_256(op, w[0], w[1]);
      st_global_256(op + 32, w[2], w[3]);
    } else {  // the N tile ends inside this chunk: one 32-byte store if at least 8 floats exist, scalars for the rest
      float* o = reinterpret_cast<float*>(op);
      int j0 = 0;
      if (vec_tail && nvalid >= 8) {
        st_global_256(op, make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3])),
                      make_uint4(__float_as_uint(v[4]), __float_as_uint(v[5]), __float_as_uint(v[6]), __float_as_uint(v[7])));
        j0 = 8;
      }
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (j >= j0 && j < nvalid) o[j] = v[j];
    }
    return;
  }
  uint4 pk[2];
  __half2* h2 = reinterpret_cast<__half2*>(pk);
#pragma unroll
  for (int j = 0; j < 8; ++j) h2[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
  if (eo.mode2 == PB_OUT2_POOL2) {
    // 2x2 max over the lanes holding (row, col), (row, col^1), (row^1, col), (row^1, col^1) of the 4 x 8 pixel patch of
    // this warp (lane = row_in_patch * 8 + col): two butterfly steps, executed by every lane (a window is entirely
    // valid or entirely invalid: H, W and the tile origins are even)
    uint4 mx[2] = {pk[0], pk[1]};
    __half2* m2 = reinterpret_cast<__half2*>(mx);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t w = *reinterpret_cast<uint32_t*>(&m2[j]);
      uint32_t o = __shfl_xor_sync(0xffffffffu, w, 1);
      m2[j] = __hmax2(m2[j], *reinterpret_cast<__half2*>(&o));
      w = *reinterpret_cast<uint32_t*>(&m2[j]);
      o = __shfl_xor_sync(0xffffffffu, w, 8);
      m2[j] = __hmax2(m2[j], *reinterpret_cast<__half2*>(&o));
    }
    if (valid && eo.pool_writer) st_global_256(op2, mx[0], mx[1]);
  }
  if (!valid) return;
  st_global_256(op, pk[0], pk[1]);
  if (eo.mode2 == PB_OUT2_UP2) {
    st_global_256(op2, pk[0], pk[1]);
    st_global_256(op2 + eo.dx2, pk[0], pk[1]);
    st_global_256(op2 + eo.dy2, pk[0], pk[1]);
    st_global_256(op2 + eo.dy2 + eo.dx2, pk[0], pk[1]);
  }
  if (eo.mode == PB_OUT_F16_NHWC_UP2) {
    st_global_256(op + eo.dx, pk[0], pk[1]);
    st_global_256(op + eo.dy, pk[0], pk[1]);
    st_global_256(op + eo.dy + eo.dx, pk[0], pk[1]);
  }
}

// Epilogue of the wgmma conv kernels.  A consumer warp holds 16 pixels x N columns of each sub-tile in the wgmma
// fragment layout; per 32-column chunk a shared-memory scratch transposes them so that lane l gets 16 channels of one
// pixel (row l % 16, columns 16 (l / 16) ..), the unit of the stores above (lanes l ^ 1 / l ^ 8: the neighbours the
// PB_OUT2_POOL2 butterfly needs).  Sub-tile j occupies acc[j * 16 ceil(N / 32) ...): chunk u is acc[16 u .. 16 u + 16).
constexpr int kConvAccRegs = 128;   // fp32 accumulators per consumer thread: S * 16 * ceil(N / 32) <= 128
constexpr int kEpiScratchPitch = 36;  // floats per scratch row (32 + 4 spreads the fragment stores over the banks)
constexpr int kEpiScratchFloats = 16 * kEpiScratchPitch;  // per consumer warp

template <int kU, int kAcc>
__device__ __forceinline__ void epi_frag_store(const float (&acc)[kAcc], float* scr, int lane) {
  if constexpr (16 * kU < kAcc) {
    const int r0 = lane >> 2, q = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      *reinterpret_cast<float2*>(scr + r0 * kEpiScratchPitch + 8 * i + 2 * q) =
          make_float2(acc[16 * kU + 4 * i], acc[16 * kU + 4 * i + 1]);
      *reinterpret_cast<float2*>(scr + (r0 + 8) * kEpiScratchPitch + 8 * i + 2 * q) =
          make_float2(acc[16 * kU + 4 * i + 2], acc[16 * kU + 4 * i + 3]);
    }
  }
}

// chunk u of the accumulators -> this lane's 16 channels.  With a compile-time u (unrolled caller) the switch folds
// to one case.
template <int kAcc>
__device__ __forceinline__ void epi_transpose16(const float (&acc)[kAcc], int u, float* scr, int lane,
                                                uint32_t (&r)[16]) {
  __syncwarp();  // the previous chunk's reads are done
  switch (u) {  // CTA-uniform; the accumulator index has to be a compile-time constant
    case 0: epi_frag_store<0>(acc, scr, lane); break;
    case 1: epi_frag_store<1>(acc, scr, lane); break;
    case 2: epi_frag_store<2>(acc, scr, lane); break;
    case 3: epi_frag_store<3>(acc, scr, lane); break;
    case 4: epi_frag_store<4>(acc, scr, lane); break;
    case 5: epi_frag_store<5>(acc, scr, lane); break;
    case 6: epi_frag_store<6>(acc, scr, lane); break;
    default: epi_frag_store<7>(acc, scr, lane); break;
  }
  __syncwarp();
  const float4* src = reinterpret_cast<const float4*>(scr + (lane & 15) * kEpiScratchPitch + 16 * (lane >> 4));
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 f = src[k];
    r[4 * k + 0] = __float_as_uint(f.x);
    r[4 * k + 1] = __float_as_uint(f.y);
    r[4 * k + 2] = __float_as_uint(f.z);
    r[4 * k + 3] = __float_as_uint(f.w);
  }
}

// One lane's 16 channels (column `col` of N tile `nt`) of pixel px.  kEpi (chosen per plan, conv_epi_class): generic
// (run time), or a plain class -- SiLU / ReLU / SiLU + shortcut / fp32 head -- folded at compile time.
template <int kEpi>
__device__ __forceinline__ void epi_unit(const ConvKParams& kp, const EpiPix& px, bool pool_writer, int nt, int col,
                                         uint32_t (&r)[16], const float* __restrict__ sbias, bool fast,
                                         float (&hacc)[8]) {
  constexpr bool kSpec = kEpi != PB_EPI_GENERIC;
  const int ch = nt * kp.BN + col;  // output channel of r[0]
  int cout_n = kp.cout_store - nt * kp.BN;  // channels of this N tile that exist
  cout_n = cout_n < kp.BN ? cout_n : kp.BN;
  const bool exists = col < cout_n;
  if (fast) {
    const int act = (kEpi == PB_EPI_SILU || kEpi == PB_EPI_SILU_RES) ? PB_ACT_SILU
                    : kEpi == PB_EPI_RELU                            ? PB_ACT_RELU
                    : kEpi == PB_EPI_F32                             ? PB_ACT_NONE
                                                                     : kp.act;
    const int has_res = kEpi == PB_EPI_SILU_RES ? 1 : kSpec ? 0 : (kp.res != nullptr ? (kp.res_first ? 2 : 1) : 0);
    const bool plain_silu = kSpec ? false : (kp.dbg_flags & 1) != 0;
    EpiOut eo;
    eo.mode = kSpec ? (kEpi == PB_EPI_F32 ? PB_OUT_F32_NHWC : PB_OUT_F16_NHWC) : kp.out_mode;
    eo.mode2 = kSpec ? PB_OUT2_NONE : kp.out2_mode;
    eo.pool_writer = pool_writer;
    eo.dx = eo.dy = eo.dx2 = eo.dy2 = 0;
    const size_t esz = eo.mode == PB_OUT_F32_NHWC ? 4 : 2;
    const size_t pxb = (size_t)kp.out_C * esz;  // bytes per output pixel
    const size_t up_pix = ((size_t)px.n * (2 * kp.Ho) + 2 * px.oh) * (2 * kp.Wo) + 2 * px.ow;
    size_t opix = px.pix;
    if (eo.mode == PB_OUT_F16_NHWC_UP2) {
      opix = up_pix;
      eo.dx = pxb;
      eo.dy = (size_t)(2 * kp.Wo) * pxb;
    }
    char* op = reinterpret_cast<char*>(kp.out) + opix * pxb + (size_t)(kp.out_coff + ch) * esz;
    char* op2 = nullptr;
    if (eo.mode2 != PB_OUT2_NONE) {
      const size_t pxb2 = (size_t)kp.out2_C * 2;
      size_t pix2;
      if (eo.mode2 == PB_OUT2_UP2) {
        pix2 = up_pix;
        eo.dx2 = pxb2;
        eo.dy2 = (size_t)(2 * kp.Wo) * pxb2;
      } else {  // POOL2 (Ho, Wo even): the pooled pixel of the window whose top-left corner this lane holds
        pix2 = ((size_t)px.n * (kp.Ho >> 1) + (px.oh >> 1)) * (kp.Wo >> 1) + (px.ow >> 1);
      }
      op2 = reinterpret_cast<char*>(kp.out2) + pix2 * pxb2 + (size_t)(kp.out2_coff + ch) * 2;
    }
    const bool valid = px.valid && exists;
    uint4 rv[2] = {};
    if (has_res && valid) {
      const uint4* rp = reinterpret_cast<const uint4*>(kp.res + px.pix * kp.res_C + kp.res_coff + ch);
      rv[0] = __ldg(rp);
      rv[1] = __ldg(rp + 1);
    }
    epi_chunk(act, has_res, plain_silu, eo, r, sbias + col, op, rv, valid, cout_n - col, op2, kEpi == PB_EPI_F32);
  } else if constexpr (kEpi == PB_EPI_GENERIC) {
    if (px.valid && exists) {
      float v[16];
      bias_act16(r, sbias + col, kp.act, v,
                 (kp.res && kp.res_first) ? kp.res + px.pix * kp.res_C + kp.res_coff + ch : nullptr);
      epilogue_store16(kp, px, ch, col, v, hacc);
    }
  }
}

// One consumer warp's tile; pix_of(j, pool_writer) = this lane's pixel in sub-tile j.  Every lane runs every chunk
// (the butterfly shuffles); the fused head adds the half-pixel sums of lanes l and l ^ 16.
// kS / kNch > 0: sub-tiles / 32-column chunks per sub-tile known at compile time (the halo kernel) -- both loops unroll
// and every accumulator index is a constant; 0: taken from S / kp.BN at run time (the per-tap kernel).
template <int kEpi, int kS = 0, int kNch = 0, int kAcc, typename PixOf>
__device__ __forceinline__ void epilogue_tile(const ConvKParams& kp, const float (&acc)[kAcc], int S, int nt,
                                              const float* __restrict__ sbias, float* scr, int lane, PixOf pix_of) {
  const int nch = kNch > 0 ? kNch : (kp.BN + 31) >> 5;
  const bool fast = kEpi != PB_EPI_GENERIC || epilogue_fast_ok(kp);  // the host picks a plain class only when it holds
  const int col0 = 16 * (lane >> 4);
  auto sub_tile = [&](int j) {
    bool pool_writer = false;
    const EpiPix px = pix_of(j, pool_writer);
    float hacc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // fused 1x1 head partial sums
    auto chunk = [&](int c) {
      uint32_t r[16];
      epi_transpose16(acc, j * nch + c, scr, lane, r);
      epi_unit<kEpi>(kp, px, pool_writer, nt, 32 * c + col0, r, sbias, fast, hacc);
    };
    if constexpr (kNch > 0) {
#pragma unroll
      for (int c = 0; c < kNch; ++c) chunk(c);
    } else {
      for (int c = 0; c < nch; ++c) chunk(c);
    }
    if (kEpi == PB_EPI_GENERIC && !fast && kp.head_n > 0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) hacc[q] += __shfl_xor_sync(0xffffffffu, hacc[q], 16);
      if (lane < 16 && px.valid) {
        const size_t plane = (size_t)kp.Ho * kp.Wo;
        float* ho = kp.head_out + (size_t)px.n * kp.head_n * plane + (size_t)px.oh * kp.Wo + px.ow;
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (q < kp.head_n) ho[(size_t)q * plane] = __fdividef(1.f, 1.f + __expf(-(hacc[q] + __ldg(kp.head_b + q))));
      }
    }
  };
  if constexpr (kS > 0) {
#pragma unroll
    for (int j = 0; j < kS; ++j) sub_tile(j);
  } else {
    for (int j = 0; j < S; ++j) sub_tile(j);
  }
}

// acc (+)= A * B^T over kSteps k-steps of 16 for the warpgroup's 64 rows of kS sub-tiles (A descriptors sub_units
// apart); accum = 0 overwrites.  kN = the N tile, a compile-time constant of the instruction.
template <int kN, int kS, int kSteps, int kAcc>
__device__ __forceinline__ void mma_n(float (&acc)[kAcc], uint64_t ad, uint64_t sub_units, uint64_t bd,
                                      uint32_t accum) {
  constexpr int kAS = (kN + 31) / 32 * 16;
  if constexpr (kS * kAS <= kAcc) {
#pragma unroll
    for (int j = 0; j < kS; ++j)
#pragma unroll
      for (int k = 0; k < kSteps; ++k)
        wgmma_f16<kN>(acc + j * kAS, ad + (uint64_t)j * sub_units + (uint64_t)(2 * k), bd + (uint64_t)(2 * k),
                      k == 0 ? accum : 1u);
  }
}
template <int kS, int kSteps>
__device__ __forceinline__ void mma_group(int n, float (&acc)[kConvAccRegs], uint64_t ad, uint64_t sub_units,
                                          uint64_t bd, uint32_t accum) {
  switch (n) {  // CTA-uniform
#define PB_MMA_CASE(n_) \
  case n_: mma_n<n_, kS, kSteps>(acc, ad, sub_units, bd, accum); break;
    PB_MMA_CASE(16) PB_MMA_CASE(32) PB_MMA_CASE(48) PB_MMA_CASE(64) PB_MMA_CASE(80) PB_MMA_CASE(96)
    PB_MMA_CASE(112) PB_MMA_CASE(128) PB_MMA_CASE(144) PB_MMA_CASE(160) PB_MMA_CASE(176) PB_MMA_CASE(192)
    PB_MMA_CASE(208) PB_MMA_CASE(224) PB_MMA_CASE(240) PB_MMA_CASE(256)
#undef PB_MMA_CASE
    default: break;
  }
}

// Consumer warps release a shared-memory slot once their wgmmas reading it have completed (one arrive per warp).
__device__ __forceinline__ void consumer_release(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

}  // namespace pb
