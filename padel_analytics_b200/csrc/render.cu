// Overlay compositor of the render pass: applies a per-frame display list to uint8 BGR frames in place.
//
// The host turns every drawing call of a frame (cv2.circle / line / rectangle / putText, all LINE_8 and overwrite-
// only) into a STAMP record: the pixels the call covers, rasterised by cv2 itself on a small canvas, and one colour.
// The semi-transparent mini-court background is a BLEND record: every byte of a rectangle goes through a 256-entry
// table.  Records are applied in draw order, so overlaps resolve exactly as the sequential cv2 calls do.
//
// One CTA owns a band of kRows rows of one frame; warp w owns row band_lo + w.  The CTA walks its frame's records in
// order, skips those that miss its band, and __syncthreads() between the records it applies.  A row segment is
// processed as 16-byte chunks where they lie inside the segment, and byte by byte at its ragged ends, so no byte
// outside the record (and no byte of another CTA's row) is ever written.  Only covered rows are touched.
#include "internal.h"

namespace pb {

constexpr int kRows = 8;  // rows per CTA = warps per CTA

__device__ __forceinline__ uint8_t apply_byte(uint8_t v, int op, int px, int c, const uint8_t* sprite_row,
                                              uint32_t colour, const uint8_t* lut) {
  if (op == PB_OVERLAY_BLEND) return lut[v];
  return sprite_row[px] ? (uint8_t)(colour >> (8 * c)) : v;
}

__global__ void __launch_bounds__(kRows * 32) render_overlay_kernel(uint8_t* __restrict__ frames, int H, int W,
                                                                    const pb_overlay_rec* __restrict__ list,
                                                                    const int* __restrict__ offsets,
                                                                    const uint8_t* __restrict__ atlas,
                                                                    const uint8_t* __restrict__ blend_lut) {
  __shared__ uint8_t lut[256];
  const int f = blockIdx.y;
  const int band_lo = blockIdx.x * kRows, band_hi = min(band_lo + kRows, H);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = blend_lut[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int y = band_lo + warp;
  const long long row_bytes = 3LL * W;
  uint8_t* row = frames + ((long long)f * H + y) * row_bytes;
  const int r0 = offsets[f], r1 = offsets[f + 1];
  for (int r = r0; r < r1; ++r) {
    const pb_overlay_rec rec = list[r];
    // clip to the frame and to this band (uniform over the CTA)
    const int ry0 = max(max(rec.y0, 0), band_lo), ry1 = min(min(rec.y0 + rec.h, H), band_hi);
    const int rx0 = max(rec.x0, 0), rx1 = min(rec.x0 + rec.w, W);
    if (ry0 >= ry1 || rx0 >= rx1) continue;
    if (y >= ry0 && y < ry1) {
      const uint8_t* srow = rec.op == PB_OVERLAY_STAMP
                                ? atlas + rec.atlas_offset + (long long)(y - rec.y0) * rec.pitch - rec.x0
                                : nullptr;  // indexed by frame x
      const long long a = 3LL * rx0, b = 3LL * rx1;  // byte range within the row
      const uintptr_t base = reinterpret_cast<uintptr_t>(row);
      long long va = (long long)(((base + a + 15) & ~(uintptr_t)15) - base);
      long long vb = (long long)(((base + b) & ~(uintptr_t)15) - base);
      if (va > vb) va = vb = b;  // no whole chunk inside the segment: all bytes go the scalar way
      const int nv = (int)((vb - va) >> 4), head = (int)(va - a), tail = (int)(b - vb);
      for (int k = lane; k < nv; k += 32) {
        const long long off = va + 16LL * k;
        uint4 q = *reinterpret_cast<const uint4*>(row + off);
        uint8_t* bytes = reinterpret_cast<uint8_t*>(&q);
        int px = (int)(off / 3), c = (int)(off - 3LL * px);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          bytes[j] = apply_byte(bytes[j], rec.op, px, c, srow, rec.colour_bgr, lut);
          if (++c == 3) { c = 0; ++px; }
        }
        *reinterpret_cast<uint4*>(row + off) = q;
      }
      for (int k = lane; k < head + tail; k += 32) {
        const long long off = k < head ? a + k : vb + (k - head);
        const int px = (int)(off / 3), c = (int)(off - 3LL * px);
        row[off] = apply_byte(row[off], rec.op, px, c, srow, rec.colour_bgr, lut);
      }
    }
    __syncthreads();  // the next record may overlap this one: draw order
  }
}

}  // namespace pb

extern "C" int pb_render_overlay(uint8_t* frames, int B, int H, int W, const pb_overlay_rec* list,
                                 const int* list_offsets, const uint8_t* atlas, const uint8_t* blend_lut,
                                 void* stream) {
  using namespace pb;
  PB_CHECK(B >= 0 && H >= 1 && W >= 1, "render_overlay: B = %d, H = %d, W = %d", B, H, W);
  if (B == 0) return 0;
  PB_CHECK(frames && list_offsets && blend_lut, "render_overlay: null pointer");
  PB_CHECK(B <= 65535, "render_overlay: B = %d exceeds the grid's y limit", B);
  const dim3 grid((H + kRows - 1) / kRows, B);
  render_overlay_kernel<<<grid, kRows * 32, 0, static_cast<cudaStream_t>(stream)>>>(frames, H, W, list, list_offsets,
                                                                                   atlas, blend_lut);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
