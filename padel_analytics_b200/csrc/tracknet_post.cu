// TrackNet post-processing on device:
//  * temporal ensemble of the 8 window predictions covering each frame + threshold
//      (/root/reference/trackers/ball_tracker/ball_tracker.py:421-437,449-509 ; get_ensemble_weight :68-97)
//  * heat-map -> bounding box of the largest 8-connected component
//      (/root/reference/trackers/ball_tracker/predict.py:7-39 : cv2.findContours(RETR_EXTERNAL) + boundingRect,
//       max w*h with strict '>' over cv2's contour order == the component whose first raster pixel comes last)
#include "internal.h"

namespace pb {

// One thread per (frame, pixel); the frames may belong to several clips.  desc[f] = (global window index of the
// frame's clip's window 0, that clip's window count, the frame's index in its clip); pred row r holds global window
// first_window + r.  Each frame reads only its own clip's windows and applies the head/tail rules of that clip.
__global__ void ensemble_rows_kernel(const float* __restrict__ pred, int first_window, const int* __restrict__ desc,
                                     int nframes, int HW, float thr, uint8_t* __restrict__ mask,
                                     float* __restrict__ ens) {
  const long total = (long)nframes * HW;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int pix = (int)(i % HW);
    const int* d = desc + (i / HW) * 3;
    const int base = __ldg(d) - first_window;  // pred row of the clip's window 0
    const int total_windows = __ldg(d + 1);
    const int n = __ldg(d + 2);  // frame index within the clip
    float acc = 0.f;
    float result;
    if (n < total_windows && n >= 7) {
      // general case: sum_k w[k] * P[n-7+k][7-k], w = [1,2,3,4,4,3,2,1]/20 (products first, then summed in k order)
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float wk = (float)(k < 4 ? k + 1 : 8 - k) / 20.0f;
        const int s = base + n - 7 + k;
        acc = __fadd_rn(acc, __fmul_rn(pred[((size_t)s * 8 + (7 - k)) * HW + pix], wk));  // mul, then add (no FMA)
      }
      result = acc;
    } else {
      // head (n < 7): mean over the n+1 windows that exist; tail (n >= total_windows): divisor 8 - frame_i
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int w = n - 7 + k;
        if (w >= 0 && w < total_windows) acc += pred[((size_t)(base + w) * 8 + (7 - k)) * HW + pix];
      }
      const float div = (n < total_windows) ? (float)(n + 1) : (float)(8 - (n - (total_windows - 1)));
      result = acc / div;
    }
    mask[i] = result > thr ? 1 : 0;
    if (ens) ens[i] = result;
  }
}

// The ensemble of frames whose windows are named by a table: the frames may belong to several interleaved live
// streams, each with its own carried windows.  table[f] = (ref[0..7], rule): ref[k] is the heat-map row of window
// n-7+k of frame f's stream (its channel 7-k is read): a row of the carry pool when < carry_rows, row ref - carry_rows
// of this batch's fresh rows otherwise, or -1 when the window does not exist.  rule 0: the weighted sum of the 8
// windows; rule d > 0: the head/tail mean, the sum of the windows present divided by d.  The arithmetic is that of
// ensemble_rows_kernel term for term, so a stream's masks are bit-identical to the single-stream path.
__global__ void ensemble_table_kernel(const float* __restrict__ carry, int carry_rows, const float* __restrict__ fresh,
                                      const int* __restrict__ table, int nframes, int HW, float thr,
                                      uint8_t* __restrict__ mask, float* __restrict__ ens) {
  const long total = (long)nframes * HW;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int pix = (int)(i % HW);
    const int* t = table + (i / HW) * 9;
    const int rule = __ldg(t + 8);
    float acc = 0.f;
    float result;
    if (rule == 0) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float wk = (float)(k < 4 ? k + 1 : 8 - k) / 20.0f;
        const int r = __ldg(t + k);
        if (r < 0) continue;  // never planned: an absent window adds nothing rather than reading out of bounds
        const float* row = r < carry_rows ? carry + (size_t)r * 8 * HW : fresh + (size_t)(r - carry_rows) * 8 * HW;
        acc = __fadd_rn(acc, __fmul_rn(row[(size_t)(7 - k) * HW + pix], wk));  // mul, then add (no FMA)
      }
      result = acc;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int r = __ldg(t + k);
        if (r >= 0) {
          const float* row = r < carry_rows ? carry + (size_t)r * 8 * HW : fresh + (size_t)(r - carry_rows) * 8 * HW;
          acc += row[(size_t)(7 - k) * HW + pix];
        }
      }
      result = acc / (float)rule;
    }
    mask[i] = result > thr ? 1 : 0;
    if (ens) ens[i] = result;
  }
}

// carry[copies[2c]] = fresh[copies[2c + 1]]: whole (8, H, W) heat-map rows, 16 bytes per thread.
__global__ void carry_rows_kernel(float4* __restrict__ carry, const float4* __restrict__ fresh,
                                  const int* __restrict__ copies, int ncopies, long row_vec) {
  const long total = (long)ncopies * row_vec;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i / row_vec);
    const long e = i % row_vec;
    const size_t dst = (size_t)__ldg(copies + 2 * c) * row_vec, src = (size_t)__ldg(copies + 2 * c + 1) * row_vec;
    carry[dst + e] = __ldcs(fresh + src + e);
  }
}

__device__ __forceinline__ int uf_find(const int* parent, int i) {
  int p = __ldcg(parent + i);
  while (p != i) {
    i = p;
    p = __ldcg(parent + i);
  }
  return i;
}
__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(parent + a, b);  // link the larger root under the smaller one
    if (old == a) return;
    a = old;
  }
}

// One block per frame. scratch per frame: parent, xmin, xmax, ymin, ymax (int32 [H*W] each).
// The mask is scanned 16 bytes at a time (it is almost entirely zero); only foreground pixels touch the scratch.
template <typename F>
__device__ __forceinline__ void for_each_fg(const uint8_t* __restrict__ m, int HW, F f) {
  const int nvec = HW >> 4;
  const uint4* mv = reinterpret_cast<const uint4*>(m);
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint4 q = mv[v];
    if ((q.x | q.y | q.z | q.w) == 0u) continue;
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (w[k] == 0u) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if ((w[k] >> (8 * j)) & 0xFFu) f(v * 16 + k * 4 + j);
    }
  }
  for (int i = (nvec << 4) + threadIdx.x; i < HW; i += blockDim.x)
    if (m[i]) f(i);
}

__global__ void __launch_bounds__(1024) ccl_bbox_kernel(const uint8_t* __restrict__ mask, int H, int W,
                                                        int* __restrict__ scratch, int* __restrict__ bbox) {
  const int HW = H * W;
  const int f = blockIdx.x;
  const uint8_t* m = mask + (size_t)f * HW;
  int* parent = scratch + (size_t)f * 5 * HW;
  int* xmin = parent + HW;
  int* xmax = xmin + HW;
  int* ymin = xmax + HW;
  int* ymax = ymin + HW;
  __shared__ unsigned long long best;
  __shared__ int any;
  if (threadIdx.x == 0) {
    best = 0ull;
    any = 0;
  }
  __syncthreads();
  int mine = 0;
  for_each_fg(m, HW, [&](int i) {
    parent[i] = i;
    xmin[i] = W;
    xmax[i] = -1;
    ymin[i] = H;
    ymax[i] = -1;
    mine = 1;
  });
  if (mine) any = 1;
  __threadfence_block();
  __syncthreads();
  if (!any) {
    if (threadIdx.x < 4) bbox[f * 4 + threadIdx.x] = 0;
    return;
  }
  for_each_fg(m, HW, [&](int i) {
    const int x = i % W, y = i / W;
    if (x > 0 && m[i - 1]) uf_union(parent, i, i - 1);
    if (y > 0) {
      if (m[i - W]) uf_union(parent, i, i - W);
      if (x > 0 && m[i - W - 1]) uf_union(parent, i, i - W - 1);
      if (x < W - 1 && m[i - W + 1]) uf_union(parent, i, i - W + 1);
    }
  });
  __threadfence_block();
  __syncthreads();
  for_each_fg(m, HW, [&](int i) {
    const int r = uf_find(parent, i);
    const int x = i % W, y = i / W;
    atomicMin(xmin + r, x);
    atomicMax(xmax + r, x);
    atomicMin(ymin + r, y);
    atomicMax(ymax + r, y);
  });
  __threadfence_block();
  __syncthreads();
  for_each_fg(m, HW, [&](int i) {
    if (__ldcg(parent + i) != i) return;
    const int w = __ldcg(xmax + i) - __ldcg(xmin + i) + 1, h = __ldcg(ymax + i) - __ldcg(ymin + i) + 1;
    const unsigned long long key = ((unsigned long long)(unsigned)(w * h) << 32) | (unsigned)i;
    atomicMax(&best, key);  // max area; ties -> largest root index (latest first pixel in raster order)
  });
  __syncthreads();
  if (threadIdx.x == 0) {
    const int r = (int)(best & 0xffffffffull);
    bbox[f * 4 + 0] = __ldcg(xmin + r);
    bbox[f * 4 + 1] = __ldcg(ymin + r);
    bbox[f * 4 + 2] = __ldcg(xmax + r) - __ldcg(xmin + r) + 1;
    bbox[f * 4 + 3] = __ldcg(ymax + r) - __ldcg(ymin + r) + 1;
  }
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb_tracknet_ensemble_rows(const float* pred, int first_window, const int* desc, int nframes, int H, int W,
                              float thr, uint8_t* mask, float* ens, void* stream) {
  PB_CHECK(pred && desc && mask, "ensemble_rows: null pointer");
  PB_CHECK((reinterpret_cast<uintptr_t>(desc) & 3) == 0, "ensemble_rows: desc must be 4-byte aligned");
  if (nframes <= 0) return 0;
  const long total = (long)nframes * H * W;
  long blocks = (total + 255) / 256;
  if (blocks > (long)num_sms() * 32) blocks = (long)num_sms() * 32;
  ensemble_rows_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      pred, first_window, desc, nframes, H * W, thr, mask, ens);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int pb_tracknet_ensemble_table(const float* carry, int carry_rows, const float* fresh, const int* table, int nframes,
                               int H, int W, float thr, uint8_t* mask, float* ens, void* stream) {
  PB_CHECK(carry && fresh && table && mask, "ensemble_table: null pointer");
  PB_CHECK((reinterpret_cast<uintptr_t>(table) & 3) == 0, "ensemble_table: table must be 4-byte aligned");
  if (nframes <= 0) return 0;
  const long total = (long)nframes * H * W;
  long blocks = (total + 255) / 256;
  if (blocks > (long)num_sms() * 32) blocks = (long)num_sms() * 32;
  ensemble_table_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      carry, carry_rows, fresh, table, nframes, H * W, thr, mask, ens);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int pb_tracknet_carry_rows(float* carry, const float* fresh, const int* copies, int ncopies, int H, int W,
                           void* stream) {
  PB_CHECK(carry && fresh && copies, "carry_rows: null pointer");
  PB_CHECK(((reinterpret_cast<uintptr_t>(carry) | reinterpret_cast<uintptr_t>(fresh)) & 15) == 0,
           "carry_rows: carry and fresh must be 16-byte aligned");
  if (ncopies <= 0) return 0;
  const long row_vec = (long)8 * H * W / 4;
  const long total = (long)ncopies * row_vec;
  long blocks = (total + 255) / 256;
  if (blocks > (long)num_sms() * 32) blocks = (long)num_sms() * 32;
  carry_rows_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float4*>(carry), reinterpret_cast<const float4*>(fresh), copies, ncopies, row_vec);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int pb_ccl_bbox(const uint8_t* mask, int nframes, int H, int W, int* scratch, int* bbox, void* stream) {
  PB_CHECK(mask && scratch && bbox, "ccl: null pointer");
  PB_CHECK((H * W) % 16 == 0 && (reinterpret_cast<uintptr_t>(mask) & 15) == 0, "ccl: H*W must be a multiple of 16");
  if (nframes <= 0) return 0;
  ccl_bbox_kernel<<<nframes, 1024, 0, static_cast<cudaStream_t>(stream)>>>(mask, H, W, scratch, bbox);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
