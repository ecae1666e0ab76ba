// YOLOv8 Detect/Pose head decode + per-image NMS on device.
// Restates ultralytics' Detect._inference / Pose.kpts_decode / ops.non_max_suppression ([3P], SURVEY App. A.3-A.4),
// which the reference reaches through model.predict() at
//   /root/reference/trackers/players_tracker/players_tracker.py:351-359
//   /root/reference/trackers/players_keypoints_tracker/players_keypoints_tracker.py:285-292
//   /root/reference/trackers/keypoints_tracker/keypoints_tracker.py:238-245
#include "internal.h"

namespace pb {

constexpr int kMaxLevels = 4;
struct DecodeParams {
  const float* feat[kMaxLevels];
  int h[kMaxLevels], w[kMaxLevels], stride[kMaxLevels], start[kMaxLevels + 1];
  int nlevels, B, fC, nc, nk, kdim, cap, rowlen, cls_off, kpt_off;
  int filter;                      // 1: keep only classes whose bit is set in class_mask
  unsigned long long class_mask[4];  // classes 0..255
  float conf;
};

__device__ __forceinline__ float sigmoidf_precise(float x) { return 1.0f / (1.0f + expf(-x)); }

// Lowest logit whose float sigmoid can equal `score` (sigmoidf_precise is within 6 * 2^-24 of sigmoid, relative).
// Below 0.999 the log-sigmoid falls by at least (1 - score) per unit logit, so a logit 2^-19 / (1 - score) lower
// is more than 12 * 2^-24 below `score`, relative; at 0.999 and above only logits > 6.9 reach it.
__device__ __forceinline__ float lowest_tying_logit(float best, float score) {
  return score > 0.999f ? 6.0f : best - 0x1p-19f / (1.0f - score);
}

// One thread per (image, anchor): threshold on the best class first, decode box/keypoints only for candidates.
__global__ void yolo_decode_kernel(DecodeParams p, float* __restrict__ cand, int* __restrict__ cand_anchor,
                                   int* __restrict__ cand_count) {
  const int A = p.start[p.nlevels];
  const long total = (long)p.B * A;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int a = (int)(i % A);
    const int b = (int)(i / A);
    int l = 0;
    while (l + 1 < p.nlevels && a >= p.start[l + 1]) ++l;
    const int la = a - p.start[l];
    const int gx = la % p.w[l], gy = la / p.w[l];
    const float* f = p.feat[l] + ((size_t)b * p.h[l] * p.w[l] + la) * p.fC;
    // best class: the score is the sigmoid of the largest logit (sigmoid is monotonic); `before` is the largest
    // logit of the classes ahead of it
    const float* fc = f + p.cls_off;
    float best = fc[0], before = -INFINITY;
    int bj = 0;
    for (int j = 1; j < p.nc; ++j) {
      const float v = fc[j];
      if (v > best) {
        before = best;
        best = v;
        bj = j;
      }
    }
    const float score = sigmoidf_precise(best);
    if (!(score > p.conf)) continue;
    // ultralytics takes the first maximum of the float sigmoids (torch.max), not of the logits: above a logit of ~16.6
    // every sigmoid is 1.0f, so an earlier, smaller saturated logit wins.  Rescanned only when an earlier logit is
    // close enough to tie: an unconditional rescan (an expf per class for every anchor that passes conf) made the
    // YOLOv8n-detect decode at 384x640, batch 32, 20 % slower (40 -> 48 us on an H100 80GB HBM3 at 700 W).
    const float lo = lowest_tying_logit(best, score);
    if (before >= lo) {
      for (int j = 0; j < bj; ++j) {
        if (fc[j] >= lo && sigmoidf_precise(fc[j]) == score) {
          bj = j;
          break;
        }
      }
    }
    if (p.filter && !((p.class_mask[(bj >> 6) & 3] >> (bj & 63)) & 1ull)) continue;
    // DFL: softmax over 16 bins, expectation with arange(16)
    float dist[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const float* q = f + s * 16;
      float mx = q[0];
#pragma unroll
      for (int j = 1; j < 16; ++j) mx = fmaxf(mx, q[j]);
      float den = 0.f, num = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float e = expf(q[j] - mx);
        den += e;
        num += e * (float)j;
      }
      dist[s] = num / den;
    }
    const float ax = (float)gx + 0.5f, ay = (float)gy + 0.5f;
    const float st = (float)p.stride[l];
    // dist2bbox(xywh=True) * stride, then xywh2xyxy (same float op order as ultralytics)
    const float x1 = ax - dist[0], y1 = ay - dist[1], x2 = ax + dist[2], y2 = ay + dist[3];
    const float cx = ((x1 + x2) / 2.f) * st, cy = ((y1 + y2) / 2.f) * st;
    const float bw = (x2 - x1) * st, bh = (y2 - y1) * st;
    const float hw = bw / 2.f, hh = bh / 2.f;
    const int slot = atomicAdd(cand_count + b, 1);
    if (slot >= p.cap) continue;  // host checks cand_count <= cap
    float* row = cand + ((size_t)b * p.cap + slot) * p.rowlen;
    row[0] = cx - hw;
    row[1] = cy - hh;
    row[2] = cx + hw;
    row[3] = cy + hh;
    row[4] = score;
    row[5] = (float)bj;
    const float* kp = f + p.kpt_off;
    const int K = p.kdim > 0 ? p.nk / p.kdim : 0;
    for (int k = 0; k < K; ++k) {
      const float vx = kp[k * p.kdim], vy = kp[k * p.kdim + 1];
      row[6 + k * p.kdim] = (vx * 2.0f + (ax - 0.5f)) * st;
      row[6 + k * p.kdim + 1] = (vy * 2.0f + (ay - 0.5f)) * st;
      if (p.kdim == 3) row[6 + k * 3 + 2] = sigmoidf_precise(kp[k * 3 + 2]);
    }
    cand_anchor[(size_t)b * p.cap + slot] = a;
  }
}

// One block per image: bitonic sort of (conf desc, anchor asc) keys, then greedy NMS.
// Working set per candidate: box float4 | key u64 | slot u32 | suppressed u8 (the float4 array first, so it is
// 16-byte aligned for any P).  Images with at most kNmsSmemCap
// candidates (every realistic frame) keep it in shared memory; beyond that -- ultralytics runs NMS on up to
// max_nms = 30000 candidates -- the same code runs on a global scratch area (L2 resident), P = pow2 >= cap entries.
constexpr int kNmsSmemCap = 4096;
__global__ void __launch_bounds__(1024)
yolo_nms_kernel(const float* __restrict__ cand, const int* __restrict__ cand_anchor,
                const int* __restrict__ cand_count, int cap, int P, int rowlen, float iou_thr, int max_det,
                float* __restrict__ out, int* __restrict__ out_count, uint8_t* __restrict__ scratch) {
  extern __shared__ __align__(16) uint8_t nms_smem[];
  __shared__ int kept_n;
  const int b = blockIdx.x;
  int n = cand_count[b];
  if (n > cap) n = cap;
  uint8_t* base = nms_smem;
  int Pl = kNmsSmemCap < P ? kNmsSmemCap : P;
  if (n > kNmsSmemCap) {  // block-uniform
    base = scratch + (size_t)b * P * 32;
    Pl = P;
  }
  float4* boxes = reinterpret_cast<float4*>(base);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(boxes + Pl);
  unsigned* slots = reinterpret_cast<unsigned*>(keys + Pl);
  uint8_t* supp = reinterpret_cast<uint8_t*>(slots + Pl);
  const float* cb = cand + (size_t)b * cap * rowlen;
  const int* ab = cand_anchor + (size_t)b * cap;
  int Pe = 1;  // sort only the power of two covering this image's candidates
  while (Pe < n) Pe <<= 1;
  for (int i = threadIdx.x; i < Pe; i += blockDim.x) {
    if (i < n) {
      const unsigned cbits = __float_as_uint(cb[(size_t)i * rowlen + 4]);  // conf in (0,1): bits are monotonic
      keys[i] = ((unsigned long long)cbits << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)ab[i]);
      slots[i] = (unsigned)i;
    } else {
      keys[i] = 0ull;
      slots[i] = 0xFFFFFFFFu;
    }
  }
  if (threadIdx.x == 0) kept_n = 0;
  __syncthreads();
  // bitonic sort, descending
  for (int k = 2; k <= Pe; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < Pe; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool desc = ((i & k) == 0);
          const unsigned long long a = keys[i], c = keys[ixj];
          if (desc ? (a < c) : (a > c)) {
            keys[i] = c;
            keys[ixj] = a;
            const unsigned t = slots[i];
            slots[i] = slots[ixj];
            slots[ixj] = t;
          }
        }
      }
      __syncthreads();
    }
  }
  // class-offset boxes in sorted order (boxes + cls*7680, agnostic=False)
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float* r = cb + (size_t)slots[i] * rowlen;
    const float c = r[5] * 7680.0f;
    boxes[i] = make_float4(r[0] + c, r[1] + c, r[2] + c, r[3] + c);
    supp[i] = 0;
  }
  __syncthreads();
  float* ob = out + (size_t)b * max_det * rowlen;
  for (int i = 0; i < n; ++i) {
    if (supp[i]) continue;  // uniform across the block (read after the barrier of the previous iteration)
    const int k = kept_n;
    if (k >= max_det) break;
    const float4 bi = boxes[i];
    // torchvision's float op order, each product rounded on its own: a fused iarea + w_j * h_j moves IoUs across
    // the threshold.  iou_thr is the largest float <= the double threshold, so ovr > iou_thr is torchvision's
    // (double)ovr > iou.
    const float iarea = __fmul_rn(bi.z - bi.x, bi.w - bi.y);
    for (int j = i + 1 + threadIdx.x; j < n; j += blockDim.x) {
      if (supp[j]) continue;
      const float4 bj = boxes[j];
      const float xx1 = fmaxf(bi.x, bj.x), yy1 = fmaxf(bi.y, bj.y);
      const float xx2 = fminf(bi.z, bj.z), yy2 = fminf(bi.w, bj.w);
      const float w = fmaxf(0.f, xx2 - xx1), h = fmaxf(0.f, yy2 - yy1);
      const float inter = __fmul_rn(w, h);
      const float ovr = inter / ((iarea + __fmul_rn(bj.z - bj.x, bj.w - bj.y)) - inter);
      if (ovr > iou_thr) supp[j] = 1;
    }
    // emit row k = candidate slots[i]
    const float* r = cb + (size_t)slots[i] * rowlen;
    for (int c = threadIdx.x; c < rowlen; c += blockDim.x) ob[(size_t)k * rowlen + c] = r[c];
    __syncthreads();
    if (threadIdx.x == 0) kept_n = k + 1;
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x == 0) out_count[b] = kept_n;
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb_yolo_decode(const pb_yolo_level* levels, int nlevels, int B, int fC, int nc, int nk, int kdim, int cls_off,
                   int kpt_off, float conf, const int* classes, int n_classes, float* cand, int* cand_anchor,
                   int* cand_count, int cap, void* stream) {
  PB_CHECK(levels && cand && cand_anchor && cand_count, "yolo_decode: null pointer");
  PB_CHECK(nlevels >= 1 && nlevels <= kMaxLevels, "yolo_decode: 1..%d levels", kMaxLevels);
  PB_CHECK(nc >= 1 && fC >= 64 + nc + nk, "yolo_decode: feature width %d < 64+nc+nk", fC);
  PB_CHECK(cls_off >= 64 && cls_off + nc <= fC && (nk == 0 || (kpt_off >= 64 && kpt_off + nk <= fC)),
           "yolo_decode: bad cls/kpt offsets");
  PB_CHECK(kdim == 0 || kdim == 2 || kdim == 3, "yolo_decode: kdim must be 0, 2 or 3");
  PB_CHECK(kdim == 0 ? nk == 0 : nk % kdim == 0, "yolo_decode: nk not a multiple of kdim");
  DecodeParams p;
  p.nlevels = nlevels; p.B = B; p.fC = fC; p.nc = nc; p.nk = nk; p.kdim = kdim;
  p.cap = cap; p.rowlen = 6 + nk; p.conf = conf;
  p.filter = classes != nullptr ? 1 : 0;
  for (int i = 0; i < 4; ++i) p.class_mask[i] = 0ull;
  PB_CHECK(classes == nullptr || nc <= 256, "yolo_decode: a class filter supports nc <= 256");
  for (int i = 0; classes != nullptr && i < n_classes; ++i) {
    PB_CHECK(classes[i] >= 0 && classes[i] < 256, "yolo_decode: class %d out of range", classes[i]);
    p.class_mask[classes[i] >> 6] |= 1ull << (classes[i] & 63);
  }
  p.cls_off = cls_off; p.kpt_off = kpt_off;
  p.start[0] = 0;
  for (int l = 0; l < nlevels; ++l) {
    p.feat[l] = levels[l].feat; p.h[l] = levels[l].h; p.w[l] = levels[l].w; p.stride[l] = levels[l].stride;
    p.start[l + 1] = p.start[l] + levels[l].h * levels[l].w;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PB_CUDA(cudaMemsetAsync(cand_count, 0, sizeof(int) * B, s));
  const long total = (long)B * p.start[nlevels];
  long blocks = (total + 127) / 128;
  if (blocks > (long)num_sms() * 32) blocks = (long)num_sms() * 32;
  yolo_decode_kernel<<<(int)blocks, 128, 0, s>>>(p, cand, cand_anchor, cand_count);
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

size_t pb_yolo_nms_scratch_bytes(int B, int cap) {
  if (cap <= kNmsSmemCap) return 0;
  size_t P = 1;
  while (P < (size_t)cap) P <<= 1;
  return (size_t)B * P * 32;
}

int pb_yolo_nms(const float* cand, const int* cand_anchor, const int* cand_count, int B, int cap, int rowlen,
                double iou, int max_det, float* out, int* out_count, void* scratch, void* stream) {
  PB_CHECK(cand && cand_anchor && cand_count && out && out_count, "yolo_nms: null pointer");
  // largest float <= iou: for a float IoU x, x > iou_thr exactly when (double)x > iou
  float iou_thr = (float)iou;
  if ((double)iou_thr > iou) iou_thr = nextafterf(iou_thr, -INFINITY);
  int P = 1;
  while (P < cap) P <<= 1;
  PB_CHECK(P <= 32768, "yolo_nms: candidate capacity %d > 32768 (ultralytics max_nms is 30000)", cap);
  PB_CHECK(cap <= kNmsSmemCap || scratch != nullptr, "yolo_nms: cap %d > %d needs a scratch buffer", cap, kNmsSmemCap);
  const size_t smem = (size_t)(P < kNmsSmemCap ? P : kNmsSmemCap) * (8 + 16 + 4 + 1);
  PB_CUDA((cudaError_t)ensure_dynamic_smem(reinterpret_cast<const void*>(yolo_nms_kernel), smem));
  yolo_nms_kernel<<<B, 1024, smem, static_cast<cudaStream_t>(stream)>>>(
      cand, cand_anchor, cand_count, cap, P, rowlen, iou_thr, max_det, out, out_count, static_cast<uint8_t*>(scratch));
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
