// The pieces of torchvision's ResNet50 that are not 1x1 / 3x3 convolutions -- the court-keypoint regressor of
// /root/reference/trackers/keypoints_tracker/keypoints_tracker.py:158-167 (model) and :276-312 (forward + sigmoid),
// input pipeline keypoints_tracker/iterable.py:10-41:
//   * ToTensor + Normalize(mean, std) of the resized RGB frame            -> pb_u8_normalize_f16
//   * conv1 7x7 / stride 2 / pad 3 (3 -> 64) + BN + ReLU                   -> pb_resnet_stem7x7
//   * MaxPool2d(3, stride 2, padding 1)                                    -> pb_maxpool3x3s2
//   * AdaptiveAvgPool2d(1) + Linear(2048 -> n_out) + Sigmoid               -> pb_avgpool_fc_sigmoid
// The bottleneck stacks run on the wgmma conv kernels (res_before_act = 1, 1x1 stride-2 downsample convs).
// These four are 0.24 of the network's 4.1 GFLOP per frame; CUDA-core code, HBM / FMA bound.
#include "internal.h"
#include "ptx.cuh"

namespace pb {

// u8 (B,H,W,3) -> half (B,H,W,4): ((x / 255) - mean[c]) / std[c] in fp32 (ToTensor, Normalize), channel 3 = 0
__global__ void u8_normalize_kernel(const uint8_t* __restrict__ src, long npix, float m0, float m1, float m2, float s0,
                                    float s1, float s2, __half* __restrict__ dst) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < npix; i += (long)gridDim.x * blockDim.x) {
    const uint8_t* p = src + i * 3;
    const float a = ((float)p[0] / 255.0f - m0) / s0;
    const float b = ((float)p[1] / 255.0f - m1) / s1;
    const float c = ((float)p[2] / 255.0f - m2) / s2;
    __half2* o = reinterpret_cast<__half2*>(dst + i * 4);
    o[0] = __floats2half2_rn(a, b);
    o[1] = __floats2half2_rn(c, 0.f);
  }
}

// conv 7x7 / s2 / p3, 3 -> 64, + bias + ReLU.  in half (B,H,W,4), w float [7*7*3][64] (k = (r*7 + s)*3 + c), out half
// NHWC (B,H/2,W/2,64).  Block = 16 x 8 output pixels, one thread per pixel with all 64 accumulators; the 37 x 21 x 3
// input patch and the 147 x 64 weights live in shared memory (weights are read as warp-wide broadcasts).
constexpr int kStemTW = 16, kStemTH = 8;
__global__ void __launch_bounds__(kStemTW* kStemTH) resnet_stem7x7_kernel(const __half* __restrict__ in, int H, int W,
                                                                          const float* __restrict__ w,
                                                                          const float* __restrict__ bias,
                                                                          __half* __restrict__ out) {
  constexpr int PW = kStemTW * 2 + 5, PH = kStemTH * 2 + 5;
  __shared__ float sw[147 * 64];
  __shared__ float sin[PH * PW * 3];
  const int Ho = H / 2, Wo = W / 2;
  const int n = blockIdx.z, ty = blockIdx.y * kStemTH, tx = blockIdx.x * kStemTW;
  for (int i = threadIdx.x; i < 147 * 64; i += blockDim.x) sw[i] = w[i];
  const int iy0 = ty * 2 - 3, ix0 = tx * 2 - 3;
  for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
    const int py = i / PW, px = i - py * PW;
    const int iy = iy0 + py, ix = ix0 + px;
    float a = 0.f, b = 0.f, c = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const __half2* p = reinterpret_cast<const __half2*>(in + (((size_t)n * H + iy) * W + ix) * 4);
      const float2 ab = __half22float2(p[0]);
      a = ab.x;
      b = ab.y;
      c = __low2float(p[1]);
    }
    sin[i * 3 + 0] = a;
    sin[i * 3 + 1] = b;
    sin[i * 3 + 2] = c;
  }
  __syncthreads();
  const int lx = threadIdx.x % kStemTW, ly = threadIdx.x / kStemTW;
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = bias[c];
  for (int r = 0; r < 7; ++r) {
    for (int s = 0; s < 7; ++s) {
      const float* ip = sin + ((ly * 2 + r) * PW + (lx * 2 + s)) * 3;
      const float x0 = ip[0], x1 = ip[1], x2 = ip[2];
      const float4* w0 = reinterpret_cast<const float4*>(sw + ((r * 7 + s) * 3 + 0) * 64);
      const float4* w1 = w0 + 16;
      const float4* w2 = w0 + 32;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const float4 a = w0[q], b = w1[q], c = w2[q];
        acc[4 * q + 0] = fmaf(x0, a.x, fmaf(x1, b.x, fmaf(x2, c.x, acc[4 * q + 0])));
        acc[4 * q + 1] = fmaf(x0, a.y, fmaf(x1, b.y, fmaf(x2, c.y, acc[4 * q + 1])));
        acc[4 * q + 2] = fmaf(x0, a.z, fmaf(x1, b.z, fmaf(x2, c.z, acc[4 * q + 2])));
        acc[4 * q + 3] = fmaf(x0, a.w, fmaf(x1, b.w, fmaf(x2, c.w, acc[4 * q + 3])));
      }
    }
  }
  const int oy = ty + ly, ox = tx + lx;
  if (oy < Ho && ox < Wo) {
    uint4* op = reinterpret_cast<uint4*>(out + (((size_t)n * Ho + oy) * Wo + ox) * 64);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      uint4 v;
      __half2* h2 = reinterpret_cast<__half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        h2[j] = __floats2half2_rn(fmaxf(acc[8 * g + 2 * j], 0.f), fmaxf(acc[8 * g + 2 * j + 1], 0.f));
      op[g] = v;
    }
  }
}

__device__ __forceinline__ uint4 hmax8v(uint4 a, uint4 b) {
  uint4 r;
  const __half2* x = reinterpret_cast<const __half2*>(&a);
  const __half2* y = reinterpret_cast<const __half2*>(&b);
  __half2* z = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) z[i] = __hmax2(x[i], y[i]);
  return r;
}

// MaxPool2d(kernel 3, stride 2, padding 1) on NHWC half, 8 channels per thread
__global__ void maxpool3x3s2_kernel(const __half* __restrict__ in, int N, int H, int W, int C, __half* __restrict__ out) {
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1, cg = C / 8;
  const long total = (long)N * Ho * Wo * cg;
  griddep_launch_dependents();
  griddep_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    long p = i / cg;
    const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho), n = (int)(p / ((long)Wo * Ho));
    uint4 m;
    bool first = true;
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int iy = oy * 2 + dy, ix = ox * 2 + dx;
        if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
        const uint4 v = *reinterpret_cast<const uint4*>(in + (((size_t)n * H + iy) * W + ix) * C + g * 8);
        m = first ? v : hmax8v(m, v);
        first = false;
      }
    *reinterpret_cast<uint4*>(out + (((size_t)n * Ho + oy) * Wo + ox) * C + g * 8) = m;
  }
}

// AdaptiveAvgPool2d(1) + Linear(C -> n_out) + Sigmoid: one block per image
__global__ void __launch_bounds__(256) avgpool_fc_sigmoid_kernel(const __half* __restrict__ in, int HW, int C,
                                                                 const float* __restrict__ w, const float* __restrict__ b,
                                                                 int n_out, float* __restrict__ out) {
  extern __shared__ float pooled[];  // C
  const int n = blockIdx.x;
  griddep_wait();
  const __half* base = in + (size_t)n * HW * C;
  for (int c8 = threadIdx.x; c8 < C / 8; c8 += blockDim.x) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int p = 0; p < HW; ++p) {
      const uint4 v = *reinterpret_cast<const uint4*>(base + (size_t)p * C + c8 * 8);
      const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) pooled[c8 * 8 + j] = acc[j] / (float)HW;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = warp; o < n_out; o += blockDim.x >> 5) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(pooled[c], w[(size_t)o * C + c], s);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (lane == 0) out[(size_t)n * n_out + o] = 1.f / (1.f + expf(-(s + b[o])));
  }
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb_u8_normalize_f16(const uint8_t* src, long long npix, const float* mean3, const float* std3, void* dst,
                        void* stream) {
  PB_CHECK(src && dst && mean3 && std3, "u8_normalize: null pointer");
  long blocks = (npix + 255) / 256;
  if (blocks > (long)num_sms() * 16) blocks = (long)num_sms() * 16;
  u8_normalize_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, (long)npix, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2], reinterpret_cast<__half*>(dst));
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int pb_resnet_stem7x7(const void* in, int N, int H, int W, const float* weight, const float* bias, void* out,
                      void* stream) {
  PB_CHECK(in && weight && bias && out, "resnet_stem: null pointer");
  PB_CHECK(H % 2 == 0 && W % 2 == 0, "resnet_stem: odd input size");
  dim3 grid((W / 2 + kStemTW - 1) / kStemTW, (H / 2 + kStemTH - 1) / kStemTH, N);
  resnet_stem7x7_kernel<<<grid, kStemTW * kStemTH, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(in), H, W, weight, bias, reinterpret_cast<__half*>(out));
  PB_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int pb_maxpool3x3s2(const void* in, int N, int H, int W, int C, void* out, void* stream) {
  PB_CHECK(in && out && C % 8 == 0, "maxpool3x3s2: bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  long blocks = ((long)N * Ho * Wo * (C / 8) + 255) / 256;
  if (blocks > (long)num_sms() * 16) blocks = (long)num_sms() * 16;
  PB_CUDA(launch_pdl(maxpool3x3s2_kernel, dim3((int)blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), 1,
                     reinterpret_cast<const __half*>(in), N, H, W, C, reinterpret_cast<__half*>(out)));
  count_launch();
  return 0;
}

int pb_avgpool_fc_sigmoid(const void* in, int N, int HW, int C, const float* weight, const float* bias, int n_out,
                          float* out, void* stream) {
  PB_CHECK(in && weight && bias && out && C % 8 == 0 && C <= 8192, "avgpool_fc: bad arguments");
  PB_CUDA(launch_pdl(avgpool_fc_sigmoid_kernel, dim3(N), dim3(256), (size_t)C * sizeof(float),
                     static_cast<cudaStream_t>(stream), 1, reinterpret_cast<const __half*>(in), HW, C, weight, bias, n_out,
                     out));
  count_launch();
  return 0;
}

}  // extern "C"
