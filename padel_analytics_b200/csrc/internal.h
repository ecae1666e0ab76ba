// Internal helpers shared by the translation units of libpadel_b200.so (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <string>

#include "../../include/padel_b200.h"

namespace pb {

void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int num_sms();
// Raise a kernel's dynamic shared-memory limit to at least `bytes` on the CURRENT device (the attribute is per device
// and per function; remembered per (device, function) so the driver call happens once).  Returns a cudaError_t.
int ensure_dynamic_smem(const void* func, size_t bytes);
// Programmatic dependent launch for the kernels of a program (PADEL_B200_PDL=0 disables; default on)
bool pdl_enabled();
int plan_pdl();  // the value a plan built now captures

#ifdef __CUDACC__
// Launch `kernel` with the programmatic-stream-serialization attribute (see ptx.cuh::griddep_wait): only for kernels
// that call griddep_wait() before touching data another kernel may have written / may still be reading.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                             int cluster, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (cluster > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = (unsigned)cluster;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = (unsigned)na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  return e == cudaSuccess ? cudaGetLastError() : e;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              int cluster, Args... args) {
  return launch_ex(kernel, grid, block, smem, stream, cluster, pdl_enabled(), args...);
}
#endif

#define PB_CHECK(cond, ...)         \
  do {                              \
    if (!(cond)) {                  \
      pb::set_error(__VA_ARGS__);   \
      return 1;                     \
    }                               \
  } while (0)

#define PB_CUDA(expr)                                                                          \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      pb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)

// ---- conv plan (built once per layer; holds TMA descriptors + launch geometry) -------------------------------
constexpr int kConvMaxStages = 12;
// Conv kernels: warpgroup 0 = TMA producers (w0 activations, w1 weights), warpgroups 1-2 = wgmma consumers of 64 rows
// each; setmaxnreg moves the producers' registers to the consumers' fp32 accumulators (<= 128 per thread).
constexpr int kConvThreads = 384;
constexpr int kConvConsumerWarps = 8;
constexpr int kConvProducerRegs = 40;
constexpr int kConvConsumerRegs = 232;
constexpr int kConvMaxCout = 2048;  // ResNet50 layer4 (keypoints_tracker.py:158)

// Division by a launch-time constant as multiply-high + shift (dividend < 2^31): the per-tile coordinate decode of the
// persistent kernels would otherwise spend ~25 instructions per runtime `/` or `%` in every warp, every tile.
struct FastDiv {
  uint32_t d, mul, shr;
};
inline FastDiv make_fastdiv(int d) {
  FastDiv f{(uint32_t)d, 0u, 0u};
  if (d > 1) {
    int lg = 0;
    while ((1u << lg) < (uint32_t)d) ++lg;  // ceil(log2 d)
    const int p = 31 + lg;
    f.mul = (uint32_t)(((1ull << p) + (uint32_t)d - 1) / (uint32_t)d);
    f.shr = (uint32_t)(p - 32);
  }
  return f;
}
#ifdef __CUDACC__
__device__ __forceinline__ void fast_divmod(int& q, int& r, int n, const FastDiv& f) {
  q = f.d != 1u ? (int)(__umulhi((uint32_t)n, f.mul) >> f.shr) : n;
  r = n - q * (int)f.d;
}
#endif

struct ConvKParams {
  int N, Ho, Wo;
  int tiles_w, tiles_h, tiles_n, n_ntiles, total_tiles;
  FastDiv fd_w, fd_h, fd_nt;  // dividers by tiles_w, tiles_h, n_ntiles
  int tw_log2, th_log2;  // TW*TH*TN == 128
  int taps, kblocks, KB, BN, stages, cout_pad;
  int c_in_off;
  int tap_dc[9], tap_dw[9], tap_d2[9], tap_dh[9];
  const float* bias;
  int act;
  const __half* res;
  int res_C, res_coff;
  int res_first;  // 1: residual added before the activation (ResNet), 0: after (YOLO Bottleneck)
  void* out;
  int out_C, out_coff, out_mode, cout_store;
  void* out2;  // secondary output (PB_OUT2_*), fast epilogue only
  int out2_C, out2_coff, out2_mode;
  uint32_t a_bytes, b_bytes, b_tx_bytes;
  const float* head_w;
  const float* head_b;
  int head_n;
  float* head_out;
  int b_resident;  // halo variant: 1 = every weight box is fetched once per CTA and stays in shared memory
  int hs_S, hs_P, hs_G, a_stages, b_stages;  // halo variant: sub-tiles, halo pitch (px), taps per weight box, rings
  uint32_t halo_bytes;
  uint32_t hs_a_row_bytes;  // bytes of one halo row in shared memory (KB*2; 2*KB*2 for the stride-2 pixel-pair rows)
  int hs_ntaps, hs_sbo_rows, hs_x0, hs_y0, hs_tile_h;  // taps served from the halo, 8-row group stride (rows), box origin offsets
  int hs_tap_off[9];                                   // smem row offset of each tap's first pixel
  int hs_tap_desc[9];                                  // the same in 16-byte descriptor units (offset * row_bytes / 16)
  int dbg_flags;   // PADEL_B200_CONV_DEBUG: bit0 = plain two-MUFU SiLU (default: one reciprocal per four values), bit1 = no fast epilogue
  // halo variant, TMA-store epilogue: staging bytes per CTA (0 = per-lane stores), number of output maps the staging
  // tile is stored through (1 plain, 4 for a 2x2-replicated output, +4 for a PB_OUT2_UP2 copy), 1 = PB_OUT2_POOL2
  // through map st_maps
  uint32_t st_bytes;
  int st_maps, st_pool;
};

// Output tensor maps of the halo kernel's TMA-store epilogue (ConvKParams::st_maps, st_pool).
constexpr int kHaloStoreMaps = 5;
struct HaloStoreMaps {
  CUtensorMap m[kHaloStoreMaps];
};

struct ConvPlan {
  pb_conv_desc desc;
  ConvKParams kp;
  CUtensorMap tmap_a;
  CUtensorMap tmap_w;
  HaloStoreMaps tmap_o;
  int grid;
  int threads;
  size_t smem_bytes;
  int variant;  // 0 = per-tap boxes (conv_tc_kernel), 1 = shared halo tile (conv_halo_kernel)
  int pdl;      // programmatic dependent launch for this plan (captured from pb_set_plan_options at build time)
  int epi;      // PB_EPI_*: which epilogue instantiation of the kernel this layer runs
};

// epilogue classes (kernel template parameter kEpi)
#define PB_EPI_GENERIC 0
#define PB_EPI_SILU 1
#define PB_EPI_RELU 2
#define PB_EPI_SILU_RES 3  // SiLU, then + residual (ultralytics Bottleneck shortcut), fp16 NHWC
#define PB_EPI_F32 4       // no activation, fp32 NHWC slice (YOLO head outputs)
int conv_epi_class(const pb_conv_desc* d, const ConvKParams& kp);

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// The set-ups choose a plan by their rules, or take the tunable fields from `fp` (pb_conv_plan) when it is not null;
// the choice of set-up (the routing) never depends on fp.
int conv_halo_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode, bool force,
                    const pb_conv_plan* fp);  // -1: not applicable
int conv_stem_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode, const pb_conv_plan* fp);
int conv_halo_s2_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode,
                       const pb_conv_plan* fp);  // -1: not applicable
int conv_halo_1x1_setup(const pb_conv_desc* d, ConvPlan* plan, EncodeTiledFn encode,
                        const pb_conv_plan* fp);  // -1: not applicable
int conv_halo_launch(const ConvPlan* plan, cudaStream_t stream);
int conv_plan_build(const pb_conv_desc* d, ConvPlan* plan, const pb_conv_plan* fp = nullptr);
int conv_list_plans(const pb_conv_desc* d, pb_conv_plan* out, int cap);  // pb_conv_list_plans
int conv_plan_launch(const ConvPlan* plan, cudaStream_t stream);
int conv_reference_launch(const pb_conv_desc* d, cudaStream_t stream);

// aux kernels (aux_kernels.cu)
int launch_maxpool2(const void* in, int N, int H, int W, int C, int c_off, int c, void* out, int out_C,
                    int out_coff, cudaStream_t s);
int launch_upsample2(const void* in, int N, int H, int W, int C, int c_off, int c, void* out, int out_C,
                     int out_coff, cudaStream_t s);
int launch_sppf_pool(void* buf, int N, int H, int W, int C, int c, cudaStream_t s);
int launch_pointwise_head(const void* in, int N, int H, int W, int C, const float* w, const float* b, int n_out,
                          float* out, cudaStream_t s);

}  // namespace pb
