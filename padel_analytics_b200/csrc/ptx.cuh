// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), stmatrix, setmaxnreg, wgmma.
// Hand-written for this repo; no CUTLASS/CuTe dependency.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace pb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization
// may start while its predecessor in the stream is still running: everything before griddep_wait() (barrier init,
// tensor-map prefetch, bias staging = constant data only) overlaps the predecessor's tail;
// griddep_wait() returns once the predecessor has completed and its writes are visible.  griddep_launch_dependents()
// lets the successor's CTAs be scheduled as SMs free up.  Both are no-ops for kernels launched without the attribute.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA tiled loads (global -> shared), completion on an mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, "
      "%7}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA tiled stores (shared -> global), completion tracked per thread in bulk groups
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory sources of all committed stores have been read (the staging area may be rewritten)
__device__ __forceinline__ void bulk_wait_group_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// all committed stores have completed
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// barrier over `count` threads (a multiple of 32) on hardware barrier `id` (0 is __syncthreads)
__device__ __forceinline__ void named_barrier_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Four 8x8 fp16 matrices, one 16-byte row per lane address (lane l: row l % 8 of matrix l / 8); register j of every
// lane holds its two elements of matrix j in the mma fragment layout (row l / 4, columns 2 (l % 4) + {0, 1}).
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}

// setmaxnreg: producers give registers back, consumers take them (executed by every warp of the warpgroup)
template <int kRegs>
__device__ __forceinline__ void warpgroup_reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs));
}
template <int kRegs>
__device__ __forceinline__ void warpgroup_reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs));
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// wgmma: D[64 x N, regs] (+)= A[64 x 16, smem] * B[N x 16, smem]^T, fp16 in, fp32 out, K-major.  Warp w, lane l:
// d[4i + 0, 1] = row 16w + l/4, columns 8i + 2(l%4) + {0, 1};  d[4i + 2, 3] = the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Keeps accumulator reads and writes from moving across an asynchronous wgmma.
template <int kN>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[kN]) {
#pragma unroll
  for (int i = 0; i < kN; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, K-major: addr>>4 | LBO>>4 << 16 | SBO>>4 << 32 | layout << 62 (1/2/3 = 128/64/32-byte
// swizzle rows of `row_bytes`, 0 = 16-byte un-swizzled rows whose second K half is `lbo_bytes` on); 8-row groups
// `sbo_bytes` apart.  The swizzle uses absolute address bits: a descriptor may start at any row of an aligned box.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t row_bytes, uint32_t sbo_bytes,
                                               uint32_t lbo_bytes = 16) {
  const uint64_t layout = row_bytes == 128 ? 1ull : (row_bytes == 64 ? 2ull : (row_bytes == 32 ? 3ull : 0ull));
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (layout << 62);
}
// dense K-major tile (TMA box of rows of `row_bytes`): 8-row groups 8 rows apart
__device__ __forceinline__ uint64_t wgmma_desc_kmajor(uint32_t saddr, uint32_t row_bytes) {
  return wgmma_desc(saddr, row_bytes, 8u * row_bytes);
}

// m64nNk16, N = 16 .. 256 in steps of 16: d[0 .. N/2) of the fragment above.  scale_d = 0 overwrites D.
template <int kN>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t a, uint64_t b, uint32_t scale_d);
// Operand lists of the specialisations: 8 accumulator registers per macro, RS<k> / DS<k> = the first 8k.
#define PB_WG_R0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define PB_WG_R1 "%8, %9, %10, %11, %12, %13, %14, %15"
#define PB_WG_R2 "%16, %17, %18, %19, %20, %21, %22, %23"
#define PB_WG_R3 "%24, %25, %26, %27, %28, %29, %30, %31"
#define PB_WG_R4 "%32, %33, %34, %35, %36, %37, %38, %39"
#define PB_WG_R5 "%40, %41, %42, %43, %44, %45, %46, %47"
#define PB_WG_R6 "%48, %49, %50, %51, %52, %53, %54, %55"
#define PB_WG_R7 "%56, %57, %58, %59, %60, %61, %62, %63"
#define PB_WG_R8 "%64, %65, %66, %67, %68, %69, %70, %71"
#define PB_WG_R9 "%72, %73, %74, %75, %76, %77, %78, %79"
#define PB_WG_R10 "%80, %81, %82, %83, %84, %85, %86, %87"
#define PB_WG_R11 "%88, %89, %90, %91, %92, %93, %94, %95"
#define PB_WG_R12 "%96, %97, %98, %99, %100, %101, %102, %103"
#define PB_WG_R13 "%104, %105, %106, %107, %108, %109, %110, %111"
#define PB_WG_R14 "%112, %113, %114, %115, %116, %117, %118, %119"
#define PB_WG_R15 "%120, %121, %122, %123, %124, %125, %126, %127"
#define PB_WG_D(k) "+f"(d[8 * k]), "+f"(d[8 * k + 1]), "+f"(d[8 * k + 2]), "+f"(d[8 * k + 3]), "+f"(d[8 * k + 4]), \
      "+f"(d[8 * k + 5]), "+f"(d[8 * k + 6]), "+f"(d[8 * k + 7])
#define PB_WGMMA(n_, a_, b_, s_, regs_, ops_)                                                              \
  template <>                                                                                                  \
  __device__ __forceinline__ void wgmma_f16<n_>(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {          \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #s_ ", 0;\n\t"                                        \
                 "wgmma.mma_async.sync.aligned.m64n" #n_ "k16.f32.f16.f16 {" regs_ "}, %" #a_ ", %" #b_             \
                 ", p, 1, 1, 0, 0;\n\t}"                                                                          \
                 : ops_                                                                                        \
                 : "l"(a), "l"(b), "r"(scale_d));                                                              \
  }
#define PB_COMMA ,
#define PB_WG_RS1 PB_WG_R0
#define PB_WG_RS2 PB_WG_RS1 ", " PB_WG_R1
#define PB_WG_RS3 PB_WG_RS2 ", " PB_WG_R2
#define PB_WG_RS4 PB_WG_RS3 ", " PB_WG_R3
#define PB_WG_RS5 PB_WG_RS4 ", " PB_WG_R4
#define PB_WG_RS6 PB_WG_RS5 ", " PB_WG_R5
#define PB_WG_RS7 PB_WG_RS6 ", " PB_WG_R6
#define PB_WG_RS8 PB_WG_RS7 ", " PB_WG_R7
#define PB_WG_RS9 PB_WG_RS8 ", " PB_WG_R8
#define PB_WG_RS10 PB_WG_RS9 ", " PB_WG_R9
#define PB_WG_RS11 PB_WG_RS10 ", " PB_WG_R10
#define PB_WG_RS12 PB_WG_RS11 ", " PB_WG_R11
#define PB_WG_RS13 PB_WG_RS12 ", " PB_WG_R12
#define PB_WG_RS14 PB_WG_RS13 ", " PB_WG_R13
#define PB_WG_RS15 PB_WG_RS14 ", " PB_WG_R14
#define PB_WG_RS16 PB_WG_RS15 ", " PB_WG_R15
#define PB_WG_DS1 PB_WG_D(0)
#define PB_WG_DS2 PB_WG_DS1 PB_COMMA PB_WG_D(1)
#define PB_WG_DS3 PB_WG_DS2 PB_COMMA PB_WG_D(2)
#define PB_WG_DS4 PB_WG_DS3 PB_COMMA PB_WG_D(3)
#define PB_WG_DS5 PB_WG_DS4 PB_COMMA PB_WG_D(4)
#define PB_WG_DS6 PB_WG_DS5 PB_COMMA PB_WG_D(5)
#define PB_WG_DS7 PB_WG_DS6 PB_COMMA PB_WG_D(6)
#define PB_WG_DS8 PB_WG_DS7 PB_COMMA PB_WG_D(7)
#define PB_WG_DS9 PB_WG_DS8 PB_COMMA PB_WG_D(8)
#define PB_WG_DS10 PB_WG_DS9 PB_COMMA PB_WG_D(9)
#define PB_WG_DS11 PB_WG_DS10 PB_COMMA PB_WG_D(10)
#define PB_WG_DS12 PB_WG_DS11 PB_COMMA PB_WG_D(11)
#define PB_WG_DS13 PB_WG_DS12 PB_COMMA PB_WG_D(12)
#define PB_WG_DS14 PB_WG_DS13 PB_COMMA PB_WG_D(13)
#define PB_WG_DS15 PB_WG_DS14 PB_COMMA PB_WG_D(14)
#define PB_WG_DS16 PB_WG_DS15 PB_COMMA PB_WG_D(15)
PB_WGMMA(16, 8, 9, 10, PB_WG_RS1, PB_WG_DS1)
PB_WGMMA(32, 16, 17, 18, PB_WG_RS2, PB_WG_DS2)
PB_WGMMA(48, 24, 25, 26, PB_WG_RS3, PB_WG_DS3)
PB_WGMMA(64, 32, 33, 34, PB_WG_RS4, PB_WG_DS4)
PB_WGMMA(80, 40, 41, 42, PB_WG_RS5, PB_WG_DS5)
PB_WGMMA(96, 48, 49, 50, PB_WG_RS6, PB_WG_DS6)
PB_WGMMA(112, 56, 57, 58, PB_WG_RS7, PB_WG_DS7)
PB_WGMMA(128, 64, 65, 66, PB_WG_RS8, PB_WG_DS8)
PB_WGMMA(144, 72, 73, 74, PB_WG_RS9, PB_WG_DS9)
PB_WGMMA(160, 80, 81, 82, PB_WG_RS10, PB_WG_DS10)
PB_WGMMA(176, 88, 89, 90, PB_WG_RS11, PB_WG_DS11)
PB_WGMMA(192, 96, 97, 98, PB_WG_RS12, PB_WG_DS12)
PB_WGMMA(208, 104, 105, 106, PB_WG_RS13, PB_WG_DS13)
PB_WGMMA(224, 112, 113, 114, PB_WG_RS14, PB_WG_DS14)
PB_WGMMA(240, 120, 121, 122, PB_WG_RS15, PB_WG_DS15)
PB_WGMMA(256, 128, 129, 130, PB_WG_RS16, PB_WG_DS16)
}  // namespace pb
