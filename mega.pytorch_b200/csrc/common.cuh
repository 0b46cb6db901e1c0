// Common device/host helpers for the sm_90a kernels of the MEGA hot path.
// Everything here is inline PTX for Hopper (wgmma / TMA / mbarrier);
// there is no dependency on CUTLASS or torch.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define MEGA_OK 0
#define MEGA_ERR_ARG 1
#define MEGA_ERR_CUDA 2
#define MEGA_ERR_UNSUPPORTED 3

#define MEGA_CUDA_CHECK(expr)                                                      \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      mega_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,                 \
                     cudaGetErrorString(_e));                                      \
      return MEGA_ERR_CUDA;                                                        \
    }                                                                              \
  } while (0)

#define MEGA_ARG_CHECK(cond, ...)                                                  \
  do {                                                                             \
    if (!(cond)) {                                                                 \
      mega_set_error(__VA_ARGS__);                                                 \
      return MEGA_ERR_ARG;                                                         \
    }                                                                              \
  } while (0)

// error string shared by every translation unit (defined in api.cu)
void mega_set_error(const char* fmt, ...);

static inline int mega_ceil_div(int a, int b) { return (a + b - 1) / b; }

#ifdef __CUDACC__
namespace mega {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xffffffff;\n"
      "selp.b32 %0, 1, 0, px;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier --
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a pipeline bug traps after ~2 s instead of hanging the GPU. No report is printed: printf is a function
// call, and a call anywhere in a kernel that issues wgmma makes ptxas serialise every one of its wgmma groups.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
#ifndef MEGA_NO_WATCHDOG
  uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
#endif
  while (!mbar_try_wait(bar, parity)) {
#ifndef MEGA_NO_WATCHDOG
    if ((++spins & 0x3ff) == 0 && globaltimer_ns() - t0 > 2000000000ull) __trap();
#endif
  }
}

// --------------------------------------------------------------------- TMA --
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tm, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tm),
      "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA store reads them)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------- wgmma --
// order register / shared-memory accesses of this warpgroup before the wgmma.mma_async that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed wgmma groups of this warpgroup still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait_regs(float (&d)[N]) {
  // the accumulators are read by ordinary instructions next: they must not be moved across the wait
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Per-warpgroup register budget: every warp of the warpgroup executes the same call. dec hands registers back to the
// CTA's pool; inc waits until the pool holds enough (the decs of the other warpgroups) and ptxas allocates the code that
// follows within the new count.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// blockIdx.x read where it is used (volatile: not merged with an earlier read). After setmaxnreg, ptxas keeps a value that
// lives from the kernel's prologue into the regions of different register counts in local memory.
__device__ __forceinline__ int ctaid_x_here() {
  int r;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(r));
  return r;
}

// K-major operand tile stored as rows of exactly 128 bytes with the 128B swizzle
// (what TMA writes for a box whose inner extent is 128 B): 8-row groups are 1024 B apart.
// Advancing the start address by 32 B selects the next 32 bytes of K inside the swizzle row.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);  // start address, 16 B units
  d |= static_cast<uint64_t>(1) << 16;                  // leading byte offset (unused for SW128 K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;          // stride byte offset: 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;                  // layout: SWIZZLE_128B
  return d;
}

// ------------------------------------------------- programmatic dependent launch --
// wait: blocks until every kernel this launch depends on has completed and flushed its writes (no-op for a
// launch without the programmatic-serialization attribute); launch_dependents: the next kernel on the stream
// may begin its prologue once every CTA of this grid has executed it (or exited).
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ------------------------------------------------------------------- fp16 packing --
__device__ __forceinline__ uint32_t f2_to_h2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// same, saturating to the largest finite half instead of inf
__device__ __forceinline__ uint32_t f2_to_h2_sat(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 h2_to_f2(uint32_t h) {
  float2 f;
  asm("{\n.reg .b16 l, h;\nmov.b32 {l, h}, %2;\ncvt.f32.f16 %0, l;\ncvt.f32.f16 %1, h;\n}" : "=f"(f.x), "=f"(f.y) : "r"(h));
  return f;
}

__device__ __forceinline__ float4 ldg_f4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

}  // namespace mega
#endif  // __CUDACC__
