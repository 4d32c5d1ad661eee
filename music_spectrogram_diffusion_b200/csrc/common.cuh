// Shared device-side helpers for the sm_90a kernels: mbarrier and TMA PTX
// wrappers and the wgmma descriptor builder.  Hand-written inline PTX; no CUTLASS.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace msd {

// ----------------------------------------------------------------------------
// Host-side error plumbing (thread-local last error string, see capi.cu)
// ----------------------------------------------------------------------------
void set_error(const char* fmt, ...);

#define MSD_CUDA_CHECK(expr)                                                     \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) {                                                     \
      ::msd::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,             \
                       cudaGetErrorString(_e));                                  \
      return -2;                                                                 \
    }                                                                            \
  } while (0)

#define MSD_REQUIRE(cond, ...)                                                   \
  do {                                                                           \
    if (!(cond)) {                                                               \
      ::msd::set_error(__VA_ARGS__);                                             \
      return -1;                                                                 \
    }                                                                            \
  } while (0)

// Propagates a non-zero return code (of a launcher or another int-returning helper)
#define MSD_TRY(expr)                                                            \
  do {                                                                           \
    int _rc = (expr);                                                            \
    if (_rc != 0) return _rc;                                                    \
  } while (0)

// ----------------------------------------------------------------------------
// Small device utilities
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ----------------------------------------------------------------------------
// Programmatic dependent launch (PDL): every kernel lets its successor's CTAs be scheduled as
// SMs free up (launch_dependents at entry) and orders its own global-memory traffic after the
// predecessor's completion (wait).  Threads that never touch dependent memory may skip wait.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void griddep_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void griddep_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
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
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes
// (or ~10 ms pass) instead of spinning and stealing issue slots from the working warps.
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
// Bounded: a protocol bug traps (launch failure) after ~10 s instead of hanging the GPU.
#ifndef MSD_MBAR_SPIN_LIMIT
#define MSD_MBAR_SPIN_LIMIT 1024u
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > MSD_MBAR_SPIN_LIMIT) __trap();
  }
}

// ----------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads, 2D, completion on an mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)),
      "r"(c0), "r"(c1)
      : "memory");
}

// TMA stores shared -> global, tracked per issuing thread in bulk async-groups.  Generic-proxy
// writes to the source must be made visible to the async proxy first (fence_proxy_async_smem,
// then a barrier over the writers); wait_group_read<N> returns once at most N of the thread's
// groups still read shared memory, wait_group_all once all of them have completed their writes.
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// all of the thread's groups complete (at a kernel's exit: no memory clobber, nothing follows)
__device__ __forceinline__ void bulk_wait_group_all() { asm volatile("cp.async.bulk.wait_group 0;"); }

// ----------------------------------------------------------------------------
// wgmma shared-memory matrix descriptors (PTX ISA "asynchronous warpgroup-level matrix
// shared memory layout / matrix descriptor")
// ----------------------------------------------------------------------------
//   bits [0,14)  start address >> 4
//   bits [16,30) leading-dim byte offset >> 4
//   bits [32,46) stride-dim  byte offset >> 4
//   bits [62,64) layout type: 1 = SWIZZLE_128B
// K-major operand tile [rows][64 bf16] (128-byte rows, TMA SWIZZLE_128B): 8-row groups are
//   1024 B apart (SBO); LBO is unused for swizzled K-major; a k-step of 16 elements advances the
//   start address by 32 B inside the swizzle atom.
// MN-major operand tile [k][64 bf16] (128-byte rows indexed by k): 8-k groups are 1024 B apart
//   (SBO); LBO (stride between 64-wide MN atoms) unused for MN = 64; a k-step of 16 advances the
//   start address by 2048 B.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ----------------------------------------------------------------------------
// Math
// ----------------------------------------------------------------------------
__device__ __forceinline__ float gelu_tanh(float x) {
  // flax.linen.gelu(approximate=True): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))).
  // tanh.approx.f32 is one SFU instruction (abs. error ~5e-4, below the bf16 output's half-ulp
  // for the product that follows); the exp-based form cost ~12 instructions per element and made
  // the gated-MLP epilogue as long as its main loop.
  const float k0 = 0.7978845608028654f, k1 = 0.044715f * 0.7978845608028654f;
  const float x2 = x * x;
  const float u = x * fmaf(k1, x2, k0);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  const float hx = 0.5f * x;
  return fmaf(hx, t, hx);
}

}  // namespace msd
