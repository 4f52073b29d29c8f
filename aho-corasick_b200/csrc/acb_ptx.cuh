// acb_ptx.cuh -- the inline-PTX primitives of the kernels (sm_90a), in one place:
// mbarrier + bulk async copy (TMA) for the haystack ring, shared-memory reads by 32-bit shared
// address, the streaming global load of the walk kernel, and the kernel launch macro.
//
// Everything hardware-specific the kernels need beyond plain CUDA C++ goes through this header,
// which is also the seam of the CPU dry-run build under tests/emu/ (it substitutes its own
// version through ACB_PTX_HEADER; the product always compiles this file).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define ACB_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
// the kernel's dynamic shared memory as a byte array
#define ACB_DYNAMIC_SMEM(name) extern __shared__ __align__(128) unsigned char name[]

namespace acb {
namespace ptx {

// 32-bit shared-window address of a pointer into shared memory
__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier (transaction barrier in shared memory) ----
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// cp.async.bulk (TMA, SASS UBLKCP): `bytes` (multiple of 16) from 16-byte aligned global memory
// into shared memory, completion signalled on the mbarrier as transaction bytes.
__device__ __forceinline__ void tma_load_1d(uint32_t smem_dst, const void* gmem_src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_dst), "l"(gmem_src), "r"(bytes), "r"(bar)
               : "memory");
}
// cp.async.bulk.prefetch.L2 (SASS UBLKPF): bring `bytes` (multiple of 16) of 16-byte aligned global
// memory into L2 ahead of the bulk copy that will read them; no shared memory, no completion.
__device__ __forceinline__ void bulk_prefetch_l2(const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// ---- shared-memory reads by shared address (volatile: they stay behind the mbarrier wait) ----
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
// shared-memory fetch-and-add by one thread (the plain atomicAdd is compiled into a warp-aggregated
// sequence that costs a dozen instructions even when a single lane calls it)
__device__ __forceinline__ uint32_t atoms_add(uint32_t addr, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(addr), "r"(v) : "memory");
  return old;
}
// 64-bit shared-memory fetch-and-add / exchange (the CTA's tile-draw state: super-tile | offset)
__device__ __forceinline__ uint64_t atoms_add64(uint32_t addr, uint64_t v) {
  uint64_t old;
  asm volatile("atom.shared.add.u64 %0, [%1], %2;" : "=l"(old) : "r"(addr), "l"(v) : "memory");
  return old;
}
__device__ __forceinline__ void atoms_exch64(uint32_t addr, uint64_t v) {
  uint64_t old;
  asm volatile("atom.shared.exch.b64 %0, [%1], %2;" : "=l"(old) : "r"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds32_volatile(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts32_volatile(uint32_t addr, uint32_t v) {
  asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t lds64_volatile(uint32_t addr) {
  uint64_t v;
  asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
  return v;
}
// make three values opaque to the compiler so that they stay in registers instead of being
// re-derived (from the thread index) at every use
__device__ __forceinline__ void keep_in_registers(uint32_t& a, uint32_t& b, uint32_t& c) {
  asm volatile("" : "+r"(a), "+r"(b), "+r"(c));
}

// ---- streaming 16-byte global load (read-only path, no L1 allocation) ----
__device__ __forceinline__ uint4 ld_nc_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

}  // namespace ptx
}  // namespace acb
