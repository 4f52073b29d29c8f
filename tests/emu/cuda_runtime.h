// tests/emu/cuda_runtime.h -- CPU dry-run stand-in for the CUDA runtime and the device-side
// language features the kernels of aho-corasick_b200/csrc use.  TEST INFRASTRUCTURE ONLY: it lets
// the unmodified kernel sources be compiled with g++ and executed on a CPU-only machine so that
// their *logic* (tile/chunk partitioning, ownership of start offsets, queues, ordering keys, the
// host glue around them) can be checked against the oracle without a GPU.  It models none of the
// hardware's concurrency or memory model and says nothing about performance; the real `-m gpu`
// suite on an H100 remains the parity gate.
//
// Execution model: one CTA at a time; every CUDA thread of the CTA is a fiber (ucontext) scheduled
// round-robin and switched only at warp/CTA collectives and mbarrier waits.  "Device memory" is
// host memory.
#pragma once
#include <ucontext.h>

#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <vector>

// ---- language keywords ------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n)

struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct ulonglong2 { unsigned long long x, y; };
inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }
struct dim3 {
  unsigned x = 1, y = 1, z = 1;
  dim3() = default;
  dim3(unsigned x_, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}  // NOLINT
};

// ---- runtime API ------------------------------------------------------------------------------
enum cudaError_t { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum { cudaStreamNonBlocking = 1 };
struct CUstream_st { int unused; };
struct CUevent_st { std::chrono::steady_clock::time_point t; };
typedef CUstream_st* cudaStream_t;
typedef CUevent_st* cudaEvent_t;

inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
inline const char* cudaGetErrorName(cudaError_t e) { return e == cudaSuccess ? "cudaSuccess" : "cudaErrorEmulated"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) {
  const char* e = std::getenv("ACB_EMU_SMS");
  *v = e ? std::atoi(e) : 3;  // few "SMs": fewer CTAs to run one after the other, still several chunks
  return cudaSuccess;
}
template <class T>
inline cudaError_t cudaMalloc(T** p, size_t n) {
  void* q = nullptr;
  if (posix_memalign(&q, 256, n ? n : 1)) return cudaErrorMemoryAllocation;
  std::memset(q, 0xCD, n);  // device memory is not zero-initialised
  *p = static_cast<T*>(q);
  return cudaSuccess;
}
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
template <class T>
inline cudaError_t cudaMallocHost(T** p, size_t n) { *p = static_cast<T*>(std::malloc(n ? n : 1)); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFreeHost(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = new CUstream_st{0}; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new CUevent_st{}; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void* devicePointer; void* hostPointer; };
// every pointer is "ordinary host memory" in the dry run: the pageable-source staging path gets exercised
inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void*) { a->type = cudaMemoryTypeUnregistered; a->device = 0; return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = new CUevent_st{}; return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
  *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
  return cudaSuccess;
}
template <class F>
inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
template <class F>
inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t smem) {
  *n = (smem * 2 <= 227 * 1024) ? 2 : 1;
  return cudaSuccess;
}

// ---- device side: fibers -----------------------------------------------------------------------
namespace emu {

constexpr size_t kStackBytes = 128 * 1024;
constexpr size_t kDynSmemBytes = 232 * 1024;

struct Fiber {
  ucontext_t ctx;
  void* stack = nullptr;
  bool done = false;
  dim3 tid;
  const char* where = "running";  // what the thread last waited for (deadlock report)
};

struct Warp {
  uint32_t alive = 0;      // lanes that have not returned from the kernel
  uint32_t arrived = 0;
  uint32_t vals[32];
  uint64_t gen = 0;
  uint32_t result[2];
  uint32_t snap[2][32];
  int op = 0;
};

struct Cta {
  dim3 bidx, bdim, gdim;
  std::vector<Fiber> fibers;
  std::vector<Warp> warps;
  unsigned alive_threads = 0, bar_arrived = 0;
  uint64_t bar_gen = 0;
  uint64_t progress = 0;   // bumped whenever a collective completes or a fiber finishes
  uint64_t spins = 0;      // polls of shared words (each counts as progress until the budget is spent)
  std::function<void()> body;
};

inline Cta* g_cta = nullptr;
inline Fiber* g_cur = nullptr;
inline ucontext_t g_sched;
inline std::mutex g_one_launch_at_a_time;
inline unsigned char* g_dyn_smem = nullptr;  // exactly the requested bytes per launch: overruns are visible to ASAN
inline size_t g_dyn_smem_bytes = 0;

inline void yield(const char* where = "yield") { g_cur->where = where; swapcontext(&g_cur->ctx, &g_sched); }
// A thread that polls a shared word lets the others run first.  The poll itself is progress (the
// value may have changed while the thread was away) -- up to a budget, so that a spin nobody ever
// satisfies still ends in the deadlock report instead of a hang.
inline void yield_poll(const char* where) {
  if (++g_cta->spins < (1ull << 24)) g_cta->progress++;
  yield(where);
}
[[noreturn]] inline void die(const char* what) {
  std::fprintf(stderr, "emu: %s\n", what);
  std::abort();
}

enum { kOpSync = 1, kOpBallot, kOpAny, kOpAdd, kOpShfl };

inline uint32_t warp_collective(int op, uint32_t mask, uint32_t v, uint32_t src_lane = 0) {
  Cta& c = *g_cta;
  const unsigned t = g_cur->tid.x, lane = t & 31;
  Warp& w = c.warps[t >> 5];
  const uint32_t need = mask & w.alive;
  if (!(need >> lane & 1)) die("lane calls a collective it is not named in");
  auto reduce = [&](const uint32_t* vals) -> uint32_t {
    uint32_t r = 0;
    for (unsigned l = 0; l < 32; ++l) {
      if (!(need >> l & 1)) continue;
      if (op == kOpBallot) r |= (vals[l] ? 1u : 0u) << l;
      else if (op == kOpAny) r |= vals[l] ? 1u : 0u;
      else if (op == kOpAdd) r += vals[l];
    }
    return r;
  };
  if ((need & ~(1u << lane)) == 0) {  // nobody to wait for
    uint32_t one[32] = {0};
    one[lane] = v;
    return op == kOpShfl ? v : reduce(one);
  }
  if (w.arrived == 0) w.op = op;
  else if (w.op != op) die("lanes of one warp disagree on the collective they execute");
  w.vals[lane] = v;
  w.arrived |= 1u << lane;
  const uint64_t my = w.gen;
  if ((w.arrived & need) == need) {
    w.result[my & 1] = reduce(w.vals);
    std::memcpy(w.snap[my & 1], w.vals, sizeof(w.vals));
    w.arrived = 0;
    w.gen++;
    c.progress++;
  } else {
    while (w.gen == my) yield();
  }
  return op == kOpShfl ? w.snap[my & 1][src_lane & 31] : w.result[my & 1];
}

inline void cta_barrier() {
  Cta& c = *g_cta;
  const uint64_t my = c.bar_gen;
  if (++c.bar_arrived == c.alive_threads) {
    c.bar_arrived = 0;
    c.bar_gen++;
    c.progress++;
  } else {
    while (c.bar_gen == my) yield();
  }
}

inline void trampoline() {
  g_cta->body();
  Fiber* f = g_cur;
  Cta& c = *g_cta;
  f->done = true;
  c.warps[f->tid.x >> 5].alive &= ~(1u << (f->tid.x & 31));
  c.alive_threads--;
  c.progress++;
  if (c.warps[f->tid.x >> 5].arrived || c.bar_arrived) {
    // a thread left while others wait in a collective: the kernels under test never do that
    const Warp& w = c.warps[f->tid.x >> 5];
    if ((w.arrived && (w.arrived & w.alive) == w.alive) || (c.bar_arrived && c.bar_arrived == c.alive_threads))
      die("thread exit would have to complete a pending collective (not modelled)");
  }
  swapcontext(&f->ctx, &g_sched);
}

inline std::vector<void*>& stack_pool() {
  static std::vector<void*> pool;
  return pool;
}

template <class K, class... A>
inline void launch(K kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t, A... args) {
  std::lock_guard<std::mutex> lock(g_one_launch_at_a_time);  // the fiber scheduler's state is global
  if (smem > kDynSmemBytes) die("dynamic shared memory request too large");
  if (block.x % 32 && block.x > 32) die("block size must be a multiple of the warp size");
  auto& pool = stack_pool();
  while (pool.size() < block.x) pool.push_back(std::malloc(kStackBytes));
  for (unsigned b = 0; b < grid.x; ++b) {
    Cta cta;
    cta.bidx = dim3(b);
    cta.bdim = block;
    cta.gdim = grid;
    cta.fibers.resize(block.x);
    cta.warps.resize((block.x + 31) / 32);
    cta.alive_threads = block.x;
    cta.body = [&]() { kernel(args...); };
    void* sm = nullptr;
    if (posix_memalign(&sm, 128, smem ? smem : 128)) die("out of memory");
    g_dyn_smem = static_cast<unsigned char*>(sm);
    g_dyn_smem_bytes = smem;
    std::memset(g_dyn_smem, 0xCD, smem);  // shared memory is not zero-initialised
    g_cta = &cta;
    for (unsigned t = 0; t < block.x; ++t) {
      Fiber& f = cta.fibers[t];
      f.tid = dim3(t);
      f.stack = pool[t];
      cta.warps[t >> 5].alive |= 1u << (t & 31);
      getcontext(&f.ctx);
      f.ctx.uc_stack.ss_sp = f.stack;
      f.ctx.uc_stack.ss_size = kStackBytes;
      f.ctx.uc_link = nullptr;
      makecontext(&f.ctx, reinterpret_cast<void (*)()>(trampoline), 0);
    }
    // Schedule: which runnable thread goes next is not defined by CUDA between synchronisation
    // points, so the order is a knob -- ACB_EMU_SCHED=forward (default) | reverse | random:<seed>.
    // Results that depend on it reveal a missing __syncwarp / __syncthreads.
    static const char* sched_env = std::getenv("ACB_EMU_SCHED");
    const bool reverse = sched_env && !std::strcmp(sched_env, "reverse");
    const bool random = sched_env && !std::strncmp(sched_env, "random", 6);
    static uint64_t rng = random && std::strlen(sched_env) > 7 ? std::strtoull(sched_env + 7, nullptr, 10) * 2 + 1 : 12345;
    std::vector<unsigned> order(block.x);
    for (unsigned t = 0; t < block.x; ++t) order[t] = reverse ? block.x - 1 - t : t;
    unsigned remaining = block.x;
    while (remaining) {
      const uint64_t before = cta.progress;
      remaining = 0;
      if (random)
        for (unsigned t = block.x; t > 1; --t) {
          rng = rng * 6364136223846793005ull + 1442695040888963407ull;
          std::swap(order[t - 1], order[(rng >> 33) % t]);
        }
      for (unsigned t : order) {
        Fiber& f = cta.fibers[t];
        if (f.done) continue;
        g_cur = &f;
        swapcontext(&g_sched, &f.ctx);
        if (!f.done) ++remaining;
      }
      if (remaining && cta.progress == before) {
        for (unsigned t = 0; t < block.x; ++t)
          if (!cta.fibers[t].done && (t % 32 == 0 || std::strcmp(cta.fibers[t].where, cta.fibers[t - 1].where)))
            std::fprintf(stderr, "emu: cta %u thread %u waits in %s\n", b, t, cta.fibers[t].where);
        die("deadlock: no thread of the CTA can make progress");
      }
    }
    g_cta = nullptr;
    g_cur = nullptr;
    std::free(g_dyn_smem);
    g_dyn_smem = nullptr;
    g_dyn_smem_bytes = 0;
  }
}

}  // namespace emu

#define threadIdx (emu::g_cur->tid)
#define blockIdx (emu::g_cta->bidx)
#define blockDim (emu::g_cta->bdim)
#define gridDim (emu::g_cta->gdim)

// ---- device intrinsics ---------------------------------------------------------------------------
inline void __syncthreads() { emu::cta_barrier(); }
inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_collective(emu::kOpSync, mask, 0); }
inline unsigned __ballot_sync(unsigned mask, int pred) { return emu::warp_collective(emu::kOpBallot, mask, pred != 0); }
inline int __any_sync(unsigned mask, int pred) { return (int)emu::warp_collective(emu::kOpAny, mask, pred != 0); }
inline unsigned __reduce_add_sync(unsigned mask, unsigned v) { return emu::warp_collective(emu::kOpAdd, mask, v); }
inline unsigned long long __shfl_sync(unsigned mask, unsigned long long v, int src) {
  const uint32_t lo = emu::warp_collective(emu::kOpShfl, mask, (uint32_t)v, (uint32_t)src);
  const uint32_t hi = emu::warp_collective(emu::kOpShfl, mask, (uint32_t)(v >> 32), (uint32_t)src);
  return ((unsigned long long)hi << 32) | lo;
}
inline unsigned __shfl_down_sync(unsigned mask, unsigned v, unsigned delta) {
  const unsigned lane = emu::g_cur->tid.x & 31;
  return emu::warp_collective(emu::kOpShfl, mask, v, lane + delta < 32 ? lane + delta : lane);
}
// Any subset of the converged lanes that contains the caller is a legal answer; the fiber model
// has no notion of convergence, so the caller alone it is.
inline unsigned __activemask() { return 1u << (emu::g_cur->tid.x & 31); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline unsigned __brev(unsigned v) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((v >> i) & 1u) << (31 - i); return r; }
inline unsigned __byte_perm(unsigned x, unsigned y, unsigned sel) {
  const unsigned long long v = ((unsigned long long)y << 32) | x;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xFF) << (8 * i);
  return r;
}
inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned shift) {
  return (unsigned)((((unsigned long long)hi << 32) | lo) >> (shift & 31));
}
// clamped variant: shift = min(shift, 32)
inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned shift) {
  return (unsigned)((((unsigned long long)hi << 32) | lo) >> (shift < 32 ? shift : 32));
}
template <class T>
inline T __ldg(const T* p) { return *p; }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; *p = o + v; return o; }
inline unsigned atomicAdd(unsigned* p, unsigned v) { const unsigned o = *p; *p = o + v; return o; }
inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)((const unsigned char*)p - emu::g_dyn_smem); }
template <class T>
inline T min(T a, T b) { return a < b ? a : b; }
template <class T>
inline T max(T a, T b) { return a < b ? b : a; }
