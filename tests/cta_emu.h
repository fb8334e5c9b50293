// Test infrastructure: a CTA of the CUDA execution model on host threads, just enough of it to run the block-cooperative
// device functions of chromap_b200/csrc/ (shared arrays, __syncthreads, warp shuffles) unchanged on a machine without a GPU.
// One OS thread per CUDA thread; barriers are counting barriers that threads may leave; a warp shuffle is an exchange through a per-warp buffer
// bracketed by two warp barriers.  Every lane of a warp must reach a shuffle (true of the functions under test: their scans
// are unconditional).  Not a performance tool.
// The kernel headers test CMX_HOST_EMU to leave out the few spots that have no host form (the end of this file supplies them).
#pragma once
#include <pthread.h>
#include <sched.h>

#include <atomic>
#include <mutex>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <numeric>
#include <random>
#include <string>
#include <thread>
#include <vector>

#define CMX_HOST_EMU 1

typedef unsigned long long u64;
typedef unsigned int u32;
typedef unsigned char u8;
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __global__
#define __shared__ static
#define __launch_bounds__(...)
#define __ldg(p) (*(p))
struct ulonglong2 { u64 x, y; };
using std::max;
using std::min;

struct EmuDim { int x; };
static thread_local EmuDim threadIdx, blockDim, blockIdx, gridDim;

// A barrier whose participants may leave: a CUDA thread that has returned from the kernel no longer takes part in
// __syncthreads / __syncwarp (the kernels' `if (slot >= n) return;` prologues rely on it).
struct EmuBarrier {  // (C++20: sleepers wait on the generation counter itself, so a release does not funnel them through the mutex)
  std::mutex m;
  int expected = 0, waiting = 0;
  std::atomic<unsigned> gen{0};
  void init(int n) { expected = n; waiting = 0; gen.store(0); }
  void wait() {
    unsigned g;
    bool last;
    {
      std::lock_guard<std::mutex> lk(m);
      g = gen.load(std::memory_order_relaxed);
      last = ++waiting >= expected;
      if (last) { waiting = 0; gen.store(g + 1, std::memory_order_release); }
    }
    if (last) gen.notify_all();
    else gen.wait(g, std::memory_order_acquire);
  }
  void drop() {
    bool release = false;
    {
      std::lock_guard<std::mutex> lk(m);
      --expected;
      if (expected > 0 && waiting >= expected) { waiting = 0; gen.store(gen.load(std::memory_order_relaxed) + 1, std::memory_order_release); release = true; }
    }
    if (release) gen.notify_all();
  }
};
// Kernels whose threads all stay to the end run on plain pthread barriers (faster); set g_emu_leavable for kernels with
// `if (slot >= n) return;` prologues followed by barriers among the rest.
static bool g_emu_leavable = false;
struct EmuSync {
  pthread_barrier_t fixed;
  EmuBarrier leav;
  bool leavable = false;
  void init(int n, bool l) { leavable = l; if (l) leav.init(n); else pthread_barrier_init(&fixed, nullptr, (unsigned)n); }
  void wait() { if (leavable) leav.wait(); else pthread_barrier_wait(&fixed); }
  void drop() { if (leavable) leav.drop(); }
  void destroy() { if (!leavable) pthread_barrier_destroy(&fixed); }
};
struct EmuCta {
  int nt = 0;
  EmuSync block;
  std::vector<EmuSync> warp;
  std::vector<u64> xch;  // [nt] exchange slots
};
static EmuCta *g_cta = nullptr;

static inline void __syncthreads() { g_cta->block.wait(); }
static inline int __syncthreads_or(int pred) {  // barrier + OR of pred over the CTA (threads that have left count as 0)
  g_cta->xch[threadIdx.x] = pred ? 1u : 0u;
  g_cta->block.wait();
  int r = 0;
  for (int t = 0; t < g_cta->nt; ++t) r |= (int)(g_cta->xch[(size_t)t] & 1u);
  g_cta->block.wait();
  return r;
}
static inline void __syncwarp(unsigned = 0xffffffffu) { g_cta->warp[threadIdx.x >> 5].wait(); }
template <typename T>
static inline T emu_shfl(T x, int src_lane) {  // value of lane src_lane of this warp (own value if out of range)
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  g_cta->xch[threadIdx.x] = (u64)x;
  g_cta->warp[w].wait();
  const int n_in_warp = std::min(32, g_cta->nt - w * 32);
  const T r = (src_lane >= 0 && src_lane < n_in_warp) ? (T)g_cta->xch[w * 32 + src_lane] : x;
  g_cta->warp[w].wait();
  (void)lane;
  return r;
}
template <typename T> static inline T __shfl_up_sync(unsigned, T x, int o) { const int l = threadIdx.x & 31; return emu_shfl(x, l - o >= 0 ? l - o : -1); }
template <typename T> static inline T __shfl_down_sync(unsigned, T x, int o) { const int l = threadIdx.x & 31; return emu_shfl(x, l + o < 32 ? l + o : -1); }
template <typename T> static inline T __shfl_xor_sync(unsigned, T x, int o) { return emu_shfl(x, (threadIdx.x & 31) ^ o); }
template <typename T> static inline T __shfl_sync(unsigned, T x, int src) { return emu_shfl(x, src & 31); }

static inline unsigned __ballot_sync(unsigned, bool pred) {
  const int w = threadIdx.x >> 5;
  g_cta->xch[threadIdx.x] = pred ? 1u : 0u;
  g_cta->warp[w].wait();
  unsigned m = 0;
  const int n_in_warp = std::min(32, g_cta->nt - w * 32);
  for (int l = 0; l < n_in_warp; ++l) m |= (unsigned)(g_cta->xch[w * 32 + l] & 1u) << l;
  g_cta->warp[w].wait();
  return m;
}
template <typename T, typename Op>
static inline T emu_reduce(T x, Op op) {  // every lane gets op over the warp
  const int w = threadIdx.x >> 5;
  g_cta->xch[threadIdx.x] = (u64)(long long)x;
  g_cta->warp[w].wait();
  const int n_in_warp = std::min(32, g_cta->nt - w * 32);
  T r = (T)(long long)g_cta->xch[w * 32];
  for (int l = 1; l < n_in_warp; ++l) r = op(r, (T)(long long)g_cta->xch[w * 32 + l]);
  g_cta->warp[w].wait();
  return r;
}
static inline int __reduce_add_sync(unsigned, int x) { return emu_reduce<int>(x, [](int a, int b) { return a + b; }); }
static inline unsigned __reduce_add_sync(unsigned, unsigned x) { return emu_reduce<unsigned>(x, [](unsigned a, unsigned b) { return a + b; }); }
static inline int __reduce_max_sync(unsigned, int x) { return emu_reduce<int>(x, [](int a, int b) { return a > b ? a : b; }); }
static inline int __reduce_min_sync(unsigned, int x) { return emu_reduce<int>(x, [](int a, int b) { return a < b ? a : b; }); }
struct int4 { int x, y, z, w; };
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }

// run `body` as CTA number `block` of a grid of `grid` CTAs, nt threads (nt a multiple of 32)
static inline void emu_launch(int nt, const std::function<void()> &body, int block = 0, int grid = 1) {
  EmuCta cta;
  cta.nt = nt;
  const bool leavable = g_emu_leavable;
  cta.block.init(nt, leavable);
  cta.warp = std::vector<EmuSync>((size_t)(nt + 31) / 32);
  for (size_t w = 0; w < cta.warp.size(); ++w) cta.warp[w].init(std::min(32, nt - (int)w * 32), leavable);
  cta.xch.assign((size_t)nt, 0);
  g_cta = &cta;
  std::vector<std::thread> th;
  for (int t = 0; t < nt; ++t)
    th.emplace_back([&, t]() {
      threadIdx.x = t;
      blockDim.x = nt;
      blockIdx.x = block;
      gridDim.x = grid;
      body();
      cta.xch[(size_t)t] = 0;
      cta.warp[(size_t)t >> 5].drop();
      cta.block.drop();
    });
  for (auto &x : th) x.join();
  cta.block.destroy();
  for (auto &b : cta.warp) b.destroy();
  g_cta = nullptr;
}
// a whole grid, one CTA after the other (CTAs of these kernels do not talk to each other except through atomics)
static inline void emu_grid(int grid, int nt, const std::function<void()> &body) {
  for (int b = 0; b < grid; ++b) emu_launch(nt, body, b, grid);
}
// the same for kernels without barriers or warp primitives (elementwise kernels): the CUDA threads one after the other on the
// calling OS thread
static inline void emu_grid_serial(int grid, int nt, const std::function<void()> &body) {
  for (int b = 0; b < grid; ++b)
    for (int t = 0; t < nt; ++t) {
      threadIdx.x = t; blockDim.x = nt; blockIdx.x = b; gridDim.x = grid;
      body();
    }
}

// ---- dynamic shared memory: tests/emu.py rewrites `extern __shared__ T name[];` as `T *name = (T *)g_dyn_smem;`, the test
// points it at a buffer of the launch's size
static u64 *g_dyn_smem = nullptr;

// ---- atomics and intrinsics
static inline u64 atomicAdd(u64 *p, u64 v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicAdd(int *p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline u32 atomicAdd(u32 *p, u32 v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicExch(int *p, int v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
static inline u64 atomicCAS(u64 *p, u64 cmp, u64 val) { __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED); return cmp; }
template <typename T> static inline T emu_atomic_max(T *p, T v) { T o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o < v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
template <typename T> static inline T emu_atomic_min(T *p, T v) { T o = __atomic_load_n(p, __ATOMIC_RELAXED); while (v < o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
static inline u64 atomicMax(u64 *p, u64 v) { return emu_atomic_max(p, v); }
static inline u32 atomicMax(u32 *p, u32 v) { return emu_atomic_max(p, v); }
static inline u32 atomicMin(u32 *p, u32 v) { return emu_atomic_min(p, v); }
// pipeline_kernels.cuh's counter helpers: on the device one atomic per group of converged lanes, here one per thread
static inline void agg_add(u64 *addr, u64 v) { atomicAdd(addr, v); }
static inline int agg_append(int *count) { return atomicAdd(count, 1); }
static inline double __dmul_rn(double a, double b) { return a * b; }   // (built with -ffp-contract=off: no FMA contraction either)
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
static inline u32 __funnelshift_r(u32 lo, u32 hi, u32 s) { return (u32)((((u64)hi << 32) | lo) >> (s & 31)); }

// ---- host equivalents of seed_front.cuh's six PTX wrappers (mbarrier + cp.async.bulk).
// An mbarrier word: bits 0-31 = bytes still expected, bits 32-47 = arrivals still expected, bits 48-63 = completed phases.  The
// "copy engine" copies at issue time and then signals its bytes, like complete_tx.
static inline void emu_mbar_settle(u64 *bar) {   // a phase completes when no arrival and no byte is outstanding: re-arm with one arrival
  u64 v = __atomic_load_n(bar, __ATOMIC_ACQUIRE);
  if ((v & 0xFFFFFFFFFFFFull) == 0) __atomic_store_n(bar, ((v >> 48) + 1) << 48 | (1ull << 32), __ATOMIC_RELEASE);
}
static inline u32 smem_u32(const void *p) { return (u32)(size_t)p; }
static inline void mbar_init(u64 *bar, u32 count) { __atomic_store_n(bar, (u64)count << 32, __ATOMIC_RELEASE); }
static inline void mbar_fence_init() {}
static inline void mbar_arrive_expect_tx(u64 *bar, u32 bytes) {   // (called by one thread, before its copies)
  u64 v = __atomic_load_n(bar, __ATOMIC_ACQUIRE);
  v = (v & 0xFFFF000000000000ull) | ((((v >> 32) & 0xFFFF) - 1) << 32) | (u64)((u32)v + bytes);
  __atomic_store_n(bar, v, __ATOMIC_RELEASE);
  emu_mbar_settle(bar);
}
static inline bool mbar_try_wait(u64 *bar, u32 parity) {
  const bool done = (((__atomic_load_n(bar, __ATOMIC_ACQUIRE) >> 48) & 1u) != parity);
  if (!done) sched_yield();
  return done;
}
static inline void bulk_g2s(void *dst, const void *src, u32 bytes, u64 *bar) {
  memcpy(dst, src, bytes);
  u64 v = __atomic_load_n(bar, __ATOMIC_ACQUIRE);
  __atomic_store_n(bar, (v & 0xFFFFFFFF00000000ull) | (u64)((u32)v - bytes), __ATOMIC_RELEASE);
  emu_mbar_settle(bar);
}
