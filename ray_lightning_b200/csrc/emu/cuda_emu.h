// cuda_emu.h — just enough of the CUDA device environment to run the libb2d KERNEL SOURCES on CPU threads.
//
// TEST INFRASTRUCTURE ONLY (tests/test_kernel_emulation.py).  The product never includes this file: it is
// pulled in by b2d_device.cuh only when B2D_EMU is defined, which only emu_harness.cpp does.  One OS thread
// plays one CUDA thread; a CUDA block is 512 such threads sharing a barrier object; the W ranks of a job run
// their kernels concurrently inside one process, their "arenas" being plain host allocations that every
// "GPU" can address — so the inter-rank protocol (epoch flags, per-block barriers, double buffering, the
// (block, thread) -> pack mappings) executes for real, under whatever interleaving the OS scheduler produces.
// What this does NOT model: GPU memory-ordering weaknesses (x86 is TSO), NVLink, performance.
#pragma once

#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <map>
#include <memory>
#include <mutex>
#include <sched.h>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __grid_constant__
#define __restrict__

struct uint4 {
  uint32_t x, y, z, w;
};
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct EmuDim3 {
  unsigned x = 1, y = 1, z = 1;
};

namespace emu {

// everything a block's threads share
struct Block {
  explicit Block(int nthreads) : n(nthreads), bar0(nthreads) {}
  int n;
  int scratch = 0;   // stands in for a __shared__ int (b2d_staged.cuh: "was this the last block?")
  double dscratch[256] = {};   // stands in for a __shared__ double[256] (b2d_clip.cuh: the block's summation tree)
  std::barrier<> bar0;
  std::mutex mu;
  std::map<int, std::unique_ptr<std::barrier<>>> named;  // id -> barrier(count)
  std::barrier<>& get_named(int id, int count) {
    std::lock_guard<std::mutex> lk(mu);
    auto& p = named[id];
    if (!p) p = std::make_unique<std::barrier<>>(count);
    return *p;
  }
};

// the multicast alias of the arenas (NVLS): a fake base address + the real bases
struct Multicast {
  unsigned char* fake_base = nullptr;
  int world = 0;
  unsigned char* arena[8] = {};
};
inline Multicast& multicast() {
  static Multicast m;
  return m;
}

}  // namespace emu

extern thread_local EmuDim3 threadIdx, blockIdx, blockDim, gridDim;
extern thread_local emu::Block* emu_block;

// B2D_EMU_JITTER=<permille>: every barrier entry sleeps a random 0-300 us with that probability, so that
// roles / blocks / ranks drift apart far more than the scheduler alone would make them (straggler stress)
inline void emu_jitter() {
  const char* e = std::getenv("B2D_EMU_JITTER");   // read per call: tests switch it on and off within one process
  const int permille = e ? std::atoi(e) : 0;
  if (permille <= 0) return;
  thread_local uint32_t state = 0x9e3779b9u ^ static_cast<uint32_t>(reinterpret_cast<uintptr_t>(&state));
  state = state * 1664525u + 1013904223u;
  if (static_cast<int>((state >> 16) % 1000u) < permille) {
    timespec ts{0, static_cast<long>((state >> 8) % 300u) * 1000L};
    nanosleep(&ts, nullptr);
  }
}
inline void __syncthreads() { emu_jitter(); emu_block->bar0.arrive_and_wait(); }
inline void emu_named_barrier(int id, int count) { emu_jitter(); emu_block->get_named(id, count).arrive_and_wait(); }
inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
[[noreturn]] inline void __trap() {
  std::fprintf(stderr, "emulated kernel trapped (peer timeout)\n");
  std::abort();
}

inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }   // no contraction, one rounding
inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
inline float __fsqrt_rn(float a) { volatile float r = std::sqrt(a); return r; }
inline float __frcp_rn(float a) { volatile float r = 1.f / a; return r; }
inline float __fmaf_rn(float a, float b, float c) { volatile float r = std::fma(a, b, c); return r; }   // libm: one rounding
inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
inline double __dsqrt_rn(double a) { volatile double r = std::sqrt(a); return r; }
inline float __double2float_rn(double a) { volatile float r = static_cast<float>(a); return r; }

// fp32 -> bf16 bits, round to nearest even, NaN kept quiet (what cvt.rn.bf16.f32 does)
inline uint16_t emu_f32_to_bf16(float x) {
  uint32_t u = __float_as_uint(x);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x0040u);
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}
inline float emu_bf16_to_f32(uint16_t b) { return __uint_as_float(static_cast<uint32_t>(b) << 16); }

// relaxed atomic 32-bit accesses: the emulated "GPUs" race on flags and payload by design
inline uint32_t emu_ld32(const void* p) { return __atomic_load_n(static_cast<const uint32_t*>(p), __ATOMIC_RELAXED); }
inline void emu_st32(void* p, uint32_t v) { __atomic_store_n(static_cast<uint32_t*>(p), v, __ATOMIC_RELAXED); }
inline uint4 emu_ld128(const void* p) {
  const uint32_t* q = static_cast<const uint32_t*>(p);
  return uint4{emu_ld32(q), emu_ld32(q + 1), emu_ld32(q + 2), emu_ld32(q + 3)};
}
inline void emu_st128(void* p, const uint4& v) {
  uint32_t* q = static_cast<uint32_t*>(p);
  emu_st32(q, v.x); emu_st32(q + 1, v.y); emu_st32(q + 2, v.z); emu_st32(q + 3, v.w);
}
inline unsigned long long emu_timer_ns() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  sched_yield();  // the only place kernels spin: give the thousands of sibling threads a chance
  return static_cast<unsigned long long>(ts.tv_sec) * 1000000000ull + ts.tv_nsec;
}
