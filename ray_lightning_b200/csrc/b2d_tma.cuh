// b2d_tma.cuh — K2T: the two-shot allreduce with TMA bulk staging through shared memory.
//
// Why: the load/store kernels (b2d_kernels.cuh) are capped by what one SM's LSU/L1 can keep in
// flight, so they need many SMs to run the HBM phases at speed.  Here every load is a
// `cp.async.bulk` (Hopper TMA, SASS: UBLKCP) issued by one thread into a 3-deep shared-memory ring:
// 192 KiB in flight per SM (within sm_90's 227 KiB per block) with no registers and no L1 miss
// slots, so a few dozen CTAs can keep NVLink (peer loads, microseconds of latency) and HBM busy while
// the rest of the chip keeps running backward kernels.  Results leave with plain 16-byte stores
// (fire-and-forget, no latency to hide).
//
// Ownership: the slice index space is cut into macro tiles of `mt` packs; block b owns macro tiles
// m == b (mod grid) of EVERY slice in EVERY phase, so the per-block inter-GPU barrier of the
// load/store kernels carries over unchanged.  Arithmetic is the same Acc<> code: results are
// bit-identical to K1/K2.
#pragma once

#include "b2d_kernels.cuh"

namespace b2d {

constexpr int kTmaStages = 3;
constexpr int kTmaStageBytes = 64 * 1024;          // one ring slot
constexpr int kTmaMaxMt = kTmaStageBytes / 16;      // packs per macro tile (<= 4096)
constexpr int kTmaThreads = 512;
constexpr int kTmaSmemBytes = kTmaStages * kTmaStageBytes + 64;  // ring + mbarriers

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global (local or peer-mapped) -> shared, completion counted on `bar` in bytes.  SASS: UBLKCP.
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// One phase = a list of jobs; job q of this block loads up to `nsrc` pieces into ring slot
// q % kTmaStages.  The callbacks keep the three phases in one pipeline body.
struct TmaRing {
  unsigned char* slot[kTmaStages];
  uint64_t* full;       // [kTmaStages]
  uint32_t issued = 0;  // jobs whose loads were issued (thread 0 only)
  uint32_t done = 0;    // jobs consumed (all threads)
};

template <int W, bool BF16>
__global__ void __launch_bounds__(kTmaThreads, 1) k2t_two_shot_tma_kernel(const __grid_constant__ ArParams P, int mt) {
  static_assert(BF16, "the TMA path is written for the bf16 wire");
  constexpr int EPP = 8;
  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  const int world = W > 0 ? W : P.world;
  extern __shared__ __align__(128) unsigned char smem[];
  TmaRing ring;
#pragma unroll
  for (int s = 0; s < kTmaStages; ++s) ring.slot[s] = smem + static_cast<size_t>(s) * kTmaStageBytes;
  ring.full = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(kTmaStages) * kTmaStageBytes);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kTmaStages; ++s) mbar_init(&ring.full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const size_t npacks = (P.n + EPP - 1) / EPP;          // host guarantees n % 8 == 0 on this path
  const size_t slice = (npacks + world - 1) / world;
  const size_t n_mt = (slice + mt - 1) / mt;            // macro tiles per slice
  const size_t my_mt = n_mt > blockIdx.x ? (n_mt - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  uint4* my_stage = reinterpret_cast<uint4*>(P.peers.arena[P.rank] + P.stage_off);
  const int tid = threadIdx.x;
  trace_stamp(P.trace, 0);

  // number of valid packs of macro tile m inside slice s
  auto mt_len = [&](int s, size_t m) -> size_t {
    const size_t j0 = m * mt;
    size_t len = j0 < slice ? (slice - j0 < static_cast<size_t>(mt) ? slice - j0 : mt) : 0;
    const size_t p0 = static_cast<size_t>(s) * slice + j0;
    if (p0 >= npacks) return 0;
    return p0 + len > npacks ? npacks - p0 : len;
  };

  // ------------------------------------------------------------------ phase 0: stage (HBM)
  // job = (macro tile i, slice s, half h): mt/2 packs of wire = mt*16 bytes of fp32 gradients in
  {
    const uint32_t jobs = static_cast<uint32_t>(my_mt) * world * 2;
    auto issue = [&](uint32_t q) {
      const size_t m = blockIdx.x + static_cast<size_t>(q / (2 * world)) * gridDim.x;
      const int s = (q / 2) % world, h = q & 1;
      const size_t len = mt_len(s, m), half0 = (static_cast<size_t>(mt) / 2) * h;
      const size_t cnt = len > half0 ? (len - half0 < static_cast<size_t>(mt) / 2 ? len - half0 : mt / 2) : 0;
      uint64_t* bar = &ring.full[q % kTmaStages];
      mbar_expect_tx(bar, static_cast<uint32_t>(cnt * 32));
      if (cnt > 0) {
        const size_t p0 = static_cast<size_t>(s) * slice + m * mt + half0;
        bulk_load(ring.slot[q % kTmaStages], P.grad + p0 * EPP, static_cast<uint32_t>(cnt * 32), bar);
      }
    };
    uint32_t issued = 0;
    if (tid == 0)
      for (; issued < jobs && issued < kTmaStages; ++issued) issue(issued);
    for (uint32_t q = 0; q < jobs; ++q) {
      mbar_wait(&ring.full[q % kTmaStages], (ring.done / kTmaStages) & 1u);
      const size_t m = blockIdx.x + static_cast<size_t>(q / (2 * world)) * gridDim.x;
      const int s = (q / 2) % world, h = q & 1;
      const size_t len = mt_len(s, m), half0 = (static_cast<size_t>(mt) / 2) * h;
      const size_t cnt = len > half0 ? (len - half0 < static_cast<size_t>(mt) / 2 ? len - half0 : mt / 2) : 0;
      const size_t p0 = static_cast<size_t>(s) * slice + m * mt + half0;
      const uint4* in = reinterpret_cast<const uint4*>(ring.slot[q % kTmaStages]);
      for (size_t k = tid; k < cnt; k += kTmaThreads) {
        uint4 raw[2] = {in[2 * k], in[2 * k + 1]};
        st_v4(my_stage + p0 + k, to_wire<true>(raw, P.scale));
      }
      ring.done++;
      __syncthreads();  // every thread is done with the slot before it is refilled
      if (tid == 0 && issued < jobs) issue(issued++);
    }
  }
  trace_stamp(P.trace, 1);
  block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
  asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy stores (ours, the peers') before async-proxy reads
  trace_stamp(P.trace, 2);

  // ------------------------------------------------------------------ phase 1: reduce my slice (NVLink)
  // job = (macro tile i, part c of W): mt/W packs from each of the W ranks -> mt/W reduced packs
  {
    const int part = mt / world > 0 ? mt / world : 1;   // packs per rank per job (mt is a multiple of 8)
    const uint32_t parts = (mt + part - 1) / part;
    const uint32_t jobs = static_cast<uint32_t>(my_mt) * parts;
    auto geom = [&](uint32_t q, size_t& p0, size_t& cnt) {
      const size_t m = blockIdx.x + static_cast<size_t>(q / parts) * gridDim.x;
      const size_t len = mt_len(P.rank, m), off = static_cast<size_t>(q % parts) * part;
      cnt = len > off ? (len - off < static_cast<size_t>(part) ? len - off : part) : 0;
      p0 = static_cast<size_t>(P.rank) * slice + m * mt + off;
    };
    auto issue = [&](uint32_t q) {
      size_t p0, cnt;
      geom(q, p0, cnt);
      uint64_t* bar = &ring.full[(ring.issued + q) % kTmaStages];
      mbar_expect_tx(bar, static_cast<uint32_t>(cnt * 16 * world));
      if (cnt > 0) {
        for (int r = 0; r < world; ++r)
          bulk_load(ring.slot[(ring.issued + q) % kTmaStages] + static_cast<size_t>(r) * part * 16,
                    reinterpret_cast<const uint4*>(P.peers.arena[r] + P.stage_off) + p0, static_cast<uint32_t>(cnt * 16), bar);
      }
    };
    ring.issued = ring.done;  // slot/parity bookkeeping continues across phases
    const uint32_t base = ring.done;
    uint32_t issued = 0;
    if (tid == 0)
      for (; issued < jobs && issued < kTmaStages; ++issued) issue(issued);
    for (uint32_t q = 0; q < jobs; ++q) {
      const uint32_t slot = (base + q) % kTmaStages;
      mbar_wait(&ring.full[slot], ((base + q) / kTmaStages) & 1u);
      size_t p0, cnt;
      geom(q, p0, cnt);
      const uint4* in = reinterpret_cast<const uint4*>(ring.slot[slot]);
      for (size_t k = tid; k < cnt; k += kTmaThreads) {
        Acc<true> acc;
        acc.set(in[k]);
#pragma unroll
        for (int r = 1; r < WW; ++r)
          if (r < world) acc.add(in[static_cast<size_t>(r) * part + k]);
        st_v4(my_stage + p0 + k, acc.wire());
      }
      ring.done++;
      __syncthreads();
      if (tid == 0 && issued < jobs) issue(issued++);
    }
  }
  trace_stamp(P.trace, 3);
  block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
  asm volatile("fence.proxy.async;" ::: "memory");
  trace_stamp(P.trace, 4);

  // ------------------------------------------------------------------ phase 2: gather + fp32 write-back
  // job = (macro tile i, slice s): mt reduced packs from rank s -> 8*mt fp32 gradients out
  {
    const uint32_t jobs = static_cast<uint32_t>(my_mt) * world;
    auto geom = [&](uint32_t q, int& s, size_t& p0, size_t& cnt) {
      const size_t m = blockIdx.x + static_cast<size_t>(q / world) * gridDim.x;
      s = (q + P.rank) % world;   // start with the own (local) slice, spread the peers
      cnt = mt_len(s, m);
      p0 = static_cast<size_t>(s) * slice + m * mt;
    };
    ring.issued = ring.done;
    const uint32_t base = ring.done;
    auto issue = [&](uint32_t q) {
      int s; size_t p0, cnt;
      geom(q, s, p0, cnt);
      uint64_t* bar = &ring.full[(base + q) % kTmaStages];
      mbar_expect_tx(bar, static_cast<uint32_t>(cnt * 16));
      if (cnt > 0)
        bulk_load(ring.slot[(base + q) % kTmaStages], reinterpret_cast<const uint4*>(P.peers.arena[s] + P.stage_off) + p0,
                  static_cast<uint32_t>(cnt * 16), bar);
    };
    uint32_t issued = 0;
    if (tid == 0)
      for (; issued < jobs && issued < kTmaStages; ++issued) issue(issued);
    for (uint32_t q = 0; q < jobs; ++q) {
      const uint32_t slot = (base + q) % kTmaStages;
      mbar_wait(&ring.full[slot], ((base + q) / kTmaStages) & 1u);
      int s; size_t p0, cnt;
      geom(q, s, p0, cnt);
      const uint4* in = reinterpret_cast<const uint4*>(ring.slot[slot]);
      for (size_t k = tid; k < cnt; k += kTmaThreads) {
        uint4 raw[2];
        from_wire<true>(in[k], raw);
        grad_store<EPP>(P.grad, P.n, p0 + k, raw);
      }
      ring.done++;
      __syncthreads();
      if (tid == 0 && issued < jobs) issue(issued++);
    }
  }
  trace_stamp(P.trace, 5);
}

}  // namespace b2d
