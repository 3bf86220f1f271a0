// b2d_staged.cuh — the staged exchange (K7..K10): the bucket allreduce as a pipeline of SHORT kernels that
// never wait after they have signalled.
//
//     S  stage_kernel    local   fp32 gradients x scale -> wire format in the own arena; last block ARRIVES
//                                (staged[rank] = epoch in every peer's signal pad)
//     X  exch_kernel     NVLink  waits (at its start only) until staged[r] >= epoch for every r, then reduces
//                                the rank's own 1/W slice and PUSHES the result into every arena:
//                                  P2P : W peer loads (16 B each), rank-ordered fp32 adds, W peer stores
//                                  NVLS: one multimem.ld_reduce + one multimem.st per 16 bytes (in-switch sum)
//                                last block arrives (published[rank] = epoch)
//     W  wait_kernel     1 warp  waits until published[r] >= epoch for every r
//     U  unstage_kernel  local   wire format in the own arena -> fp32 gradients
//
// Why this shape (the fused K2 runs its phases strictly one after the other, and inside a training step its
// 64 x 512-thread CTAs sit spinning on whole SMs while they wait for slower peers):
//   * the HBM-bound passes (S, U) are plain grid-wide streaming kernels that hold SMs for microseconds and
//     never spin; only X (a few dozen CTAs) and W (one warp) ever wait for a peer;
//   * S, X and W+U run on three internal streams, so chunk c+1 is staged and chunk c-1 is written back while
//     chunk c crosses NVLink — inside one big bucket (chunks) and across consecutive DDP buckets;
//   * a kernel only ever waits at its START for flags that EARLIER launches set at their END, so any launch
//     order that respects the phases (S of all ranks, X of all ranks, W+U of all ranks) runs to completion even
//     when every kernel of a process is serialised — the single-GPU loopback ranks therefore survive ncu;
//   * the NVLS variant moves (1 + 1/W) x N x w bytes per GPU and direction instead of 2 (W-1)/W x N x w.
// The P2P variant adds in rank order in fp32 and rounds once: bit-identical to K1/K2 and to the oracle.  The
// NVLS variant sums inside the switch (fp32 accumulation, switch-defined order): tolerance contract only.
//
// IN-PLACE mode (fp32 wire, bucket storage inside the symmetric arena — SURVEY §8 f-1): there is nothing to
// stage or write back; S and U disappear, X works on the bucket itself (x scale), an `arrive_kernel` replaces S.
#pragma once

#include "b2d_kernels.cuh"

namespace b2d {

constexpr int kStThreads = 256;   // S / U: plain streaming CTAs
// X: 256 threads x <= 128 registers = half an SM's register file.  A 512-thread / 128-register CTA needs an EMPTY SM,
// which never comes up while the stage kernel of the next chunk (or a backward kernel) keeps refilling SMs: the
// pipeline then degenerates to stage-all | exchange-all.
constexpr int kExThreads = 256;

// spin until *ptr >= target (wrap-safe); trap with diagnostics after timeout_ns
__device__ __forceinline__ void spin_until_ge(const uint32_t* ptr, uint32_t target, unsigned long long timeout_ns,
                                              Diag* diag, int rank, int peer) {
  uint32_t got = ld_flag(ptr);
  if (static_cast<int32_t>(got - target) >= 0) return;
  const unsigned long long t0 = global_timer_ns();
  unsigned spins = 0;
  while (static_cast<int32_t>((got = ld_flag(ptr)) - target) < 0) {
    if ((++spins & 0xffu) == 0 && timeout_ns != 0 && global_timer_ns() - t0 > timeout_ns) {
      if (diag != nullptr) {
        diag->rank = rank; diag->block = blockIdx.x; diag->peer = peer; diag->expect = target; diag->got = got;
        diag->code = 1;
        fence_sys();
      }
      __trap();
    }
  }
}

// The block that finishes LAST publishes `epoch` into slot `which` (staged / published) of every peer's pad.
// Every block releases its writes at system scope before taking a ticket; the last block acquires the tickets
// and releases again before the flag stores (the classic threadfence-reduction pattern, lifted to .sys).
__device__ __forceinline__ void arrive_when_grid_done(const Peers& peers, int rank, int world, int which,
                                                      uint32_t epoch) {
#ifdef B2D_EMU
  int& s_last = emu_block->scratch;
#else
  __shared__ int s_last;
#endif
  __syncthreads();
  Signal* self = peers.signal[rank];
  if (threadIdx.x == 0) {
    fence_sys();
    const unsigned ticket = atomicAdd(&self->done_ctr[which], 1u);
    const int last = ticket == gridDim.x - 1u;
    if (last) {
      self->done_ctr[which] = 0u;   // the next kernel of this kind starts after this one ended (same stream)
      fence_sys();
    }
    s_last = last;
  }
  __syncthreads();
  if (s_last && threadIdx.x < static_cast<unsigned>(world)) {
    fence_sys();
    uint32_t* slot = which == 0 ? &peers.signal[threadIdx.x]->staged[rank] : &peers.signal[threadIdx.x]->published[rank];
    st_flag(slot, epoch);
  }
}

struct StParams {
  float* grad;      // this chunk's fp32 elements (already offset)
  size_t n;         // elements in the chunk
  uint4* wire;      // the chunk's wire region in the OWN arena
  float scale;
  int rank, world;
  uint32_t epoch;
  Peers peers;
};

// ---- S -------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(kStThreads, 4) stage_kernel(const __grid_constant__ StParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  constexpr int B = BF16 ? 4 : 8;   // 8 x 16-byte loads in flight per thread
  const size_t npacks = (P.n + EPP - 1) / EPP;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t j = g; j < npacks; j += gt * B) {
    size_t p[B];
    bool ok[B];
#pragma unroll
    for (int i = 0; i < B; ++i) { p[i] = j + i * gt; ok[i] = p[i] < npacks; }
    stage_batch<BF16, B>(P.grad, P.n, P.wire, p, ok, P.scale);
  }
  arrive_when_grid_done(P.peers, P.rank, P.world, 0, P.epoch);
}

// in-place mode: nothing to stage, only say "my bucket is ready" (stream-ordered after its producer)
__global__ void __launch_bounds__(32) arrive_kernel(const __grid_constant__ StParams P) {
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    fence_sys();
    st_flag(&P.peers.signal[threadIdx.x]->staged[P.rank], P.epoch);
  }
}

// ---- U -------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(kStThreads, 4) unstage_kernel(const __grid_constant__ StParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  constexpr int B = 8;
  const size_t npacks = (P.n + EPP - 1) / EPP;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t j = g; j < npacks; j += gt * B) {
    uint4 in[B];
#pragma unroll
    for (int i = 0; i < B; ++i)
      if (j + i * gt < npacks) in[i] = ld_peer_v4(P.wire + j + i * gt);   // peers (or the switch) wrote most of it
#pragma unroll
    for (int i = 0; i < B; ++i) {
      if (j + i * gt < npacks) {
        uint4 raw[EPP / 4];
        from_wire<BF16>(in[i], raw);
        grad_store<EPP>(P.grad, P.n, j + i * gt, raw);
      }
    }
  }
}

// ---- X -------------------------------------------------------------------------------------------------
struct ExParams {
  size_t wire_off;   // byte offset of the chunk's wire region (or of the bucket itself, in-place) in every arena
  size_t npacks;     // 16-byte packs in the chunk
  size_t n_valid;    // in-place only: fp32 elements that exist (the last pack may be partial)
  float scale;       // in-place only
  int rank, world;
  uint32_t epoch;
  unsigned long long timeout_ns;
  Diag* diag;
  Peers peers;
};

__device__ __forceinline__ uint4 scale_f32x4(const uint4& v, float s) {
  return make_uint4(__float_as_uint(__uint_as_float(v.x) * s), __float_as_uint(__uint_as_float(v.y) * s),
                    __float_as_uint(__uint_as_float(v.z) * s), __float_as_uint(__uint_as_float(v.w) * s));
}

template <int W, bool BF16, bool NVLS, bool INPLACE>
// NVLS keeps only U results in registers (64 registers -> a quarter of an SM's register file per CTA, 4 CTAs/SM); the
// P2P variant holds W copies per pack (<= 128 registers, 2 CTAs/SM).
__global__ void __launch_bounds__(kExThreads, NVLS ? 4 : 2) exch_kernel(const __grid_constant__ ExParams P) {
  static_assert(!(INPLACE && BF16), "in-place exchange exists for the fp32 wire only");
  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  const int world = W > 0 ? W : P.world;
  Signal* self = P.peers.signal[P.rank];
  if (threadIdx.x < static_cast<unsigned>(world)) {
    spin_until_ge(&self->staged[threadIdx.x], P.epoch, P.timeout_ns, P.diag, P.rank, threadIdx.x);
    fence_sys();   // acquire
  }
  __syncthreads();

  const size_t slice = (P.npacks + world - 1) / world;
  const size_t base = static_cast<size_t>(P.rank) * slice;
  size_t cnt = base < P.npacks ? P.npacks - base : 0;
  if (cnt > slice) cnt = slice;
  // in-place: a partial last pack (n_valid % 4 != 0) is handled element-wise by one thread at the end
  size_t full = cnt;
  bool ragged = false;
  if constexpr (INPLACE) {
    if (cnt > 0 && base + cnt == P.npacks && (P.n_valid & 3u) != 0) { full = cnt - 1; ragged = true; }
  }
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;

  if constexpr (NVLS) {
    constexpr int U = 8;
    uint4* mc = reinterpret_cast<uint4*>(P.peers.mc_arena + P.wire_off) + base;
    for (size_t j = g; j < full; j += gt * U) {
      uint4 red[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (j + u * gt < full) red[u] = BF16 ? multimem_ld_reduce_bf16x8(mc + j + u * gt) : multimem_ld_reduce_f32x4(mc + j + u * gt);
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (j + u * gt < full) multimem_st_v4(mc + j + u * gt, INPLACE ? scale_f32x4(red[u], P.scale) : red[u]);
    }
    if constexpr (INPLACE) {
      if (ragged && g == 0) {
        float* mcf = reinterpret_cast<float*>(mc + full);
        for (unsigned k = 0; k < (P.n_valid & 3u); ++k) multimem_st_f32(mcf + k, multimem_ld_reduce_f32(mcf + k) * P.scale);
      }
    }
  } else {
    constexpr int U = packs_per_batch(W);
    for (size_t j = g; j < full; j += gt * U) {
      uint4 in[U][WW];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (j + u * gt < full) {
#pragma unroll
          for (int r = 0; r < WW; ++r)
            if (r < world) in[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(P.peers.arena[r] + P.wire_off) + base + j + u * gt);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (j + u * gt < full) {
          Acc<BF16> acc;
          acc.set(INPLACE ? scale_f32x4(in[u][0], P.scale) : in[u][0]);
#pragma unroll
          for (int r = 1; r < WW; ++r)
            if (r < world) acc.add(INPLACE ? scale_f32x4(in[u][r], P.scale) : in[u][r]);
          const uint4 out = acc.wire();
#pragma unroll
          for (int r = 0; r < WW; ++r)
            if (r < world) st_v4(reinterpret_cast<uint4*>(P.peers.arena[r] + P.wire_off) + base + j + u * gt, out);
        }
      }
    }
    if constexpr (INPLACE) {
      if (ragged && g == 0) {
        for (unsigned k = 0; k < (P.n_valid & 3u); ++k) {
          float acc = 0.f;
          for (int r = 0; r < world; ++r) {
            const float v = __uint_as_float(ld_flag(reinterpret_cast<const uint32_t*>(P.peers.arena[r] + P.wire_off) + 4 * (base + full) + k)) * P.scale;
            acc = r == 0 ? v : __fadd_rn(acc, v);
          }
          for (int r = 0; r < world; ++r)
            st_flag(reinterpret_cast<uint32_t*>(P.peers.arena[r] + P.wire_off) + 4 * (base + full) + k, __float_as_uint(acc));
        }
      }
    }
  }
  arrive_when_grid_done(P.peers, P.rank, P.world, 1, P.epoch);
}

// ---- W -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) wait_published_kernel(const __grid_constant__ ExParams P) {
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    spin_until_ge(&P.peers.signal[P.rank]->published[threadIdx.x], P.epoch, P.timeout_ns, P.diag, P.rank, threadIdx.x);
    fence_sys();
  }
}

// ---- link probe: what one GPU can pull from ONE peer with this library's access pattern ------------------
// (the measured NVLink roofline denominator that bench.py reports next to the nominal rate)
__global__ void __launch_bounds__(kExThreads) peer_read_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t npacks) {
  constexpr int U = 16;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t j = g; j < npacks; j += gt * U) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j + u * gt < npacks) v[u] = ld_peer_v4(src + j + u * gt);
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j + u * gt < npacks) st_v4(dst + j + u * gt, v[u]);
  }
}

}  // namespace b2d
