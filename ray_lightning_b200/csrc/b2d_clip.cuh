// b2d_clip.cuh — the global gradient norm of the sharded path (K18, K19) for gradient clipping.
//
// FairScale's OSS.clip_grad_norm (recalled) computes a local norm of the owned shard, all-reduces its square over NCCL
// and then runs a separate multiply over the gradients.  On the sharded path the averaged gradients exist only as every
// owner's fp32 shard (`reduced`, written by K12), so the norm is a cross-rank reduction:
//
//     K18  sqnorm_partial_kernel   G CTAs    this rank's sum of squares over its shard, in fp64, in an order that is a
//                                            function of n alone; the LAST block pushes the partial into slot `rank` of
//                                            the clip region in EVERY rank's arena, then arrives: clip[rank] = epoch in
//                                            every peer's pad.  Never waits.
//     K19  clip_coef_kernel        one warp  waits (at its start only) until clip[src] >= epoch for every src, adds the
//                                            W partials in rank order and writes norm and coef (fp32, device memory)
//
// and the coefficient is applied inside the fused Adam step (adam_push_scaled_kernel, b2d_owner.cuh): no extra pass over
// the gradients and no host synchronisation.
//
// Arithmetic (DESIGN.md §3), every rank computes identical bits:
//   * tiles of kClipTile = 4096 elements, the tail zero-padded; thread t of a 256-thread block adds the squares of
//     vectors t, t+256, t+512, t+768 of a tile in that order (x, y, z, w within a vector) — fp32 squares are exact in
//     fp64, each add rounds once; a fixed shared-memory tree (strides 128 .. 1) gives the tile sum;
//   * G = min(gmax, ntiles) blocks (one when n == 0); block b adds tiles b, b+G, ... in tile order; the last block
//     combines the G block sums with the same fixed tree;
//   * K19: total = ((p_0 + p_1) + p_2) + ... (fp64), norm = fp32(sqrt(total)),
//          coef = rcp(norm + 1e-6f) * max_norm, clamped to 1 with NaN kept — torch's clip_grad_norm_ sequence.
//
// Signalling: the clip exchange has its own monotone word per source (Signal::clip) and its own host epoch counter, so
// no bucket arrival (staged / published) and no BatchNorm exchange (bn) can satisfy its wait.  Its region holds two
// generations of W slots, chosen by the parity of the call count: a rank pushes into a generation again only after it
// has combined the call in between, which needs every peer's push of that call, which every peer issues only after its
// own combine of the call that last used the generation (DESIGN.md §5).
#pragma once

#include "b2d_staged.cuh"

namespace b2d {

constexpr int kClipThreads = 256;
constexpr int kClipTile = 4096;                 // elements: 256 threads x 4 vectors of 4
constexpr size_t kClipSlotBytes = 16;           // one fp64 partial per source rank, padded to a 16-byte vector store

struct ClipPartialParams {
  const float* x;          // the own shard (fp32)
  size_t n;
  int vec;                 // x is 16-byte aligned: whole vectors are loaded with one access
  double* block_sums;      // [gridDim.x] per-block partials (own arena)
  size_t region_off;       // byte offset, in every arena, of this generation's W slots
  int rank, world;
  uint32_t epoch;
  Peers peers;
};

struct ClipCoefParams {
  size_t region_off;
  float max_norm;
  float* norm_out;
  float* coef_out;
  int rank, world;
  uint32_t epoch;
  unsigned long long timeout_ns;
  Diag* diag;
  Peers peers;
};

// blocks of K18 for n elements: a function of n and gmax only
__host__ __device__ __forceinline__ unsigned clip_grid(size_t n, unsigned gmax) {
  const size_t ntiles = (n + kClipTile - 1) / kClipTile;
  return ntiles == 0 ? 1u : static_cast<unsigned>(ntiles < gmax ? ntiles : gmax);
}

#ifdef B2D_EMU
__device__ __forceinline__ double ld_f64_cg(const double* p) {
  uint64_t u = __atomic_load_n(reinterpret_cast<const uint64_t*>(p), __ATOMIC_RELAXED);
  double d; std::memcpy(&d, &u, 8); return d;
}
__device__ __forceinline__ void st_f64(double* p, double v) {
  uint64_t u; std::memcpy(&u, &v, 8); __atomic_store_n(reinterpret_cast<uint64_t*>(p), u, __ATOMIC_RELAXED);
}
#else
// another block's partial, published through the ticket: bypass L1
__device__ __forceinline__ double ld_f64_cg(const double* p) { return __ldcg(p); }
__device__ __forceinline__ void st_f64(double* p, double v) { *p = v; }
#endif

// fixed binary tree over s[0..kClipThreads): afterwards s[0] holds the sum; every thread of the block must call it
__device__ __forceinline__ void tree_sum(double* s) {
  __syncthreads();
#pragma unroll
  for (int stride = kClipThreads / 2; stride > 0; stride >>= 1) {
    if (threadIdx.x < static_cast<unsigned>(stride)) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + stride]);
    __syncthreads();
  }
}

__device__ __forceinline__ double add_sq(double acc, float v) {
  const double d = static_cast<double>(v);
  return __dadd_rn(acc, __dmul_rn(d, d));   // the square is exact in fp64: one rounding per element
}

// ---- K18 ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kClipThreads) sqnorm_partial_kernel(const __grid_constant__ ClipPartialParams P) {
#ifdef B2D_EMU
  double* s = emu_block->dscratch;
  int& s_last = emu_block->scratch;
#else
  __shared__ double s[kClipThreads];
  __shared__ int s_last;
#endif
  const unsigned G = gridDim.x;
  const size_t ntiles = (P.n + kClipTile - 1) / kClipTile;
  double bsum = 0.0;                                     // thread 0: this block's tiles, in tile order
  for (size_t tile = blockIdx.x; tile < ntiles; tile += G) {
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t i = tile * kClipTile + 4 * (threadIdx.x + static_cast<size_t>(j) * kClipThreads);
      float v[4];
      if (P.vec && i + 4 <= P.n) {
        const uint4 u = ld_stream_v4(P.x + i);
        v[0] = __uint_as_float(u.x); v[1] = __uint_as_float(u.y); v[2] = __uint_as_float(u.z); v[3] = __uint_as_float(u.w);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = i + k < P.n ? P.x[i + k] : 0.f;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) acc = add_sq(acc, v[k]);
    }
    s[threadIdx.x] = acc;
    tree_sum(s);
    if (threadIdx.x == 0) bsum = __dadd_rn(bsum, s[0]);   // only thread 0 reads s[0]: it alone rewrites it next
  }
  // ticket: the last block to finish combines the block sums (own counter, not done_ctr)
  Signal* self = P.peers.signal[P.rank];
  if (threadIdx.x == 0) {
    st_f64(P.block_sums + blockIdx.x, bsum);
    fence_sys();
    const unsigned ticket = atomicAdd(&self->clip_ctr, 1u);
    const int last = ticket == G - 1u;
    if (last) {
      self->clip_ctr = 0u;   // the next K18 of this rank starts after this one ended (same stream)
      fence_sys();
    }
    s_last = last;
  }
  __syncthreads();
  if (!s_last) return;
  s[threadIdx.x] = threadIdx.x < G ? ld_f64_cg(P.block_sums + threadIdx.x) : 0.0;
  tree_sum(s);
  const double partial = s[0];
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    uint64_t bits;
#ifdef B2D_EMU
    std::memcpy(&bits, &partial, 8);
#else
    bits = static_cast<uint64_t>(__double_as_longlong(partial));
#endif
    const uint4 u = make_uint4(static_cast<uint32_t>(bits), static_cast<uint32_t>(bits >> 32), 0u, 0u);
    st_v4(P.peers.arena[threadIdx.x] + P.region_off + static_cast<size_t>(P.rank) * kClipSlotBytes, u);
  }
  __syncthreads();
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    fence_sys();   // release: the slot stores of the block, cumulative over bar.sync
    st_flag(&P.peers.signal[threadIdx.x]->clip[P.rank], P.epoch);
  }
}

// ---- K19 ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) clip_coef_kernel(const __grid_constant__ ClipCoefParams P) {
  Signal* self = P.peers.signal[P.rank];
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    spin_until_ge(&self->clip[threadIdx.x], P.epoch, P.timeout_ns, P.diag, P.rank, threadIdx.x);
    fence_sys();   // acquire
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const unsigned char* slots = P.peers.arena[P.rank] + P.region_off;
  double total = 0.0;
  for (int r = 0; r < P.world; ++r) {
    const uint4 u = ld_peer_v4(slots + static_cast<size_t>(r) * kClipSlotBytes);
    const uint64_t bits = static_cast<uint64_t>(u.x) | (static_cast<uint64_t>(u.y) << 32);
    double p;
#ifdef B2D_EMU
    std::memcpy(&p, &bits, 8);
#else
    p = __longlong_as_double(static_cast<long long>(bits));
#endif
    total = r == 0 ? p : __dadd_rn(total, p);
  }
  const float norm = __double2float_rn(__dsqrt_rn(total));
  float coef = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), P.max_norm);
  coef = coef > 1.f ? 1.f : coef;   // torch.clamp(max=1): NaN stays NaN
  *P.norm_out = norm;
  *P.coef_out = coef;
}

}  // namespace b2d
