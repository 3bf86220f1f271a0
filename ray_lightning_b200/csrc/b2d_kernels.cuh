// b2d_kernels.cuh — the gradient-sync kernels (K0..K6 of SURVEY.md §2.4C / DESIGN.md §4).
//
// All kernels are HBM/NVLink-bound byte movers with a few fp32 adds per 16 bytes; there is
// no contraction anywhere, so no tensor-core path.  Design rules followed:
//   * every global access is a 16-byte vector access, warp-contiguous (coalesced);
//   * loads are issued in explicit batches (up to 16 x 16 B per thread in flight) BEFORE any
//     of them is consumed: a peer load over NVLink takes microseconds, so bandwidth needs
//     about a megabyte in flight per GPU (NVLink 4 on H100: 450 GB/s per direction x ~2 us);
//   * the same (block, thread) touches the same pack in every phase, so one *per-block*
//     inter-GPU barrier between phases is enough — blocks of one rank never wait for each
//     other, and a comm kernel can run on a handful of SMs next to the backward pass;
//   * grids are small multiples of what the link needs (default 64 CTAs x 512 threads), not of
//     the SM count: the other SMs belong to the backward kernels this overlaps with.
#pragma once

#include "b2d_device.cuh"

namespace b2d {

constexpr int kThreads = 512;
constexpr int kMaxLoadsInFlight = 16;  // 16-byte loads per thread per batch
// packs a thread handles per batch when every pack costs `per_pack` loads (W peer copies, or W x 2 gradient loads);
// the generic-world instantiation (W = 0) takes one pack at a time
__host__ __device__ constexpr int packs_per_batch(int per_pack) {
  return per_pack > 0 && kMaxLoadsInFlight / (per_pack > 0 ? per_pack : 1) > 1 ? kMaxLoadsInFlight / (per_pack > 0 ? per_pack : 1) : 1;
}

constexpr int kTraceSlots = 8;  // globaltimer stamps per block: start, after each phase / barrier

struct ArParams {
  unsigned long long* trace;  // [gridDim.x][kTraceSlots] or nullptr (debug: b2d_ctx_trace)
  float* grad;        // this rank's flat fp32 bucket (in/out)
  size_t n;           // elements
  size_t stage_off;   // byte offset of this call's staging buffer inside every arena
  float scale;
  int rank, world;
  unsigned long long timeout_ns;
  Diag* diag;
  Peers peers;
};

__device__ __forceinline__ void trace_stamp(unsigned long long* trace, int slot) {
  if (trace != nullptr && threadIdx.x == 0)
    trace[static_cast<size_t>(blockIdx.x) * kTraceSlots + slot] = global_timer_ns();
}

// ---- pack helpers ------------------------------------------------------------------------
template <int EPP>
__device__ __forceinline__ void grad_load(const float* grad, size_t n, size_t p, uint4 (&raw)[EPP / 4]) {
  const size_t e0 = p * EPP;
  if (e0 + EPP <= n) {
#pragma unroll
    for (int q = 0; q < EPP / 4; ++q) raw[q] = ld_stream_v4(grad + e0 + 4 * q);
  } else {  // ragged tail of the bucket: scalar, zero padded
    float t[EPP];
#pragma unroll
    for (int k = 0; k < EPP; ++k) t[k] = (e0 + k < n) ? grad[e0 + k] : 0.f;
#pragma unroll
    for (int q = 0; q < EPP / 4; ++q)
      raw[q] = make_uint4(__float_as_uint(t[4 * q]), __float_as_uint(t[4 * q + 1]),
                          __float_as_uint(t[4 * q + 2]), __float_as_uint(t[4 * q + 3]));
  }
}
template <int EPP>
__device__ __forceinline__ void grad_store(float* grad, size_t n, size_t p, const uint4 (&raw)[EPP / 4]) {
  const size_t e0 = p * EPP;
  if (e0 + EPP <= n) {
#pragma unroll
    for (int q = 0; q < EPP / 4; ++q) st_stream_v4(grad + e0 + 4 * q, raw[q]);
  } else {
#pragma unroll
    for (int q = 0; q < EPP / 4; ++q) {
      const uint32_t w[4] = {raw[q].x, raw[q].y, raw[q].z, raw[q].w};
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (e0 + 4 * q + k < n) grad[e0 + 4 * q + k] = __uint_as_float(w[k]);
    }
  }
}

// fp32 gradients -> 16 bytes of wire payload
template <bool BF16>
__device__ __forceinline__ uint4 to_wire(const uint4 (&raw)[BF16 ? 2 : 1], float scale) {
  if constexpr (BF16) {
    const float a0 = wire_bf16_value(__uint_as_float(raw[0].x), scale);
    const float a1 = wire_bf16_value(__uint_as_float(raw[0].y), scale);
    const float a2 = wire_bf16_value(__uint_as_float(raw[0].z), scale);
    const float a3 = wire_bf16_value(__uint_as_float(raw[0].w), scale);
    const float a4 = wire_bf16_value(__uint_as_float(raw[1].x), scale);
    const float a5 = wire_bf16_value(__uint_as_float(raw[1].y), scale);
    const float a6 = wire_bf16_value(__uint_as_float(raw[1].z), scale);
    const float a7 = wire_bf16_value(__uint_as_float(raw[1].w), scale);
    // the values are already bf16-representable: packing is exact
    return make_uint4(pack_bf16x2(a0, a1), pack_bf16x2(a2, a3), pack_bf16x2(a4, a5),
                      pack_bf16x2(a6, a7));
  } else {
    return make_uint4(__float_as_uint(__uint_as_float(raw[0].x) * scale),
                      __float_as_uint(__uint_as_float(raw[0].y) * scale),
                      __float_as_uint(__uint_as_float(raw[0].z) * scale),
                      __float_as_uint(__uint_as_float(raw[0].w) * scale));
  }
}

// fp32 accumulator over one pack
template <bool BF16>
struct Acc {
  float v[BF16 ? 8 : 4];
  __device__ __forceinline__ void set(const uint4& w) {
    if constexpr (BF16) {
      v[0] = bf16_lo(w.x); v[1] = bf16_hi(w.x); v[2] = bf16_lo(w.y); v[3] = bf16_hi(w.y);
      v[4] = bf16_lo(w.z); v[5] = bf16_hi(w.z); v[6] = bf16_lo(w.w); v[7] = bf16_hi(w.w);
    } else {
      v[0] = __uint_as_float(w.x); v[1] = __uint_as_float(w.y);
      v[2] = __uint_as_float(w.z); v[3] = __uint_as_float(w.w);
    }
  }
  // strictly sequential fp32 adds in rank order: the result does not depend on which rank
  // computes it, nor on the algorithm (one-shot / two-shot give the same bits)
  __device__ __forceinline__ void add(const uint4& w) {
    if constexpr (BF16) {
      v[0] = __fadd_rn(v[0], bf16_lo(w.x)); v[1] = __fadd_rn(v[1], bf16_hi(w.x));
      v[2] = __fadd_rn(v[2], bf16_lo(w.y)); v[3] = __fadd_rn(v[3], bf16_hi(w.y));
      v[4] = __fadd_rn(v[4], bf16_lo(w.z)); v[5] = __fadd_rn(v[5], bf16_hi(w.z));
      v[6] = __fadd_rn(v[6], bf16_lo(w.w)); v[7] = __fadd_rn(v[7], bf16_hi(w.w));
    } else {
      v[0] = __fadd_rn(v[0], __uint_as_float(w.x)); v[1] = __fadd_rn(v[1], __uint_as_float(w.y));
      v[2] = __fadd_rn(v[2], __uint_as_float(w.z)); v[3] = __fadd_rn(v[3], __uint_as_float(w.w));
    }
  }
  // back to one wire pack (bf16: the single rounding of the sum)
  __device__ __forceinline__ uint4 wire() const {
    if constexpr (BF16) {
      return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                        pack_bf16x2(v[6], v[7]));
    } else {
      return make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]),
                        __float_as_uint(v[3]));
    }
  }
};

// 16 bytes of wire payload -> fp32 gradients
template <bool BF16>
__device__ __forceinline__ void from_wire(const uint4& w, uint4 (&raw)[BF16 ? 2 : 1]) {
  if constexpr (BF16) {
    raw[0] = make_uint4(w.x << 16, w.x & 0xffff0000u, w.y << 16, w.y & 0xffff0000u);
    raw[1] = make_uint4(w.z << 16, w.z & 0xffff0000u, w.w << 16, w.w & 0xffff0000u);
  } else {
    raw[0] = w;
  }
}

// ---- K0: world == 1 ----------------------------------------------------------------------
// In place: g <- fp32(bf16(bf16(g) * scale))  (bf16 wire)   or   g <- g * scale  (fp32 wire).
// 8 B/element of HBM traffic, nothing else.
template <bool BF16>
__global__ void __launch_bounds__(kThreads) k0_cast_scale_kernel(float* __restrict__ grad, size_t n,
                                                                 float scale) {
  constexpr int U = 4;  // 4 x 16 B in flight per thread
  const size_t nv = n / 4;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t i = g; i < nv; i += gt * U) {
    uint4 r[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (i + u * gt < nv) r[u] = ld_stream_v4(grad + 4 * (i + u * gt));
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (i + u * gt < nv) {
        float a = __uint_as_float(r[u].x), b = __uint_as_float(r[u].y);
        float c = __uint_as_float(r[u].z), d = __uint_as_float(r[u].w);
        if constexpr (BF16) {
          a = wire_bf16_value(a, scale); b = wire_bf16_value(b, scale);
          c = wire_bf16_value(c, scale); d = wire_bf16_value(d, scale);
        } else {
          a *= scale; b *= scale; c *= scale; d *= scale;
        }
        st_stream_v4(grad + 4 * (i + u * gt),
                     make_uint4(__float_as_uint(a), __float_as_uint(b), __float_as_uint(c),
                                __float_as_uint(d)));
      }
    }
  }
  // ragged tail (< 4 elements)
  if (g < n - nv * 4) {
    const size_t e = nv * 4 + g;
    const float x = grad[e];
    grad[e] = BF16 ? wire_bf16_value(x, scale) : x * scale;
  }
}

// ---- phase 0 shared by K1/K2/K3: cast + scale the own bucket into the own staging buffer --
// `count` packs starting at pack `first`, strided over the whole grid with the canonical
// (block, thread) -> pack mapping: pack first + j is handled by global thread j mod GT.
template <bool BF16, int B>
__device__ __forceinline__ void stage_batch(const float* grad, size_t n, uint4* stage,
                                            const size_t (&p)[B], const bool (&ok)[B], float scale) {
  constexpr int EPP = BF16 ? 8 : 4;
  uint4 raw[B][EPP / 4];
#pragma unroll
  for (int i = 0; i < B; ++i)
    if (ok[i]) grad_load<EPP>(grad, n, p[i], raw[i]);
#pragma unroll
  for (int i = 0; i < B; ++i)
    if (ok[i]) st_v4(stage + p[i], to_wire<BF16>(raw[i], scale));
}

// ---- K1: one-shot ------------------------------------------------------------------------
// stage -> barrier -> every rank reads all `world` staged copies of every pack, adds them in
// rank order in fp32, rounds once (bf16 wire) and writes its own fp32 bucket.
// NVLink bytes per rank: (W-1) * N * w in; best below ~0.5 MB where latency dominates.
template <int W, bool BF16>
__global__ void __launch_bounds__(kThreads, 1) k1_one_shot_kernel(const __grid_constant__ ArParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  const int world = W > 0 ? W : P.world;
  const size_t npacks = (P.n + EPP - 1) / EPP;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  uint4* my_stage = reinterpret_cast<uint4*>(P.peers.arena[P.rank] + P.stage_off);
  trace_stamp(P.trace, 0);

  {
    constexpr int B = BF16 ? 8 : 16;  // 16 x 16-byte loads in flight per thread
    for (size_t j = g; j < npacks; j += gt * B) {
      size_t p[B];
      bool ok[B];
#pragma unroll
      for (int i = 0; i < B; ++i) { p[i] = j + i * gt; ok[i] = p[i] < npacks; }
      stage_batch<BF16, B>(P.grad, P.n, my_stage, p, ok, P.scale);
    }
  }
  trace_stamp(P.trace, 1);
  block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
  trace_stamp(P.trace, 2);

  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  constexpr int U = packs_per_batch(W);
  for (size_t j = g; j < npacks; j += gt * U) {
    uint4 in[U][WW];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t p = j + u * gt;
      if (p < npacks) {
#pragma unroll
        for (int r = 0; r < WW; ++r)
          if (r < world)
            in[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(P.peers.arena[r] + P.stage_off) + p);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t p = j + u * gt;
      if (p < npacks) {
        Acc<BF16> acc;
        acc.set(in[u][0]);
#pragma unroll
        for (int r = 1; r < WW; ++r)
          if (r < world) acc.add(in[u][r]);
        uint4 raw[EPP / 4];
        from_wire<BF16>(acc.wire(), raw);
        grad_store<EPP>(P.grad, P.n, p, raw);
      }
    }
  }
  trace_stamp(P.trace, 3);
}

// ---- K2: two-shot ------------------------------------------------------------------------
// The bucket is cut into `world` slices of `slice` packs.  stage -> barrier -> rank r reduces
// slice r from all peers and overwrites slice r of its OWN staging buffer with the result ->
// barrier -> every rank reads slice s from rank s and writes its fp32 bucket.
// NVLink bytes per rank: 2 * (W-1)/W * N * w in (the bus-bandwidth convention of BASELINE.md).
// NVLS variant (K3): the reduce is one multimem.ld_reduce and the publish one multimem.st per
// pack; the all-gather read then becomes local.
template <int W, bool BF16, bool NVLS>
__global__ void __launch_bounds__(kThreads, 1) k2_two_shot_kernel(const __grid_constant__ ArParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  const int world = W > 0 ? W : P.world;
  const size_t npacks = (P.n + EPP - 1) / EPP;
  const size_t slice = (npacks + world - 1) / world;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  uint4* my_stage = reinterpret_cast<uint4*>(P.peers.arena[P.rank] + P.stage_off);
  trace_stamp(P.trace, 0);

  // phase 0: stage pack j of EVERY slice (peers' thread g will read exactly these);
  // UJ consecutive j per iteration so that 16 x 16-byte loads are in flight per thread
  {
    constexpr int LPP = BF16 ? 2 : 1;                       // 16-byte loads per pack
    constexpr int UJ = packs_per_batch(W * LPP);
    constexpr int B = WW * UJ;
    for (size_t j = g; j < slice; j += gt * UJ) {
      size_t p[B];
      bool ok[B];
#pragma unroll
      for (int u = 0; u < UJ; ++u) {
#pragma unroll
        for (int s = 0; s < WW; ++s) {
          const size_t jj = j + u * gt;
          p[u * WW + s] = static_cast<size_t>(s) * slice + jj;
          ok[u * WW + s] = s < world && jj < slice && p[u * WW + s] < npacks;
        }
      }
      stage_batch<BF16, B>(P.grad, P.n, my_stage, p, ok, P.scale);
    }
  }
  trace_stamp(P.trace, 1);
  block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
  trace_stamp(P.trace, 2);

  // phase 1: reduce my slice
  {
    const size_t base = static_cast<size_t>(P.rank) * slice;
    if constexpr (NVLS) {
      constexpr int U = kMaxLoadsInFlight;
      const uint4* mc = reinterpret_cast<const uint4*>(P.peers.mc_arena + P.stage_off);
      for (size_t j = g; j < slice; j += gt * U) {
        uint4 red[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t p = base + j + u * gt;
          if (j + u * gt < slice && p < npacks)
            red[u] = BF16 ? multimem_ld_reduce_bf16x8(mc + p) : multimem_ld_reduce_f32x4(mc + p);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t p = base + j + u * gt;
          if (j + u * gt < slice && p < npacks) multimem_st_v4(const_cast<uint4*>(mc) + p, red[u]);
        }
      }
    } else {
      constexpr int U = packs_per_batch(W);
      for (size_t j = g; j < slice; j += gt * U) {
        uint4 in[U][WW];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t p = base + j + u * gt;
          if (j + u * gt < slice && p < npacks) {
#pragma unroll
            for (int r = 0; r < WW; ++r)
              if (r < world)
                in[u][r] =
                    ld_peer_v4(reinterpret_cast<const uint4*>(P.peers.arena[r] + P.stage_off) + p);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t p = base + j + u * gt;
          if (j + u * gt < slice && p < npacks) {
            Acc<BF16> acc;
            acc.set(in[u][0]);
#pragma unroll
            for (int r = 1; r < WW; ++r)
              if (r < world) acc.add(in[u][r]);
            st_v4(my_stage + p, acc.wire());
          }
        }
      }
    }
  }
  trace_stamp(P.trace, 3);
  constexpr int UJ2 = packs_per_batch(W);
  constexpr int B2 = WW * UJ2;
  // one gather pass over this block's packs of the slices in `mask` (16 loads in flight per thread)
  auto gather = [&](uint32_t mask) {
    for (size_t j = g; j < slice; j += gt * UJ2) {
      uint4 in[B2];
      size_t p[B2];
      bool ok[B2];
#pragma unroll
      for (int u = 0; u < UJ2; ++u) {
#pragma unroll
        for (int s = 0; s < WW; ++s) {
          const int i = u * WW + s;
          const size_t jj = j + u * gt;
          p[i] = static_cast<size_t>(s) * slice + jj;
          ok[i] = s < world && ((mask >> s) & 1u) && jj < slice && p[i] < npacks;
          if (ok[i]) {
            const unsigned char* src = NVLS ? P.peers.arena[P.rank] : P.peers.arena[s];
            in[i] = ld_peer_v4(reinterpret_cast<const uint4*>(src + P.stage_off) + p[i]);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < B2; ++i) {
        if (ok[i]) {
          uint4 raw[EPP / 4];
          from_wire<BF16>(in[i], raw);
          grad_store<EPP>(P.grad, P.n, p[i], raw);
        }
      }
    }
  };
  // phase 2: all-gather + fp32 write-back after ONE barrier.  (An arrival-order variant — gather whichever
  // peers have finished first, barrier_arrive/poll_arrived in b2d_device.cuh — loses: every extra round pays
  // a full NVLink round trip.)
  block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
  trace_stamp(P.trace, 4);
  gather(world >= 32 ? 0xffffffffu : ((1u << world) - 1u));
  trace_stamp(P.trace, 5);
}

// ---- K4/K5/K6: sharded step ----------------------------------------------------------------
// The fp32 kernel arguments of torch's Adam / AdamW, each one cast of Python's float64 value (adam_consts in
// b2d_launch.cuh).
struct AdamConsts {
  float beta2, eps, weight_decay;
  float lerp_w;           // 1 - beta1, the weight of exp_avg.lerp_
  float lerp_w_rest;      // 1 - lerp_w in fp32: the factor of lerp's second branch
  float one_minus_beta2;
  float neg_step_size;    // -(lr / (1 - beta1^step))
  float bc2_sqrt;         // (1 - beta2^step) ** 0.5
  float decay_mul;        // 1 - lr * weight_decay (AdamW)
  int lerp_small;         // |lerp_w| < 0.5: lerp's first branch
  int l2;                 // Adam with weight_decay != 0: grad += weight_decay * param
  int decoupled;          // AdamW with weight_decay != 0: param *= decay_mul
};

struct ShParams {
  const float* grads;   // flat fp32 [n] local gradients (not necessarily in the arena)
  float* grads_rw;      // same pointer when zero_grads, else nullptr
  float* params;        // flat fp32 [n], own mapping; lives in the arena at byte param_off
  size_t param_off;
  float* exp_avg;       // own shard only
  float* exp_avg_sq;
  float* rs_out;        // reduce-scatter-only output (own shard) or nullptr
  size_t n;
  long long off[B2D_MAX_WORLD + 1];  // element offsets of the owner shards (multiples of 8)
  size_t stage_off;
  float scale;
  int rank, world;
  int do_stage_reduce;  // phases 0+1
  int do_adam;          // phase 1 applies Adam (else writes rs_out)
  int do_gather;        // phase 2
  int end_barrier;      // standalone all-gather: fence the shard against the caller's next write
  AdamConsts adam;
  unsigned long long timeout_ns;
  Diag* diag;
  Peers peers;
};

// One element of torch.optim.Adam / AdamW as torch runs it on CUDA with its default multi-tensor path
// (torch/optim/adam.py `_multi_tensor_adam`, non-capturable): one fp32 rounding per ATen operation, in torch's order,
// and a fused multiply-add exactly where ATen's kernel computes `a + b * c`.  Every operation is spelled out
// (__f*_rn), so that the compiler contracts nothing else and the host build of the emulator rounds identically.
__device__ __forceinline__ void adam_update(float g, float& p, float& m, float& v, const AdamConsts& a) {
  if (a.decoupled) {
    p = __fmul_rn(p, a.decay_mul);                              // _foreach_mul_(params, 1 - lr * weight_decay)
  } else if (a.l2) {
    g = __fmaf_rn(a.weight_decay, p, g);                        // _foreach_add(grads, params, alpha=weight_decay)
  }
  const float d = __fadd_rn(g, -m);                             // _foreach_lerp_(exp_avgs, grads, 1 - beta1):
  m = a.lerp_small ? __fmaf_rn(a.lerp_w, d, m)                  //   m + w * (g - m)             for |w| < 0.5,
                   : __fmaf_rn(-d, a.lerp_w_rest, g);           //   g - (g - m) * (1 - w)       otherwise (Lerp.h)
  v = __fmaf_rn(a.one_minus_beta2, __fmul_rn(g, g), __fmul_rn(v, a.beta2));  // _foreach_mul_(v, beta2), _foreach_addcmul_
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), a.bc2_sqrt), a.eps);  // _foreach_sqrt, _foreach_div_, _foreach_add_
  p = __fmaf_rn(a.neg_step_size, __fdiv_rn(m, denom), p);       // _foreach_addcdiv_(params, exp_avgs, denom, -step_size)
}

template <int W, bool BF16>
__global__ void __launch_bounds__(kThreads, 1) k456_sharded_kernel(const __grid_constant__ ShParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  const int world = W > 0 ? W : P.world;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  uint4* my_stage = reinterpret_cast<uint4*>(P.peers.arena[P.rank] + P.stage_off);

  size_t max_len = 0;  // longest shard in elements
#pragma unroll
  for (int s = 0; s < WW; ++s)
    if (s < world) {
      const size_t l = static_cast<size_t>(P.off[s + 1] - P.off[s]);
      max_len = l > max_len ? l : max_len;
    }

  if (P.do_stage_reduce) {
    // phase 0: stage pack j of every owner shard
    constexpr int B = BF16 ? 4 : 8;
    const size_t max_packs = max_len / EPP;
    for (size_t j = g; j < max_packs; j += gt) {
      for (int s0 = 0; s0 < world; s0 += B) {
        size_t p[B];
        bool ok[B];
        uint4 raw[B][EPP / 4];
#pragma unroll
        for (int i = 0; i < B; ++i) {
          const int s = s0 + i;
          ok[i] = s < world && j < static_cast<size_t>(P.off[s + 1] - P.off[s]) / EPP;
          p[i] = ok[i] ? static_cast<size_t>(P.off[s]) / EPP + j : 0;
        }
#pragma unroll
        for (int i = 0; i < B; ++i)
          if (ok[i]) grad_load<EPP>(P.grads, P.n, p[i], raw[i]);
#pragma unroll
        for (int i = 0; i < B; ++i)
          if (ok[i]) {
            st_v4(my_stage + p[i], to_wire<BF16>(raw[i], P.scale));
            if (P.grads_rw != nullptr) {
              const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
              for (int q = 0; q < EPP / 4; ++q) st_v4(P.grads_rw + p[i] * EPP + 4 * q, z);
            }
          }
      }
    }
    block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);

    // phase 1: reduce the owned shard; Adam in registers on the reduced gradient
    const size_t my_off = static_cast<size_t>(P.off[P.rank]);
    const size_t my_packs = static_cast<size_t>(P.off[P.rank + 1] - P.off[P.rank]) / EPP;
    constexpr int U = (W > 0 && W <= 4) ? 2 : 1;  // p/m/v rows ride along: keep the batch small
    for (size_t j = g; j < my_packs; j += gt * U) {
      uint4 in[U][WW];
      uint4 pr[U][EPP / 4], mr[U][EPP / 4], vr[U][EPP / 4];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t jj = j + u * gt;
        if (jj < my_packs) {
          const size_t p = my_off / EPP + jj;
#pragma unroll
          for (int r = 0; r < WW; ++r)
            if (r < world)
              in[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(P.peers.arena[r] + P.stage_off) + p);
          if (P.do_adam) {
#pragma unroll
            for (int q = 0; q < EPP / 4; ++q) {
              pr[u][q] = ld_stream_v4(P.params + my_off + jj * EPP + 4 * q);
              mr[u][q] = ld_stream_v4(P.exp_avg + jj * EPP + 4 * q);
              vr[u][q] = ld_stream_v4(P.exp_avg_sq + jj * EPP + 4 * q);
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t jj = j + u * gt;
        if (jj < my_packs) {
          Acc<BF16> acc;
          acc.set(in[u][0]);
#pragma unroll
          for (int r = 1; r < WW; ++r)
            if (r < world) acc.add(in[u][r]);
          if (P.do_adam) {
#pragma unroll
            for (int q = 0; q < EPP / 4; ++q) {
              float pp[4] = {__uint_as_float(pr[u][q].x), __uint_as_float(pr[u][q].y),
                             __uint_as_float(pr[u][q].z), __uint_as_float(pr[u][q].w)};
              float mm[4] = {__uint_as_float(mr[u][q].x), __uint_as_float(mr[u][q].y),
                             __uint_as_float(mr[u][q].z), __uint_as_float(mr[u][q].w)};
              float vv[4] = {__uint_as_float(vr[u][q].x), __uint_as_float(vr[u][q].y),
                             __uint_as_float(vr[u][q].z), __uint_as_float(vr[u][q].w)};
#pragma unroll
              for (int k = 0; k < 4; ++k) adam_update(acc.v[4 * q + k], pp[k], mm[k], vv[k], P.adam);
              st_v4(P.params + my_off + jj * EPP + 4 * q,
                    make_uint4(__float_as_uint(pp[0]), __float_as_uint(pp[1]), __float_as_uint(pp[2]),
                               __float_as_uint(pp[3])));
              st_v4(P.exp_avg + jj * EPP + 4 * q,
                    make_uint4(__float_as_uint(mm[0]), __float_as_uint(mm[1]), __float_as_uint(mm[2]),
                               __float_as_uint(mm[3])));
              st_v4(P.exp_avg_sq + jj * EPP + 4 * q,
                    make_uint4(__float_as_uint(vv[0]), __float_as_uint(vv[1]), __float_as_uint(vv[2]),
                               __float_as_uint(vv[3])));
            }
          } else {
#pragma unroll
            for (int q = 0; q < EPP / 4; ++q)
              st_v4(P.rs_out + jj * EPP + 4 * q,
                    make_uint4(__float_as_uint(acc.v[4 * q]), __float_as_uint(acc.v[4 * q + 1]),
                               __float_as_uint(acc.v[4 * q + 2]), __float_as_uint(acc.v[4 * q + 3])));
          }
        }
      }
    }
  }

  if (P.do_gather) {
    // phase 2: pull every other owner's updated fp32 parameters.
    // The unit is the SAME pack (EPP elements) with the same (block, thread) -> pack mapping as in the
    // Adam phase: owner s's per-block flag only vouches for what owner s's block b wrote.
    constexpr int Q = EPP / 4;                               // 16-byte fp32 loads per pack
    constexpr int B = (W > 0) ? (W * Q > 16 ? 16 / Q : W) : 4;
    const size_t max_packs = max_len / EPP;
    block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
    const uint32_t mask = ((1u << world) - 1u) & ~(1u << P.rank);   // the own shard is already in place
    {
      for (size_t j = g; j < max_packs; j += gt) {
        for (int s0 = 0; s0 < world; s0 += B) {
          uint4 in[B][Q];
          bool ok[B];
#pragma unroll
          for (int i = 0; i < B; ++i) {
            const int s = s0 + i;
            ok[i] = s < world && ((mask >> s) & 1u) && j < static_cast<size_t>(P.off[s + 1] - P.off[s]) / EPP;
            if (ok[i]) {
#pragma unroll
              for (int q = 0; q < Q; ++q)
                in[i][q] = ld_peer_v4(reinterpret_cast<const float*>(P.peers.arena[s] + P.param_off) +
                                      static_cast<size_t>(P.off[s]) + j * EPP + 4 * q);
            }
          }
#pragma unroll
          for (int i = 0; i < B; ++i) {
            if (ok[i]) {
#pragma unroll
              for (int q = 0; q < Q; ++q)
                st_v4(P.params + static_cast<size_t>(P.off[s0 + i]) + j * EPP + 4 * q, in[i][q]);
            }
          }
        }
      }
    }
    if (P.end_barrier) block_barrier(P.peers, P.rank, world, P.timeout_ns, P.diag);
  }
}

// ---- standalone barrier ------------------------------------------------------------------
__global__ void __launch_bounds__(32) barrier_kernel(const __grid_constant__ ArParams P) {
  block_barrier(P.peers, P.rank, P.world, P.timeout_ns, P.diag);
}

}  // namespace b2d
