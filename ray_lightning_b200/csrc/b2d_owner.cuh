// b2d_owner.cuh — the sharded path on the staged machinery (K11..K13): what FairScale's ShardedDataParallel + OSS
// do for RayShardedStrategy (ray_lightning/ray_ddp_sharded.py:12-13), cut the way the reference cuts it in TIME —
// gradients travel to their owners WHILE backward runs, the optimizer step only pays for the parameter exchange:
//
//     during backward, per reduce bucket (a set of parameters that become ready together):
//       K11 seg_stage_kernel    local   the bucket's gradient segments, grouped by owner rank, are cast + scaled
//                                       into ONE contiguous staging region of the own arena (and zeroed in place);
//                                       last block arrives (staged[rank] = epoch)
//       K12 seg_reduce_kernel   NVLink  rank r waits for every rank's `staged`, reads ITS sub-range of the staging
//                                       region from all W arenas (or one multimem.ld_reduce), adds in rank order in
//                                       fp32 and writes fp32 into its local reduced-gradient shard
//     at optimizer.step():
//       K13 adam_push_kernel    NVLink  Adam on the owned shard in registers (torch.optim.Adam arithmetic, per
//                                       parameter group), new parameters PUSHED into every rank's flat parameter
//                                       buffer (W peer stores, or one multimem.st); last block arrives (published)
//           wait_published_kernel       one warp; after it the parameters are whole on this rank
//
// Like b2d_staged.cuh, no kernel waits after it has signalled, so the phases of several loopback ranks can be
// issued phase-major and survive a serialising profiler.  A bucket's segments are (flat offset, length) runs of the
// flat gradient space (8-element aligned, whole packs); the table is sorted by owner, so an owner's share of the
// bucket is one contiguous range of the staging region and lands in its reduced shard at (flat offset - shard start).
#pragma once

#include "b2d_staged.cuh"

namespace b2d {

struct SegParams {
  const long long* seg_flat_off;   // [nseg] element offset of each segment in the flat gradient space (device memory)
  const unsigned* seg_start;       // [nseg + 1] first staging pack of each segment, cumulative (device memory)
  int nseg;
  unsigned owner_pack[B2D_MAX_WORLD + 1];   // staging packs [owner_pack[r], owner_pack[r+1]) belong to owner r
  float* grads;          // flat fp32 gradients (local)
  float* reduced;        // own reduced-gradient shard, fp32, indexed by (flat offset - shard_lo)
  long long shard_lo;    // first flat element of the own shard
  size_t wire_off;       // byte offset of the bucket's staging region in every arena
  float scale;
  int zero_grads;        // K11: overwrite the local gradients with 0 once staged
  int accumulate;        // K12: reduced += sum (gradient accumulation) instead of reduced = sum
  int rank, world;
  uint32_t epoch;
  unsigned long long timeout_ns;
  Diag* diag;
  Peers peers;
};

// segment that holds staging pack q: the last i with seg_start[i] <= q
__device__ __forceinline__ int seg_find(const unsigned* seg_start, int nseg, unsigned q) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg_start[mid] <= q) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- K11 -------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(kStThreads, 4) seg_stage_kernel(const __grid_constant__ SegParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  constexpr int B = BF16 ? 4 : 8;
  const unsigned total = P.seg_start[P.nseg];
  uint4* wire = reinterpret_cast<uint4*>(P.peers.arena[P.rank] + P.wire_off);
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t j = g; j < total; j += gt * B) {
    uint4 raw[B][EPP / 4];
    float* src[B];
#pragma unroll
    for (int i = 0; i < B; ++i) {
      const size_t q = j + i * gt;
      src[i] = nullptr;
      if (q < total) {
        const int s = seg_find(P.seg_start, P.nseg, static_cast<unsigned>(q));
        src[i] = P.grads + P.seg_flat_off[s] + static_cast<size_t>(q - P.seg_start[s]) * EPP;
#pragma unroll
        for (int k = 0; k < EPP / 4; ++k) raw[i][k] = ld_stream_v4(src[i] + 4 * k);
      }
    }
#pragma unroll
    for (int i = 0; i < B; ++i) {
      if (src[i] != nullptr) {
        st_v4(wire + j + i * gt, to_wire<BF16>(raw[i], P.scale));
        if (P.zero_grads) {
          const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
          for (int k = 0; k < EPP / 4; ++k) st_v4(src[i] + 4 * k, z);
        }
      }
    }
  }
  arrive_when_grid_done(P.peers, P.rank, P.world, 0, P.epoch);
}

// ---- K12 -------------------------------------------------------------------------------------------------
template <int W, bool BF16, bool NVLS>
__global__ void __launch_bounds__(kExThreads, 2) seg_reduce_kernel(const __grid_constant__ SegParams P) {
  constexpr int EPP = BF16 ? 8 : 4;
  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  const int world = W > 0 ? W : P.world;
  Signal* self = P.peers.signal[P.rank];
  if (threadIdx.x < static_cast<unsigned>(world)) {
    spin_until_ge(&self->staged[threadIdx.x], P.epoch, P.timeout_ns, P.diag, P.rank, threadIdx.x);
    fence_sys();
  }
  __syncthreads();
  const unsigned q0 = P.owner_pack[P.rank], q1 = P.owner_pack[P.rank + 1];
  const size_t cnt = q1 - q0;
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  constexpr int U = NVLS ? 8 : packs_per_batch(W);
  for (size_t j = g; j < cnt; j += gt * U) {
    uint4 in[U][NVLS ? 1 : WW];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t q = q0 + j + u * gt;
      if (j + u * gt < cnt) {
        if constexpr (NVLS) {
          const uint4* mc = reinterpret_cast<const uint4*>(P.peers.mc_arena + P.wire_off) + q;
          in[u][0] = BF16 ? multimem_ld_reduce_bf16x8(mc) : multimem_ld_reduce_f32x4(mc);
        } else {
#pragma unroll
          for (int r = 0; r < WW; ++r)
            if (r < world) in[u][r] = ld_peer_v4(reinterpret_cast<const uint4*>(P.peers.arena[r] + P.wire_off) + q);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t q = q0 + j + u * gt;
      if (j + u * gt < cnt) {
        Acc<BF16> acc;
        acc.set(in[u][0]);
        if constexpr (!NVLS) {
#pragma unroll
          for (int r = 1; r < WW; ++r)
            if (r < world) acc.add(in[u][r]);
        }
        const int s = seg_find(P.seg_start, P.nseg, static_cast<unsigned>(q));
        float* dst = P.reduced + (P.seg_flat_off[s] - P.shard_lo) + static_cast<size_t>(q - P.seg_start[s]) * EPP;
#pragma unroll
        for (int k = 0; k < EPP / 4; ++k) {
          float o[4] = {acc.v[4 * k], acc.v[4 * k + 1], acc.v[4 * k + 2], acc.v[4 * k + 3]};
          if (P.accumulate) {
            const uint4 old = ld_stream_v4(dst + 4 * k);
            o[0] = __fadd_rn(__uint_as_float(old.x), o[0]); o[1] = __fadd_rn(__uint_as_float(old.y), o[1]);
            o[2] = __fadd_rn(__uint_as_float(old.z), o[2]); o[3] = __fadd_rn(__uint_as_float(old.w), o[3]);
          }
          st_v4(dst + 4 * k, make_uint4(__float_as_uint(o[0]), __float_as_uint(o[1]), __float_as_uint(o[2]), __float_as_uint(o[3])));
        }
      }
    }
  }
}

// ---- K13 -------------------------------------------------------------------------------------------------
constexpr int kMaxAdamGroups = 8;

struct PushParams {
  float* params;          // own mapping of the flat fp32 parameters (in the arena, byte offset param_off)
  size_t param_off;
  float* exp_avg;         // own shard, fp32 [hi - lo]
  float* exp_avg_sq;
  const float* reduced;   // own reduced-gradient shard
  long long lo, hi;       // own shard in flat elements (multiples of 8)
  int ngroups;            // 0: push only (the caller's optimizer has already updated the shard)
  long long group_lo[kMaxAdamGroups], group_hi[kMaxAdamGroups];   // element ranges relative to `lo`
  AdamConsts group[kMaxAdamGroups];
  int rank, world;
  uint32_t epoch;
  Peers peers;
  const float* grad_scale;   // adam_push_scaled_kernel: device fp32 factor applied to every gradient (clip coefficient)
};

// SCALED: g = g * (*grad_scale) before the update, one rounding — torch's `grad.mul_(clip_coef)` followed by the step
template <int W, bool NVLS, bool SCALED>
__device__ __forceinline__ void adam_push_body(const PushParams& P) {
  constexpr int WW = W > 0 ? W : B2D_MAX_WORLD;
  const int world = W > 0 ? W : P.world;
  const size_t nv = static_cast<size_t>(P.hi - P.lo) / 4;   // 16-byte vectors of the own shard
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  constexpr int U = 2;
  float gscale = 1.f;
  if constexpr (SCALED) gscale = *P.grad_scale;
  for (size_t j = g; j < nv; j += gt * U) {
    uint4 pr[U], gr[U], mr[U], vr[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t i = j + u * gt;
      if (i < nv) {
        pr[u] = ld_stream_v4(P.params + P.lo + 4 * i);
        if (P.ngroups > 0) {
          gr[u] = ld_stream_v4(P.reduced + 4 * i);
          mr[u] = ld_stream_v4(P.exp_avg + 4 * i);
          vr[u] = ld_stream_v4(P.exp_avg_sq + 4 * i);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t i = j + u * gt;
      if (i < nv) {
        uint4 out = pr[u];
        if (P.ngroups > 0) {
          int gi = -1;
          for (int k = 0; k < P.ngroups; ++k)
            if (static_cast<long long>(4 * i) >= P.group_lo[k] && static_cast<long long>(4 * i) < P.group_hi[k]) gi = k;
          if (gi >= 0) {
            float pp[4] = {__uint_as_float(pr[u].x), __uint_as_float(pr[u].y), __uint_as_float(pr[u].z), __uint_as_float(pr[u].w)};
            float gg[4] = {__uint_as_float(gr[u].x), __uint_as_float(gr[u].y), __uint_as_float(gr[u].z), __uint_as_float(gr[u].w)};
            float mm[4] = {__uint_as_float(mr[u].x), __uint_as_float(mr[u].y), __uint_as_float(mr[u].z), __uint_as_float(mr[u].w)};
            float vv[4] = {__uint_as_float(vr[u].x), __uint_as_float(vr[u].y), __uint_as_float(vr[u].z), __uint_as_float(vr[u].w)};
            if constexpr (SCALED) {
#pragma unroll
              for (int k = 0; k < 4; ++k) gg[k] = __fmul_rn(gg[k], gscale);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) adam_update(gg[k], pp[k], mm[k], vv[k], P.group[gi]);
            out = make_uint4(__float_as_uint(pp[0]), __float_as_uint(pp[1]), __float_as_uint(pp[2]), __float_as_uint(pp[3]));
            st_v4(P.exp_avg + 4 * i, make_uint4(__float_as_uint(mm[0]), __float_as_uint(mm[1]), __float_as_uint(mm[2]), __float_as_uint(mm[3])));
            st_v4(P.exp_avg_sq + 4 * i, make_uint4(__float_as_uint(vv[0]), __float_as_uint(vv[1]), __float_as_uint(vv[2]), __float_as_uint(vv[3])));
          }
        }
        const size_t byte = P.param_off + (static_cast<size_t>(P.lo) + 4 * i) * 4;
        if constexpr (NVLS) {
          multimem_st_v4(P.peers.mc_arena + byte, out);
        } else {
#pragma unroll
          for (int r = 0; r < WW; ++r)
            if (r < world) st_v4(P.peers.arena[r] + byte, out);
        }
      }
    }
  }
  arrive_when_grid_done(P.peers, P.rank, P.world, 1, P.epoch);
}

template <int W, bool NVLS>
__global__ void __launch_bounds__(kExThreads, 2) adam_push_kernel(const __grid_constant__ PushParams P) {
  adam_push_body<W, NVLS, false>(P);
}

// K13 with the clip coefficient of K19 (b2d_clip.cuh) applied to the gradients
template <int W, bool NVLS>
__global__ void __launch_bounds__(kExThreads, 2) adam_push_scaled_kernel(const __grid_constant__ PushParams P) {
  adam_push_body<W, NVLS, true>(P);
}

// ---- K14: optimizer step of one DDP bucket, right behind its allreduce (SURVEY §8 f-2) --------------------------
// Replaces torch's `_hook_then_optimizer` (optimizer_overlap_hooks.py:131-163: allreduce future .then(functional
// optimizer per parameter)).  The bucket's averaged gradients are contiguous; its parameters are separate
// allocations, so the kernel walks a small table (first bucket element of each parameter, cumulative) and touches
// parameters with coalesced 4-byte accesses.  Optimizer state (momentum buffer, or exp_avg / exp_avg_sq) is one
// tensor per parameter, owned by the caller (it survives DDP's bucket re-layout).  Arithmetic is torch.optim.SGD's
// on CUDA (sgd.py, dampening 0, no nesterov; both of torch's paths issue the same element-wise operations) and
// torch.optim.Adam / AdamW's (adam_update above), bit for bit.
struct OptimParams {
  float* const* param_ptr;      // [nseg] device table: start of each parameter
  const unsigned* seg_start;    // [nseg + 1] first bucket element of each parameter, cumulative
  int nseg;
  const float* grads;           // the bucket (averaged gradients), n elements
  size_t n;
  float* const* state1_ptr;     // [nseg] momentum buffer | exp_avg      of each parameter
  float* const* state2_ptr;     // [nseg] unused          | exp_avg_sq
  int kind;                     // 0 SGD, 1 Adam / AdamW
  float lr, momentum, weight_decay;
  int first_step;               // SGD: the momentum buffer starts as a copy of the gradient (torch.clone(grad))
  AdamConsts adam;
};

__global__ void __launch_bounds__(kStThreads) bucket_optim_kernel(const __grid_constant__ OptimParams P) {
  const size_t gt = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < P.n; e += gt) {
    const int s = seg_find(P.seg_start, P.nseg, static_cast<unsigned>(e));
    const size_t k = e - P.seg_start[s];
    float* pp = P.param_ptr[s] + k;
    float g = P.grads[e], p = *pp;
    if (P.kind == 0) {
      if (P.weight_decay != 0.f) g = __fmaf_rn(P.weight_decay, p, g);  // grad = grad.add(param, alpha=weight_decay)
      if (P.momentum != 0.f) {
        float* bp = P.state1_ptr[s] + k;
        // buf = torch.clone(grad) on the first step, then buf.mul_(momentum).add_(grad): two roundings
        const float b = P.first_step ? g : __fadd_rn(__fmul_rn(P.momentum, *bp), g);
        *bp = b;
        g = b;
      }
      *pp = __fmaf_rn(-P.lr, g, p);                                    // param.add_(grad, alpha=-lr)
    } else {
      float* mp = P.state1_ptr[s] + k;
      float* vp = P.state2_ptr[s] + k;
      float m = *mp, v = *vp;
      adam_update(g, p, m, v, P.adam);
      *pp = p; *mp = m; *vp = v;
    }
  }
}

}  // namespace b2d
