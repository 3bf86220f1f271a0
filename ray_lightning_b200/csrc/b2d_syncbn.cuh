// b2d_syncbn.cuh — synchronised BatchNorm statistics over peer stores (K15..K17).
//
// torch's SyncBatchNorm (torch/nn/modules/_functions.py) gathers every rank's per-channel statistics with a cat +
// NCCL all_gather_into_tensor + a host-side mask + batch_norm_gather_stats_with_counts in forward (:65-115), and
// sums the per-channel gradient reductions with a cat + NCCL all_reduce + split in backward (:155-165).  Here:
//
//     K15  bn_push_kernel     one CTA   writes this rank's row into row `rank` of the layer's region in EVERY rank's
//                                       arena (16-byte stores), then arrives: bn[rank] = epoch in every peer's pad
//     K16  bn_combine_kernel  waits (at its start only) until bn[src] >= epoch for every src, then merges the W
//          <FWD = true>       forward rows per channel in rank order (Chan's parallel variance, rows with count 0
//                             skipped) -> mean, invstd, counts and, optionally, the running statistics in place
//     K17  bn_combine_kernel  the same wait, then the rank-ordered fp32 sum of the W backward rows
//          <FWD = false>
//
// Rows, in fp32:  forward  [mean[0..C) | invstd[0..C) | count | pad]    backward  [sum_dy[0..C) | sum_dy_xmu[0..C) | pad]
// padded to a multiple of 4 floats, so every row starts 16-byte aligned and the peer stores are all 16-byte vectors.
// The sources are read element by element: the second half of a row starts at C, which need not be a multiple of 4.
//
// Every arithmetic step is one correctly rounded fp32 operation (__fadd_rn, __fmul_rn, __fdiv_rn, __fsqrt_rn): a
// float32 restatement reproduces the outputs bit for bit, and every rank computes identical bits.
//
// Signalling: the BN exchanges run on the caller's compute stream while bucket exchanges run on the library's internal
// streams, so they have their own monotone word per source (Signal::bn) and their own host epoch counter.  A region is
// double-buffered per layer and direction (generation = parity of the layer's call count): a rank can only push into a
// generation again after it has combined the exchange in between, which needs every peer's push of that exchange, which
// every peer issues only after it has combined the exchange that last used the generation (DESIGN.md §5).
#pragma once

#include "b2d_staged.cuh"

namespace b2d {

constexpr int kBnThreads = 256;

// floats per row
__host__ __device__ __forceinline__ size_t bn_fwd_row(int channels) { return (2 * static_cast<size_t>(channels) + 1 + 3) / 4 * 4; }
__host__ __device__ __forceinline__ size_t bn_bwd_row(int channels) { return (2 * static_cast<size_t>(channels) + 3) / 4 * 4; }

struct BnPushParams {
  const float* a;       // mean | sum_dy        (C floats; NULL: zeros)
  const float* b;       // invstd | sum_dy_xmu  (C floats; NULL: zeros)
  float count;          // forward: this rank's elements per channel (0: an empty rank)
  int channels;
  int fwd;
  size_t region_off;    // byte offset, in every arena, of this generation's W rows
  int rank, world;
  uint32_t epoch;
  Peers peers;
};

struct BnCombineParams {
  size_t region_off;
  int channels;
  float eps, momentum;
  float* out_a;          // mean | sum_dy
  float* out_b;          // invstd | sum_dy_xmu
  int32_t* counts;       // forward: [W] (zeros kept)
  float* running_mean;   // forward, optional
  float* running_var;    // forward, optional
  int rank, world;
  uint32_t epoch;
  unsigned long long timeout_ns;
  Diag* diag;
  Peers peers;
};

__device__ __forceinline__ float ld_row(const float* p) { return __uint_as_float(ld_flag(reinterpret_cast<const uint32_t*>(p))); }

// ---- K15 ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBnThreads) bn_push_kernel(const __grid_constant__ BnPushParams P) {
  const int C = P.channels;
  const size_t row = P.fwd ? bn_fwd_row(C) : bn_bwd_row(C);
  const size_t row_byte = static_cast<size_t>(P.rank) * row * 4;
  for (size_t v = threadIdx.x; v < row / 4; v += blockDim.x) {
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const size_t i = 4 * v + k;
      float x = 0.f;
      if (i < static_cast<size_t>(C)) x = P.a != nullptr ? P.a[i] : 0.f;
      else if (i < 2 * static_cast<size_t>(C)) x = P.b != nullptr ? P.b[i - C] : 0.f;
      else if (P.fwd && i == 2 * static_cast<size_t>(C)) x = P.count;
      w[k] = __float_as_uint(x);
    }
    const uint4 u = make_uint4(w[0], w[1], w[2], w[3]);
    for (int p = 0; p < P.world; ++p) st_v4(P.peers.arena[p] + P.region_off + row_byte + v * 16, u);
  }
  __syncthreads();
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    fence_sys();   // release: the block's row stores, cumulative over bar.sync
    st_flag(&P.peers.signal[threadIdx.x]->bn[P.rank], P.epoch);
  }
}

// ---- K16 / K17 ---------------------------------------------------------------------------------------------------
template <bool FWD>
__global__ void __launch_bounds__(kBnThreads) bn_combine_kernel(const __grid_constant__ BnCombineParams P) {
  Signal* self = P.peers.signal[P.rank];
  if (threadIdx.x < static_cast<unsigned>(P.world)) {
    spin_until_ge(&self->bn[threadIdx.x], P.epoch, P.timeout_ns, P.diag, P.rank, threadIdx.x);
    fence_sys();   // acquire
  }
  __syncthreads();
  const int C = P.channels;
  const size_t row = FWD ? bn_fwd_row(C) : bn_bwd_row(C);
  const float* rows = reinterpret_cast<const float*>(P.peers.arena[P.rank] + P.region_off);
  if (FWD && blockIdx.x == 0 && threadIdx.x < static_cast<unsigned>(P.world))
    P.counts[threadIdx.x] = static_cast<int32_t>(ld_row(rows + threadIdx.x * row + 2 * C));
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    if constexpr (FWD) {
      // ATen's batch_norm_reduce_statistics_kernel (Normalization.cuh, recalled), one rounding per operation, with
      // the rows of empty ranks skipped on the device instead of masked out on the host (_functions.py:88-100)
      float avg = 0.f, var_n = 0.f, n = 0.f;
      for (int j = 0; j < P.world; ++j) {
        const float* r = rows + j * row;
        const float cnt = ld_row(r + 2 * C);
        if (cnt == 0.f) continue;
        const float m = ld_row(r + c);
        float v = __fdiv_rn(1.f, ld_row(r + C + c));
        v = __fmul_rn(__fadd_rn(__fmul_rn(v, v), -P.eps), cnt);
        const float factor = __fdiv_rn(1.f, __fadd_rn(n, cnt));
        const float d = __fadd_rn(avg, -m);
        var_n = __fadd_rn(var_n, __fadd_rn(v, __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), n), cnt), factor)));
        avg = __fadd_rn(__fmul_rn(__fmul_rn(n, factor), avg), __fmul_rn(__fmul_rn(cnt, factor), m));
        n = __fadd_rn(n, cnt);
      }
      P.out_a[c] = avg;
      P.out_b[c] = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fdiv_rn(var_n, n), P.eps)));
      const float keep = __fadd_rn(1.f, -P.momentum);
      if (P.running_mean != nullptr)
        P.running_mean[c] = __fadd_rn(__fmul_rn(keep, P.running_mean[c]), __fmul_rn(P.momentum, avg));
      if (P.running_var != nullptr) {
        const float unbiased = __fdiv_rn(var_n, __fadd_rn(n, -1.f));
        P.running_var[c] = __fadd_rn(__fmul_rn(keep, P.running_var[c]), __fmul_rn(P.momentum, unbiased));
      }
    } else {
      float sa = ld_row(rows + c), sb = ld_row(rows + C + c);
      for (int j = 1; j < P.world; ++j) {
        sa = __fadd_rn(sa, ld_row(rows + j * row + c));
        sb = __fadd_rn(sb, ld_row(rows + j * row + C + c));
      }
      P.out_a[c] = sa;
      P.out_b[c] = sb;
    }
  }
}

}  // namespace b2d
