// b2d_launch.cuh — the host-side decisions around the kernel launches that b2d.cu and the CPU emulator
// (emu/emu_harness.cpp) share: which template specialisation of a kernel family the runtime choices select, the
// peer-wait fields of a kernel's parameters, Adam's host constants, the chunk geometry of the staged exchange and the
// owner-segment table of a reduce bucket.  Pure host code without CUDA runtime calls, so that the emulated launches
// exercise the very decisions the library makes.
#pragma once

#include <math.h>

#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "b2d_kernels.cuh"
#include "b2d_owner.cuh"
#include "b2d_staged.cuh"
#include "b2d_syncbn.cuh"

namespace b2d {

// The kernels that read peers are specialised for 2, 4 and 8 ranks; W = 0 is the generic build for any other world
// size.  Returns f(std::integral_constant<int, W>{}) for the specialisation that `world` runs.
template <typename F>
auto dispatch_world(int world, F&& f) {
  switch (world) {
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    default: return f(std::integral_constant<int, 0>{});
  }
}

// ---- kernel selectors ----------------------------------------------------------------------------------------------
// One per templated kernel family: the runtime choices in, the kernel to launch out.  The library launches
// select_...(...)<<<grid, block, smem, stream>>>(P), the emulator calls the returned function, and b2d.cu's
// preload_kernels walks every selector over its whole domain, so any kernel a selector can return is loaded up front.
// (K2T's selector lives in b2d.cu: the emulator does not compile b2d_tma.cuh.)
inline auto select_k0(bool bf16) { return bf16 ? &k0_cast_scale_kernel<true> : &k0_cast_scale_kernel<false>; }

inline auto select_k1(int world, bool bf16) {
  return dispatch_world(world, [=](auto w) {
    constexpr int W = decltype(w)::value;
    return bf16 ? &k1_one_shot_kernel<W, true> : &k1_one_shot_kernel<W, false>;
  });
}

inline auto select_k2(int world, bool bf16, bool nvls_fused) {
  return dispatch_world(world, [=](auto w) {
    constexpr int W = decltype(w)::value;
    if (bf16) return nvls_fused ? &k2_two_shot_kernel<W, true, true> : &k2_two_shot_kernel<W, true, false>;
    return nvls_fused ? &k2_two_shot_kernel<W, false, true> : &k2_two_shot_kernel<W, false, false>;
  });
}

inline auto select_k456(int world, bool bf16) {
  return dispatch_world(world, [=](auto w) {
    constexpr int W = decltype(w)::value;
    return bf16 ? &k456_sharded_kernel<W, true> : &k456_sharded_kernel<W, false>;
  });
}

inline auto select_stage(bool bf16) { return bf16 ? &stage_kernel<true> : &stage_kernel<false>; }
inline auto select_unstage(bool bf16) { return bf16 ? &unstage_kernel<true> : &unstage_kernel<false>; }

// An in-place exchange reads the fp32 bucket itself, so `inplace` ignores `bf16`: there is no bf16 in-place kernel.
inline auto select_exch(int world, bool bf16, bool nvls, bool inplace) {
  return dispatch_world(world, [=](auto w) {
    constexpr int W = decltype(w)::value;
    if (inplace) return nvls ? &exch_kernel<W, false, true, true> : &exch_kernel<W, false, false, true>;
    if (bf16) return nvls ? &exch_kernel<W, true, true, false> : &exch_kernel<W, true, false, false>;
    return nvls ? &exch_kernel<W, false, true, false> : &exch_kernel<W, false, false, false>;
  });
}

inline auto select_seg_stage(bool bf16) { return bf16 ? &seg_stage_kernel<true> : &seg_stage_kernel<false>; }

inline auto select_seg_reduce(int world, bool bf16, bool nvls) {
  return dispatch_world(world, [=](auto w) {
    constexpr int W = decltype(w)::value;
    if (bf16) return nvls ? &seg_reduce_kernel<W, true, true> : &seg_reduce_kernel<W, true, false>;
    return nvls ? &seg_reduce_kernel<W, false, true> : &seg_reduce_kernel<W, false, false>;
  });
}

// scaled: K13 with the gradients multiplied by *grad_scale on the device (adam_push_scaled_kernel)
inline auto select_adam_push(int world, bool nvls, bool scaled) {
  return dispatch_world(world, [=](auto w) {
    constexpr int W = decltype(w)::value;
    if (scaled) return nvls ? &adam_push_scaled_kernel<W, true> : &adam_push_scaled_kernel<W, false>;
    return nvls ? &adam_push_kernel<W, true> : &adam_push_kernel<W, false>;
  });
}

inline auto select_bn_combine(bool fwd) { return fwd ? &bn_combine_kernel<true> : &bn_combine_kernel<false>; }

// The fields of a kernel's parameters that let it wait for peers: who is who, and the watchdog (0: never trap).
template <typename Params>
void set_peer_wait(Params* P, int rank, int world, const Peers& peers, unsigned long long timeout_ns, Diag* diag) {
  P->rank = rank;
  P->world = world;
  P->peers = peers;
  P->timeout_ns = timeout_ns;
  P->diag = diag;
}

// Most blocks the global-norm kernel K18 (b2d_clip.cuh) runs: its summation order depends on this value and on the
// element count only, never on the device.  At most kClipThreads, the width of the final tree.
constexpr unsigned kClipGMax = 256;

// torch/optim/adam.py's host arithmetic on Python floats (`1 - beta2`, `beta1 ** step`, `lr / bias_correction1`,
// `bias_correction2 ** 0.5`, `1 - lr * weight_decay`) in double with the same libm pow, then one cast to fp32 each, as
// ATen casts a Python scalar for its kernels.
inline AdamConsts adam_consts(const b2d_adam64& adam) {
  AdamConsts a{};
  a.beta2 = static_cast<float>(adam.beta2);
  a.eps = static_cast<float>(adam.eps);
  a.weight_decay = static_cast<float>(adam.weight_decay);
  a.lerp_w = static_cast<float>(1.0 - adam.beta1);
  a.lerp_w_rest = 1.0f - a.lerp_w;                             // Lerp.h computes `1 - weight` in fp32
  a.lerp_small = fabsf(a.lerp_w) < 0.5f;
  a.one_minus_beta2 = static_cast<float>(1.0 - adam.beta2);
  const double bc1 = 1.0 - pow(adam.beta1, static_cast<double>(adam.step));
  const double bc2 = 1.0 - pow(adam.beta2, static_cast<double>(adam.step));
  a.neg_step_size = static_cast<float>(adam.lr / bc1 * -1.0);
  a.bc2_sqrt = static_cast<float>(pow(bc2, 0.5));
  a.decay_mul = static_cast<float>(1.0 - adam.lr * adam.weight_decay);
  a.l2 = !adam.adamw && adam.weight_decay != 0.0;
  a.decoupled = adam.adamw && adam.weight_decay != 0.0;
  return a;
}

// The fp32 hyper-parameters of b2d_adam, widened exactly: the constants are then formed from the rounded values.
inline b2d_adam64 adam64(const b2d_adam& a) {
  return b2d_adam64{a.lr, a.beta1, a.beta2, a.eps, a.weight_decay, a.step, a.adamw, a.zero_grads, 0};
}

// Chunk c of a staged exchange of n elements: npacks wire packs of epp elements, chunk_packs packs per chunk.
struct ChunkSpan {
  size_t p0;        // first pack of the chunk
  size_t packs;     // packs in the chunk
  size_t n;         // elements of the bucket in the chunk (S and U)
  size_t n_valid;   // fp32 elements in the chunk when the bucket is exchanged in place (X; the last pack may be partial)
};

inline ChunkSpan chunk_span(int c, size_t npacks, size_t chunk_packs, size_t n, size_t epp) {
  ChunkSpan s;
  s.p0 = static_cast<size_t>(c) * chunk_packs;
  s.packs = npacks - s.p0 < chunk_packs ? npacks - s.p0 : chunk_packs;
  s.n = (s.p0 + s.packs) * epp <= n ? s.packs * epp : n - s.p0 * epp;
  s.n_valid = n - s.p0 * 4 < s.packs * 4 ? n - s.p0 * 4 : s.packs * 4;
  return s;
}

// The segment table of a reduce bucket (b2d_owner.cuh) in the order the owner kernels walk it.
struct OwnerTable {
  std::vector<long long> flat_off;         // flat offset of each merged segment
  std::vector<unsigned> start;             // its first staging pack; one entry more, the bucket's total
  unsigned owner_pack[B2D_MAX_WORLD + 1];  // staging packs [owner_pack[r], owner_pack[r+1]) belong to owner r
};

// Sorts the segments by (owner, offset) and merges runs that touch.  Returns an empty string, or why the segments
// do not form a valid bucket.
inline std::string build_owner_table(const b2d_seg* segs, int nseg, int world, int wire, OwnerTable* t) {
  const long long epp = wire == B2D_WIRE_BF16 ? 8 : 4;
  std::vector<b2d_seg> v(segs, segs + nseg);
  for (const b2d_seg& sgm : v) {
    if (sgm.owner < 0 || sgm.owner >= world) return "segment owner " + std::to_string(sgm.owner) + " out of range";
    if (sgm.flat_off < 0 || sgm.len <= 0 || sgm.flat_off % 8 != 0 || sgm.len % 8 != 0)
      return "segments must be non-empty, 8-element aligned runs (got " + std::to_string(sgm.flat_off) + " + " +
             std::to_string(sgm.len) + ")";
  }
  std::stable_sort(v.begin(), v.end(), [](const b2d_seg& a, const b2d_seg& b) { return a.owner != b.owner ? a.owner < b.owner : a.flat_off < b.flat_off; });
  std::vector<b2d_seg> m;
  for (const b2d_seg& sgm : v) {
    if (!m.empty() && m.back().owner == sgm.owner && m.back().flat_off + m.back().len == sgm.flat_off) m.back().len += sgm.len;
    else m.push_back(sgm);
  }
  t->flat_off.assign(m.size(), 0);
  t->start.assign(m.size() + 1, 0);
  unsigned long long cum = 0;
  int next_owner = 0;
  for (size_t i = 0; i < m.size(); ++i) {
    while (next_owner <= m[i].owner) t->owner_pack[next_owner++] = static_cast<unsigned>(cum);
    t->flat_off[i] = m[i].flat_off;
    t->start[i] = static_cast<unsigned>(cum);
    cum += static_cast<unsigned long long>(m[i].len / epp);
    if (cum > 0xffffffffull) return "reduce bucket too large";
  }
  t->start[m.size()] = static_cast<unsigned>(cum);
  while (next_owner <= B2D_MAX_WORLD) t->owner_pack[next_owner++] = static_cast<unsigned>(cum);
  return "";
}

}  // namespace b2d
