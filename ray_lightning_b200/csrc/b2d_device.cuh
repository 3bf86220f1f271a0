// b2d_device.cuh — device-side building blocks of libb2d (sm_90a only).
//
//   * 16-byte vector loads/stores with explicit PTX cache/coherence qualifiers
//   * fp32 <-> bf16 pack conversion with the reference's rounding points
//     (torch bf16_compress_hook, default_hooks.py:57-93,116-134)
//   * the inter-GPU block barrier over system-scope flags in the peers' signal pads
//   * NVLS multimem.ld_reduce / multimem.st wrappers
//
// Nothing here is ML specific: the unit of work is a "pack" = 16 bytes of wire payload
// (8 bf16 or 4 fp32 gradient elements).
#pragma once

#ifdef B2D_EMU   // CPU emulation of the device environment: tests only (csrc/emu/cuda_emu.h)
#include "emu/cuda_emu.h"
#else
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/b2d.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libb2d is written for sm_90a (H100) only"
#endif

namespace b2d {

// ---- signal pad ------------------------------------------------------------------------
// One per rank, at the start of that rank's arena, mapped by every peer.
// flag[e&1][block][src] is written by rank `src` (system scope) when its block `block`
// reaches barrier epoch e; ctr[block] is the local epoch of that block and is touched by
// the owning rank only.  Epochs only grow (never reset), two flag sets alternate so that a
// fast peer arriving at epoch e+1 cannot overwrite a flag a slow peer still polls for e.
struct Signal {
  uint32_t flag[2][B2D_MAX_BLOCKS][B2D_MAX_WORLD];
  uint32_t ctr[B2D_MAX_BLOCKS];
  // staged exchange (b2d_staged.cuh): monotone chunk epochs, one word per source rank, written by that
  // rank's LAST block of the stage / exchange kernel; done_ctr are the local "blocks finished" tickets.
  uint32_t staged[B2D_MAX_WORLD];
  uint32_t published[B2D_MAX_WORLD];
  uint32_t done_ctr[2];
  // synchronised BatchNorm (b2d_syncbn.cuh): monotone exchange epochs, one word per source rank.  Separate from
  // `staged`: the BN exchanges run on the caller's stream, concurrently with bucket exchanges on the internal ones.
  uint32_t bn[B2D_MAX_WORLD];
  // gradient clipping (b2d_clip.cuh): monotone clip-exchange epochs, one word per source rank, with their own host
  // epoch counter; clip_ctr is K18's local "blocks finished" ticket (not done_ctr: K11 / K13 share those)
  uint32_t clip[B2D_MAX_WORLD];
  uint32_t clip_ctr;
};
static_assert(sizeof(Signal) <= 64 * 1024, "signal pad must fit its 64 KiB reservation");
constexpr size_t kSignalBytes = 64 * 1024;

// Written (host-mapped pinned memory) by a block that gives up waiting for a peer.
struct Diag {
  uint32_t code;    // 0 = nothing; 1 = peer timeout
  uint32_t rank, block, peer, expect, got;
};

struct Peers {
  unsigned char* arena[B2D_MAX_WORLD];  // every rank's arena as mapped in THIS process
  Signal* signal[B2D_MAX_WORLD];
  unsigned char* mc_arena;              // multicast alias of the arenas (NVLS) or nullptr
};

// ---- memory ops ------------------------------------------------------------------------
#ifdef B2D_EMU
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) { return emu_ld128(p); }
__device__ __forceinline__ uint4 ld_peer_v4(const void* p) { return emu_ld128(p); }
__device__ __forceinline__ void st_v4(void* p, const uint4& v) { emu_st128(p, v); }
__device__ __forceinline__ void st_stream_v4(void* p, const uint4& v) { emu_st128(p, v); }
__device__ __forceinline__ uint32_t ld_flag(const uint32_t* p) { return emu_ld32(p); }
__device__ __forceinline__ void st_flag(uint32_t* p, uint32_t v) { emu_st32(p, v); }
__device__ __forceinline__ unsigned long long global_timer_ns() { return emu_timer_ns(); }
// NVLS: the "switch" adds the 8 bf16 lanes (or 4 fp32) of every bound arena in fp32, in rank order
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc_ptr) {
  const emu::Multicast& m = emu::multicast();
  const size_t off = static_cast<const unsigned char*>(mc_ptr) - m.fake_base;
  float acc[8];
  for (int r = 0; r < m.world; ++r) {
    const uint4 v = emu_ld128(m.arena[r] + off);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    for (int k = 0; k < 4; ++k) {
      const float lo = emu_bf16_to_f32(static_cast<uint16_t>(w[k] & 0xffffu)), hi = emu_bf16_to_f32(static_cast<uint16_t>(w[k] >> 16));
      acc[2 * k] = r == 0 ? lo : __fadd_rn(acc[2 * k], lo);
      acc[2 * k + 1] = r == 0 ? hi : __fadd_rn(acc[2 * k + 1], hi);
    }
  }
  uint32_t o[4];
  for (int k = 0; k < 4; ++k) o[k] = static_cast<uint32_t>(emu_f32_to_bf16(acc[2 * k])) | (static_cast<uint32_t>(emu_f32_to_bf16(acc[2 * k + 1])) << 16);
  return make_uint4(o[0], o[1], o[2], o[3]);
}
__device__ __forceinline__ uint4 multimem_ld_reduce_f32x4(const void* mc_ptr) {
  const emu::Multicast& m = emu::multicast();
  const size_t off = static_cast<const unsigned char*>(mc_ptr) - m.fake_base;
  float acc[4];
  for (int r = 0; r < m.world; ++r) {
    const uint4 v = emu_ld128(m.arena[r] + off);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    for (int k = 0; k < 4; ++k) acc[k] = r == 0 ? __uint_as_float(w[k]) : __fadd_rn(acc[k], __uint_as_float(w[k]));
  }
  return make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]), __float_as_uint(acc[3]));
}
__device__ __forceinline__ void multimem_st_v4(void* mc_ptr, const uint4& v) {
  const emu::Multicast& m = emu::multicast();
  const size_t off = static_cast<unsigned char*>(mc_ptr) - m.fake_base;
  for (int r = 0; r < m.world; ++r) emu_st128(m.arena[r] + off, v);
}
__device__ __forceinline__ float multimem_ld_reduce_f32(const void* mc_ptr) {
  const emu::Multicast& m = emu::multicast();
  const size_t off = static_cast<const unsigned char*>(mc_ptr) - m.fake_base;
  float acc = 0.f;
  for (int r = 0; r < m.world; ++r) {
    const float v = __uint_as_float(emu_ld32(m.arena[r] + off));
    acc = r == 0 ? v : __fadd_rn(acc, v);
  }
  return acc;
}
__device__ __forceinline__ void multimem_st_f32(void* mc_ptr, float v) {
  const emu::Multicast& m = emu::multicast();
  const size_t off = static_cast<unsigned char*>(mc_ptr) - m.fake_base;
  for (int r = 0; r < m.world; ++r) emu_st32(m.arena[r] + off, __float_as_uint(v));
}
#else
// Own fp32 gradients: streamed once, keep them out of L1.
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
// Peer (or own) staged payload that another GPU wrote before the last barrier: a strong
// system-scope load, so it can never be served from a stale L1 line (peer addresses may be
// cached in L1 and bypass the local L2).
__device__ __forceinline__ uint4 ld_peer_v4(const void* p) {
  uint4 r;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void st_v4(void* p, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
// Final fp32 results: written once, not re-read by this kernel.
__device__ __forceinline__ void st_stream_v4(void* p, const uint4& v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint32_t ld_flag(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_flag(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
  return t;
}

// NVLS: one instruction makes the switch fetch the 16 bytes at this offset from every
// bound GPU, add them as 8 bf16 lanes with fp32 accumulation and return the bf16 result.
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc_ptr) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(mc_ptr)
               : "memory");
  return r;
}
__device__ __forceinline__ uint4 multimem_ld_reduce_f32x4(const void* mc_ptr) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(mc_ptr)
               : "memory");
  return r;
}
// NVLS broadcast store: the switch replicates the 16 bytes into every bound GPU.
__device__ __forceinline__ void multimem_st_v4(void* mc_ptr, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
// scalar forms, for the ragged tail of an in-place fp32 bucket
__device__ __forceinline__ float multimem_ld_reduce_f32(const void* mc_ptr) {
  float r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f32 %0, [%1];" : "=f"(r) : "l"(mc_ptr) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_f32(void* mc_ptr, float v) {
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc_ptr), "f"(v) : "memory");
}

#endif  // B2D_EMU

// ---- number formats --------------------------------------------------------------------
#ifdef B2D_EMU
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  return static_cast<uint32_t>(emu_f32_to_bf16(lo)) | (static_cast<uint32_t>(emu_f32_to_bf16(hi)) << 16);
}
#else
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);  // cvt.rn.bf16x2.f32: RNE, NaN kept
  return *reinterpret_cast<uint32_t*>(&b);
}
#endif
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
// fp32 -> bf16 -> fp32 (what `t.to(torch.bfloat16)` keeps of a value)
__device__ __forceinline__ float round_bf16(float x) {
#ifdef B2D_EMU
  return emu_bf16_to_f32(emu_f32_to_bf16(x));
#else
  return __bfloat162float(__float2bfloat16_rn(x));
#endif
}
// bf16_compress_hook prologue for one element: `buffer.to(bf16).div_(world)`.  torch's CUDA
// div-by-scalar multiplies by the fp32 reciprocal and rounds once more to bf16, so the value
// put on the wire is bf16(fp32(bf16(g)) * scale) with scale = 1.0f / world.
__device__ __forceinline__ float wire_bf16_value(float g, float scale) {
  return round_bf16(round_bf16(g) * scale);
}

// ---- system-scope fence ------------------------------------------------------------------
// Release / acquire around the flag exchange need fence.acq_rel, not the sequentially consistent fence that
// __threadfence_system() emits (SASS MEMBAR.SC.SYS + ERRBAR + CCTL.IVALL): every payload access that follows an
// acquire is itself a system-scope load (ld.relaxed.sys) or runs in a later kernel.
__device__ __forceinline__ void fence_sys() {
#ifdef B2D_EMU
  __threadfence_system();
#else
  asm volatile("fence.acq_rel.sys;" ::: "memory");
#endif
}

// ---- inter-GPU block barrier ------------------------------------------------------------
// Block `b` of this rank meets block `b` of every peer.  Everything the block's threads
// wrote before the call (own arena, peers' arenas) is visible to the peer blocks after
// their call returns (release/acquire at system scope around the flag exchange).
// A peer that does not arrive within `timeout_ns` traps the kernel (sticky CUDA error
// instead of a silent hang); details land in `diag`.
__device__ __forceinline__ void block_barrier(const Peers& peers, int rank, int world,
                                              unsigned long long timeout_ns, Diag* diag) {
  __syncthreads();
  Signal* self = peers.signal[rank];
  const int b = blockIdx.x;
  uint32_t val = 0;
  if (threadIdx.x < world) {
    val = self->ctr[b] + 1u;
    fence_sys();  // release: the block's earlier writes, cumulative over bar.sync
    st_flag(&peers.signal[threadIdx.x]->flag[val & 1u][b][rank], val);
    const uint32_t* mine = &self->flag[val & 1u][b][threadIdx.x];
    uint32_t got = ld_flag(mine);
    if (static_cast<int32_t>(got - val) < 0) {
      const unsigned long long t0 = global_timer_ns();
      unsigned spins = 0;
      while (static_cast<int32_t>((got = ld_flag(mine)) - val) < 0) {
        if ((++spins & 0xffu) == 0 && timeout_ns != 0 && global_timer_ns() - t0 > timeout_ns) {
          if (diag != nullptr) {
            diag->rank = rank;
            diag->block = b;
            diag->peer = threadIdx.x;
            diag->expect = val;
            diag->got = got;
            diag->code = 1;
            fence_sys();
          }
          __trap();
        }
      }
    }
    fence_sys();  // acquire
  }
  __syncthreads();
  if (threadIdx.x == 0) self->ctr[b] = val;
}

// ---- split barrier: arrive now, consume the peers' arrivals one by one -------------------------
// barrier_arrive() publishes this block's epoch to every peer (after making the block's writes
// visible); poll_arrived() — called by ONE thread — returns the set of not-yet-consumed peers whose
// same-index block has arrived, spinning until there is at least one.  Lets the all-gather start
// with whoever is ready instead of waiting for the slowest rank.
__device__ __forceinline__ uint32_t barrier_arrive(const Peers& peers, int rank, int world) {
  __syncthreads();
  const int b = blockIdx.x;
  const uint32_t val = peers.signal[rank]->ctr[b] + 1u;
  if (threadIdx.x < world) {
    fence_sys();
    st_flag(&peers.signal[threadIdx.x]->flag[val & 1u][b][rank], val);
  }
  return val;
}

__device__ __forceinline__ uint32_t poll_arrived(const Peers& peers, int rank, int world, uint32_t val,
                                                 uint32_t done_mask, unsigned long long timeout_ns, Diag* diag) {
  const int b = blockIdx.x;
  const uint32_t* mine = &peers.signal[rank]->flag[val & 1u][b][0];
  uint32_t mask = 0;
  const unsigned long long t0 = global_timer_ns();
  unsigned spins = 0;
  for (;;) {
    for (int s = 0; s < world; ++s)
      if (!((done_mask >> s) & 1u) && (s == rank || static_cast<int32_t>(ld_flag(mine + s) - val) >= 0)) mask |= 1u << s;
    if (mask != 0) break;
    if ((++spins & 0xffu) == 0 && timeout_ns != 0 && global_timer_ns() - t0 > timeout_ns) {
      if (diag != nullptr) {
        int first = 0;
        while (first < world && ((done_mask >> first) & 1u)) ++first;
        diag->rank = rank; diag->block = b; diag->peer = first; diag->expect = val; diag->got = ld_flag(mine + first);
        diag->code = 1;
        fence_sys();
      }
      __trap();
    }
  }
  fence_sys();  // acquire
  return mask;
}

}  // namespace b2d
