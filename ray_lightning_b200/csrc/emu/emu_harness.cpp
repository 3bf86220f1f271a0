// emu_harness.cpp — runs the libb2d kernels (the very sources nvcc compiles) on CPU threads, chosen by the same
// selectors (b2d_launch.cuh) the library launches through.
// TEST INFRASTRUCTURE ONLY: built by tests/test_kernel_emulation.py with g++ -std=c++20 -DB2D_EMU -pthread.
// See emu/cuda_emu.h for what is and is not modelled.
#ifndef B2D_EMU
#define B2D_EMU 1
#endif
#include <pthread.h>

#include <cmath>
#include <functional>
#include <vector>

#include <thread>

#include "../b2d_kernels.cuh"
#include "../b2d_staged.cuh"
#include "../b2d_owner.cuh"
#include "../b2d_syncbn.cuh"
#include "../b2d_clip.cuh"
#include "../b2d_launch.cuh"

thread_local EmuDim3 threadIdx, blockIdx, blockDim, gridDim;
thread_local emu::Block* emu_block = nullptr;

using namespace b2d;

namespace {

struct Group {
  int world = 0;
  size_t arena_bytes = 0;
  std::vector<unsigned char*> arena;
  unsigned char* fake_mc = nullptr;
};

struct ThreadArg {
  std::function<void()>* body;
  emu::Block* block;
  unsigned tid, bid, nthreads, nblocks;
};

void* thread_main(void* p) {
  ThreadArg* a = static_cast<ThreadArg*>(p);
  threadIdx.x = a->tid; blockIdx.x = a->bid; blockDim.x = a->nthreads; gridDim.x = a->nblocks;
  emu_block = a->block;
  (*a->body)();
  return nullptr;
}

// launch `bodies[r]` as a grid x block kernel for every rank r, all ranks concurrently; join
int launch_all(int world, int grid, int block, std::vector<std::function<void()>>& bodies) {
  std::vector<std::unique_ptr<emu::Block>> blocks;
  std::vector<ThreadArg> args(static_cast<size_t>(world) * grid * block);
  std::vector<pthread_t> tids(args.size());
  pthread_attr_t attr;
  pthread_attr_init(&attr);
  pthread_attr_setstacksize(&attr, 512 * 1024);
  size_t k = 0;
  for (int r = 0; r < world; ++r)
    for (int b = 0; b < grid; ++b) {
      blocks.emplace_back(new emu::Block(block));
      for (int t = 0; t < block; ++t, ++k) {
        args[k] = ThreadArg{&bodies[r], blocks.back().get(), static_cast<unsigned>(t), static_cast<unsigned>(b),
                            static_cast<unsigned>(block), static_cast<unsigned>(grid)};
        if (pthread_create(&tids[k], &attr, thread_main, &args[k]) != 0) return -1;
      }
    }
  for (size_t i = 0; i < k; ++i) pthread_join(tids[i], nullptr);
  pthread_attr_destroy(&attr);
  return 0;
}

Peers make_peers(const Group& g) {
  Peers p{};
  for (int r = 0; r < g.world; ++r) {
    p.arena[r] = g.arena[r];
    p.signal[r] = reinterpret_cast<Signal*>(g.arena[r]);
  }
  p.mc_arena = g.fake_mc;
  return p;
}

// one kernel of one rank: grid x block threads running kernel(args...), joined before returning (a stream runs these
// one after another)
template <typename Kernel, typename... Args>
int launch_one(Kernel kernel, int grid, int block, const Args&... args) {
  std::vector<std::function<void()>> bodies(1, [=] { kernel(args...); });
  return launch_all(1, grid, block, bodies);
}

// The peer-wait fields of rank r's parameters, as b2d.cu fills them from its context (no diagnostics record here).
template <typename Params>
void set_peer_wait(Params* P, int r, const Group& g, unsigned long long timeout_s) {
  set_peer_wait(P, r, g.world, make_peers(g), timeout_s * 1000000000ull, nullptr);
}

// Points the emulated multicast alias (NVLS) at the group's arenas.
void bind_multicast(const Group& g) {
  emu::Multicast& mc = emu::multicast();
  mc.fake_base = g.fake_mc; mc.world = g.world;
  for (int r = 0; r < g.world; ++r) mc.arena[r] = g.arena[r];
}

// Runs the phases of one operation, f(rank, chunk) for every rank and chunk of each phase.  `order`:
//   0  every rank is one in-order stream (every phase of chunk 0, then of chunk 1, ...); the ranks run concurrently
//   1  fully serialised, phase-major (the first phase of every chunk and rank, then the second, ...): what a
//      serialising profiler makes of the single-GPU loopback ranks
//   2  one concurrent stream per phase and rank, coupled ONLY by the kernels' flags — more freedom than the
//      event-ordered streams of b2d.cu allow
using Phase = std::function<int(int rank, int chunk)>;
int run_phases(int world, int nchunks, int order, const std::vector<Phase>& phases) {
  if (order == 1) {
    for (const Phase& f : phases)
      for (int c = 0; c < nchunks; ++c)
        for (int r = 0; r < world; ++r)
          if (f(r, c) != 0) return -1;
    return 0;
  }
  std::atomic<int> bad{0};
  std::vector<std::thread> streams;
  for (int r = 0; r < world; ++r) {
    if (order == 0) {
      streams.emplace_back([&, r] {
        for (int c = 0; c < nchunks; ++c)
          for (const Phase& f : phases)
            if (f(r, c) != 0) { bad = 1; break; }
      });
    } else {
      for (const Phase& f : phases)
        streams.emplace_back([&, r, fp = &f] { for (int c = 0; c < nchunks; ++c) if ((*fp)(r, c) != 0) bad = 1; });
    }
  }
  for (auto& t : streams) t.join();
  return bad.load() ? -1 : 0;
}

}  // namespace

extern "C" {

void* emu_group_create(int world, size_t arena_bytes) {
  Group* g = new Group();
  g->world = world;
  g->arena_bytes = arena_bytes;
  for (int r = 0; r < world; ++r) {
    void* p = nullptr;
    if (posix_memalign(&p, 4096, arena_bytes) != 0) return nullptr;
    std::memset(p, 0, arena_bytes);
    g->arena.push_back(static_cast<unsigned char*>(p));
  }
  g->fake_mc = reinterpret_cast<unsigned char*>(static_cast<uintptr_t>(1) << 44);   // never dereferenced directly
  return g;
}

void emu_group_destroy(void* h) {
  Group* g = static_cast<Group*>(h);
  for (auto p : g->arena) free(p);
  delete g;
}

size_t emu_signal_bytes(void) { return kSignalBytes; }

// The staged exchange (b2d_staged.cuh) of one bucket, cut into chunks of `chunk_packs`, epochs epoch0.. (monotone
// over calls, like ctx->epoch in b2d.cu).  wire_off: byte offset of the staging region in every arena; with
// `inplace` the fp32 buckets themselves live there (bufs is ignored).  `order` as in run_phases, over the phases S,
// X and W+U: 0 is b2d.cu's stream order, 1 and 2 are the serialised and the freest schedules.
int emu_staged_allreduce(void* h, int nvls, int bf16, int inplace, float** bufs, size_t n, float scale, size_t wire_off,
                         size_t chunk_packs, int st_grid, int ex_grid, unsigned epoch0, int order, int use_generic_w) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const size_t epp = bf16 ? 8 : 4;
  const size_t npacks = (n + epp - 1) / epp;
  if (wire_off + npacks * 16 > g->arena_bytes) return -4;
  const int nchunks = static_cast<int>((npacks + chunk_packs - 1) / chunk_packs);
  bind_multicast(*g);
  auto stage_params = [&](int r, int c) {   // S and U of chunk c
    StParams P{};
    P.scale = scale; P.rank = r; P.world = world; P.peers = make_peers(*g);
    const ChunkSpan cs = chunk_span(c, npacks, chunk_packs, n, epp);
    P.grad = bufs[r] + cs.p0 * epp;
    P.n = cs.n;
    P.wire = reinterpret_cast<uint4*>(g->arena[r] + wire_off) + cs.p0;
    P.epoch = epoch0 + c;
    return P;
  };
  auto S = [&](int r, int c) {
    if (!inplace) return launch_one(select_stage(bf16), st_grid, kStThreads, stage_params(r, c));
    if (c != 0) return 0;
    StParams P{};
    P.rank = r; P.world = world; P.peers = make_peers(*g);
    P.epoch = epoch0 + nchunks - 1;
    return launch_one(arrive_kernel, 1, 32, P);
  };
  auto X = [&](int r, int c) {
    ExParams P{};
    set_peer_wait(&P, r, *g, 120);
    P.scale = scale;
    const ChunkSpan cs = chunk_span(c, npacks, chunk_packs, n, epp);
    P.wire_off = wire_off + cs.p0 * 16; P.npacks = cs.packs; P.epoch = epoch0 + c;
    P.n_valid = inplace ? cs.n_valid : 0;
    return launch_one(select_exch(use_generic_w ? 0 : world, bf16, nvls, inplace), ex_grid, kExThreads, P);
  };
  auto WU = [&](int r, int c) {
    ExParams P{};
    set_peer_wait(&P, r, *g, 120);
    P.epoch = epoch0 + c;
    const int rc = launch_one(wait_published_kernel, 1, 32, P);
    if (rc != 0 || inplace) return rc;
    return launch_one(select_unstage(bf16), st_grid, kStThreads, stage_params(r, c));
  };
  return run_phases(world, nchunks, order, {S, X, WU});
}

// K11 + K12 (b2d_owner.cuh): one reduce bucket given as an owner-sorted segment table (seg_start in packs of the wire
// format, cumulative, nseg + 1 entries; owner_pack[world + 1]).  order as in run_phases (0 / 1).
int emu_reduce_to_owner(void* h, int bf16, int nvls, float** grads, float** reduced, const long long* shard_off,
                        const long long* seg_flat_off, const unsigned* seg_start, int nseg, const unsigned* owner_pack,
                        size_t wire_off, float scale, int zero_grads, int accumulate, unsigned epoch, int order, int use_generic_w) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  if (wire_off + static_cast<size_t>(seg_start[nseg]) * 16 > g->arena_bytes) return -4;
  bind_multicast(*g);
  auto mk = [&](int r) {
    SegParams P{};
    P.seg_flat_off = seg_flat_off; P.seg_start = seg_start; P.nseg = nseg;
    for (int i = 0; i <= B2D_MAX_WORLD; ++i) P.owner_pack[i] = owner_pack[i <= world ? i : world];
    P.grads = grads[r]; P.reduced = reduced[r]; P.shard_lo = shard_off[r]; P.wire_off = wire_off; P.scale = scale;
    P.zero_grads = zero_grads; P.accumulate = accumulate; P.epoch = epoch;
    set_peer_wait(&P, r, *g, 120);
    return P;
  };
  auto S = [&](int r, int) { return launch_one(select_seg_stage(bf16), 2, kStThreads, mk(r)); };
  auto X = [&](int r, int) { return launch_one(select_seg_reduce(use_generic_w ? 0 : world, bf16, nvls), 2, kExThreads, mk(r)); };
  return run_phases(world, 1, order, {S, X});
}

// K13: params live in every arena at param_off; m, v, reduced are the ranks' own-shard buffers.  One Adam group per
// rank covering [glo[r], ghi[r]) of its shard (ngroups = 0: push only).
static int adam_push_impl(void* h, int nvls, size_t param_off, float** m, float** v, float** reduced, size_t n,
                          const long long* shard_off, int ngroups, const long long* glo, const long long* ghi, double lr, double beta1,
                          double beta2, double eps, double wd, int step, int adamw, unsigned epoch, int order, int use_generic_w,
                          float** grad_scale) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  if (param_off + n * 4 > g->arena_bytes) return -4;
  bind_multicast(*g);
  auto X = [&](int r, int) {
    PushParams P{};
    P.params = reinterpret_cast<float*>(g->arena[r] + param_off); P.param_off = param_off;
    P.exp_avg = m ? m[r] : nullptr; P.exp_avg_sq = v ? v[r] : nullptr; P.reduced = reduced ? reduced[r] : nullptr;
    P.lo = shard_off[r]; P.hi = shard_off[r + 1]; P.ngroups = ngroups;
    if (ngroups > 0) {
      P.group_lo[0] = glo[r]; P.group_hi[0] = ghi[r];
      P.group[0] = adam_consts(b2d_adam64{lr, beta1, beta2, eps, wd, step, adamw, 0, 0});
    }
    P.rank = r; P.world = world; P.epoch = epoch; P.peers = make_peers(*g);
    P.grad_scale = grad_scale ? grad_scale[r] : nullptr;
    return launch_one(select_adam_push(use_generic_w ? 0 : world, nvls, grad_scale != nullptr), 2, kExThreads, P);
  };
  auto Wt = [&](int r, int) {
    ExParams P{};
    set_peer_wait(&P, r, *g, 120);
    P.epoch = epoch;
    return launch_one(wait_published_kernel, 1, 32, P);
  };
  return run_phases(world, 1, order, {X, Wt});
}

// The *64 entry points take the hyper-parameters as doubles (b2d_adam64); the others as fp32 (b2d_adam), widened.
int emu_adam_push64(void* h, int nvls, size_t param_off, float** m, float** v, float** reduced, size_t n, const long long* shard_off,
                    int ngroups, const long long* glo, const long long* ghi, double lr, double beta1, double beta2, double eps,
                    double wd, int step, int adamw, unsigned epoch, int order, int use_generic_w) {
  return adam_push_impl(h, nvls, param_off, m, v, reduced, n, shard_off, ngroups, glo, ghi, lr, beta1, beta2, eps, wd, step, adamw,
                        epoch, order, use_generic_w, nullptr);
}

int emu_adam_push(void* h, int nvls, size_t param_off, float** m, float** v, float** reduced, size_t n, const long long* shard_off,
                  int ngroups, const long long* glo, const long long* ghi, float lr, float beta1, float beta2, float eps, float wd,
                  int step, int adamw, unsigned epoch, int order, int use_generic_w) {
  return adam_push_impl(h, nvls, param_off, m, v, reduced, n, shard_off, ngroups, glo, ghi, lr, beta1, beta2, eps, wd, step, adamw,
                        epoch, order, use_generic_w, nullptr);
}

// K13 with the gradients multiplied by *grad_scale[r] (adam_push_scaled_kernel)
int emu_adam_push_scaled64(void* h, int nvls, size_t param_off, float** m, float** v, float** reduced, size_t n,
                           const long long* shard_off, int ngroups, const long long* glo, const long long* ghi, double lr,
                           double beta1, double beta2, double eps, double wd, int step, int adamw, unsigned epoch, int order,
                           int use_generic_w, float** grad_scale) {
  if (grad_scale == nullptr) return -1;
  return adam_push_impl(h, nvls, param_off, m, v, reduced, n, shard_off, ngroups, glo, ghi, lr, beta1, beta2, eps, wd, step, adamw,
                        epoch, order, use_generic_w, grad_scale);
}

int emu_adam_push_scaled(void* h, int nvls, size_t param_off, float** m, float** v, float** reduced, size_t n,
                         const long long* shard_off, int ngroups, const long long* glo, const long long* ghi, float lr, float beta1,
                         float beta2, float eps, float wd, int step, int adamw, unsigned epoch, int order, int use_generic_w,
                         float** grad_scale) {
  return emu_adam_push_scaled64(h, nvls, param_off, m, v, reduced, n, shard_off, ngroups, glo, ghi, lr, beta1, beta2, eps, wd, step,
                                adamw, epoch, order, use_generic_w, grad_scale);
}

// K14: one optimizer step of a bucket whose parameters (and their state tensors) are separate allocations.
int emu_bucket_optim64(float** params, float** state1, float** state2, const unsigned* seg_start, int nseg, const float* grads,
                       size_t n, int kind, double lr, float momentum, double wd, double beta1, double beta2, double eps, int step,
                       int adamw) {
  OptimParams P{};
  P.param_ptr = params; P.state1_ptr = state1; P.state2_ptr = state2; P.seg_start = seg_start; P.nseg = nseg;
  P.grads = grads; P.n = n; P.kind = kind; P.lr = static_cast<float>(lr); P.momentum = momentum;
  P.weight_decay = static_cast<float>(wd); P.first_step = step <= 1;
  if (kind == 1) P.adam = adam_consts(b2d_adam64{lr, beta1, beta2, eps, wd, step, adamw, 0, 0});
  return launch_one(bucket_optim_kernel, 2, kStThreads, P);
}

int emu_bucket_optim(float** params, float** state1, float** state2, const unsigned* seg_start, int nseg, const float* grads,
                     size_t n, int kind, float lr, float momentum, float wd, float beta1, float beta2, float eps, int step, int adamw) {
  return emu_bucket_optim64(params, state1, state2, seg_start, nseg, grads, n, kind, lr, momentum, wd, beta1, beta2, eps, step, adamw);
}

// bufs[r]: rank r's fp32 bucket, reduced in place.  algo: 1 one-shot, 2 two-shot, 3 two-shot NVLS (fused).
// parity selects the half of the (single) double-buffered slot, exactly like get_slot() in b2d.cu.
int emu_allreduce(void* h, int algo, int bf16, float** bufs, size_t n, float scale, int grid, int parity, int use_generic_w,
                  int pipe_k) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const size_t epp = bf16 ? 8 : 4;
  const size_t npacks = (n + epp - 1) / epp, slice = (npacks + world - 1) / world;
  const size_t half = (slice * world * 16 + 255) / 256 * 256;
  if (kSignalBytes + 2 * half > g->arena_bytes) return -4;
  if (algo < 1 || algo > 3) return -2;
  (void)pipe_k;
  bind_multicast(*g);
  const int w = use_generic_w ? 0 : world;
  const auto kernel = algo == 1 ? select_k1(w, bf16) : select_k2(w, bf16, algo == 3);
  std::vector<std::function<void()>> bodies(world);
  for (int r = 0; r < world; ++r) {
    ArParams P{};
    P.trace = nullptr; P.grad = bufs[r]; P.n = n; P.stage_off = kSignalBytes + (parity & 1) * half; P.scale = scale;
    set_peer_wait(&P, r, *g, 60);
    bodies[r] = [=] { kernel(P); };
  }
  return launch_all(world, grid, kThreads, bodies);
}

// K0: world 1, no peers
int emu_k0(float* buf, size_t n, float scale, int bf16, int grid) {
  return launch_one(select_k0(bf16), grid, kThreads, buf, n, scale);
}

// Fused sharded step.  params live in every arena at `param_off`; grads[r], m[r], v[r] are plain buffers.
int emu_sharded_step64(void* h, int bf16, float** grads, size_t param_off, float** m, float** v, size_t n,
                       const long long* shard_off, float scale, double lr, double beta1, double beta2, double eps, double wd,
                       int step, int adamw, int zero_grads, int grid, int parity, int use_generic_w) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const size_t half = (n * (bf16 ? 2 : 4) + 255) / 256 * 256;
  const size_t stage_base = param_off + ((n * 4 + 255) / 256 * 256);
  if (stage_base + 2 * half > g->arena_bytes) return -4;
  const auto kernel = select_k456(use_generic_w ? 0 : world, bf16);
  std::vector<std::function<void()>> bodies(world);
  for (int r = 0; r < world; ++r) {
    ShParams P{};
    P.grads = grads[r]; P.grads_rw = zero_grads ? grads[r] : nullptr;
    P.params = reinterpret_cast<float*>(g->arena[r] + param_off); P.param_off = param_off;
    P.exp_avg = m[r]; P.exp_avg_sq = v[r]; P.rs_out = nullptr; P.n = n;
    for (int i = 0; i <= world; ++i) P.off[i] = shard_off[i];
    for (int i = world + 1; i <= B2D_MAX_WORLD; ++i) P.off[i] = shard_off[world];
    P.stage_off = stage_base + (parity & 1) * half; P.scale = scale;
    P.do_stage_reduce = 1; P.do_adam = 1; P.do_gather = 1; P.end_barrier = 0;
    P.adam = adam_consts(b2d_adam64{lr, beta1, beta2, eps, wd, step, adamw, 0, 0});
    set_peer_wait(&P, r, *g, 60);
    bodies[r] = [=] { kernel(P); };
  }
  return launch_all(world, grid, kThreads, bodies);
}

int emu_sharded_step(void* h, int bf16, float** grads, size_t param_off, float** m, float** v, size_t n,
                     const long long* shard_off, float scale, float lr, float beta1, float beta2, float eps, float wd,
                     int step, int adamw, int zero_grads, int grid, int parity, int use_generic_w) {
  return emu_sharded_step64(h, bf16, grads, param_off, m, v, n, shard_off, scale, lr, beta1, beta2, eps, wd, step, adamw, zero_grads,
                            grid, parity, use_generic_w);
}

// K4 alone (reduce-scatter to owner, fp32 out) and K6 alone (all-gather of a flat arena buffer, with its end barrier)
int emu_reduce_scatter(void* h, int bf16, float** grads, float** outs, size_t n, const long long* shard_off, float scale,
                       size_t stage_base, int grid, int parity) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const size_t half = (n * (bf16 ? 2 : 4) + 255) / 256 * 256;
  if (stage_base + 2 * half > g->arena_bytes) return -4;
  const auto kernel = select_k456(0, bf16);
  std::vector<std::function<void()>> bodies(world);
  for (int r = 0; r < world; ++r) {
    ShParams P{};
    P.grads = grads[r]; P.rs_out = outs[r]; P.n = n;
    for (int i = 0; i <= world; ++i) P.off[i] = shard_off[i];
    for (int i = world + 1; i <= B2D_MAX_WORLD; ++i) P.off[i] = shard_off[world];
    P.stage_off = stage_base + (parity & 1) * half; P.scale = scale;
    P.do_stage_reduce = 1; P.do_adam = 0; P.do_gather = 0;
    set_peer_wait(&P, r, *g, 60);
    bodies[r] = [=] { kernel(P); };
  }
  return launch_all(world, grid, kThreads, bodies);
}

int emu_allgather(void* h, size_t buf_off, size_t n, const long long* shard_off, int grid) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const auto kernel = select_k456(0, false);
  std::vector<std::function<void()>> bodies(world);
  for (int r = 0; r < world; ++r) {
    ShParams P{};
    P.params = reinterpret_cast<float*>(g->arena[r] + buf_off); P.param_off = buf_off; P.n = n;
    for (int i = 0; i <= world; ++i) P.off[i] = shard_off[i];
    for (int i = world + 1; i <= B2D_MAX_WORLD; ++i) P.off[i] = shard_off[world];
    P.do_gather = 1; P.end_barrier = 1;
    set_peer_wait(&P, r, *g, 60);
    bodies[r] = [=] { kernel(P); };
  }
  return launch_all(world, grid, kThreads, bodies);
}

// b2d_bucket_register's table for segments given as (flat_off, len, owner) triples: fills flat_off[nseg], start[nseg + 1]
// and owner_pack[world + 1].  Returns the number of merged segments, or -1 if the segments are rejected.
int emu_owner_table(const long long* segs, int nseg, int world, int bf16, long long* flat_off, unsigned* start, unsigned* owner_pack) {
  std::vector<b2d_seg> v(nseg);
  for (int i = 0; i < nseg; ++i) v[i] = b2d_seg{segs[3 * i], segs[3 * i + 1], static_cast<int32_t>(segs[3 * i + 2]), 0};
  OwnerTable t;
  if (!build_owner_table(v.data(), nseg, world, bf16 ? B2D_WIRE_BF16 : B2D_WIRE_FP32, &t).empty()) return -1;
  std::copy(t.flat_off.begin(), t.flat_off.end(), flat_off);
  std::copy(t.start.begin(), t.start.end(), start);
  std::copy(t.owner_pack, t.owner_pack + world + 1, owner_pack);
  return static_cast<int>(t.flat_off.size());
}

// K15 + K16 (fwd = 1) or K15 + K17 (fwd = 0) of one BN exchange: rank r pushes (a[r], b[r], counts[r]) into the
// region at region_off of every arena (a[r] / b[r] may be NULL: a zero row), then combines into out_a[r], out_b[r],
// counts_out[r] and, when rm / rv are given, rank r's running statistics.  order as in run_phases (0 / 1).
int emu_bn_exchange(void* h, int fwd, int channels, const float** a, const float** b, const float* counts, float eps, float momentum,
                    float** out_a, float** out_b, int32_t** counts_out, float** rm, float** rv, size_t region_off, unsigned epoch,
                    int grid, int order) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const size_t row = fwd ? bn_fwd_row(channels) : bn_bwd_row(channels);
  if (region_off + static_cast<size_t>(world) * row * 4 > g->arena_bytes) return -4;
  auto push = [&](int r, int) {
    BnPushParams P{};
    P.a = a[r]; P.b = b[r]; P.count = fwd ? counts[r] : 0.f; P.channels = channels; P.fwd = fwd;
    P.region_off = region_off; P.rank = r; P.world = world; P.epoch = epoch; P.peers = make_peers(*g);
    return launch_one(bn_push_kernel, 1, kBnThreads, P);
  };
  auto combine = [&](int r, int) {
    BnCombineParams P{};
    P.region_off = region_off; P.channels = channels; P.eps = eps; P.momentum = momentum;
    P.out_a = out_a[r]; P.out_b = out_b[r]; P.counts = fwd ? counts_out[r] : nullptr;
    P.running_mean = rm ? rm[r] : nullptr; P.running_var = rv ? rv[r] : nullptr;
    P.epoch = epoch;
    set_peer_wait(&P, r, *g, 120);
    return launch_one(select_bn_combine(fwd), grid, kBnThreads, P);
  };
  return run_phases(world, 1, order, {push, combine});
}

// K18 + K19 of one clip call, laid out as b2d.cu lays out the clip region at clip_off: [gen 0 | gen 1 | block sums].
// x[r]: rank r's n[r] elements; norm_out[r] / coef_out[r]: one float each.  gmax: the block cap (kClipGMax in the
// library).  order as in run_phases (0 / 1).
int emu_clip_norm(void* h, const float** x, const size_t* n, float max_norm, float** norm_out, float** coef_out, size_t clip_off,
                  int gen, unsigned gmax, unsigned epoch, int order) {
  Group* g = static_cast<Group*>(h);
  const int world = g->world;
  const size_t gen_bytes = static_cast<size_t>(world) * kClipSlotBytes;
  if (gmax < 1 || gmax > static_cast<unsigned>(kClipThreads)) return -2;
  if (clip_off + 2 * gen_bytes + gmax * sizeof(double) > g->arena_bytes) return -4;
  auto partial = [&](int r, int) {
    ClipPartialParams P{};
    P.x = x[r]; P.n = n[r]; P.vec = (reinterpret_cast<uintptr_t>(x[r]) % 16) == 0;
    P.block_sums = reinterpret_cast<double*>(g->arena[r] + clip_off + 2 * gen_bytes);
    P.region_off = clip_off + (gen & 1) * gen_bytes; P.rank = r; P.world = world; P.epoch = epoch; P.peers = make_peers(*g);
    return launch_one(sqnorm_partial_kernel, static_cast<int>(clip_grid(n[r], gmax)), kClipThreads, P);
  };
  auto coef = [&](int r, int) {
    ClipCoefParams P{};
    P.region_off = clip_off + (gen & 1) * gen_bytes; P.max_norm = max_norm; P.norm_out = norm_out[r]; P.coef_out = coef_out[r];
    P.epoch = epoch;
    set_peer_wait(&P, r, *g, 120);
    return launch_one(clip_coef_kernel, 1, 32, P);
  };
  return run_phases(world, 1, order, {partial, coef});
}

unsigned emu_clip_gmax(void) { return kClipGMax; }

float* emu_arena_ptr(void* h, int rank, size_t off) {
  return reinterpret_cast<float*>(static_cast<Group*>(h)->arena[rank] + off);
}

}  // extern "C"
