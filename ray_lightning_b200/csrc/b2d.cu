// b2d.cu — host side of libb2d: context, symmetric arena, peer mapping (CUDA IPC / VMM fd /
// same-process), NVLS multicast binding, slot bookkeeping and the kernel launches.
// C ABI declared in include/b2d.h.  No torch, no pybind: plain CUDA runtime (static) plus the
// driver's VMM/multicast entry points resolved at run time (libcuda is not linked, so the
// library loads — and its symbols can be checked — on a box without a GPU driver).
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <vector>

#include "b2d_kernels.cuh"
#include "b2d_tma.cuh"
#include "b2d_staged.cuh"
#include "b2d_owner.cuh"
#include "b2d_syncbn.cuh"
#include "b2d_clip.cuh"
#include "b2d_launch.cuh"

using namespace b2d;

namespace {

constexpr uint32_t kMagic = 0x42324431u;  // "B2D1"
constexpr size_t kAlign = 256;
constexpr size_t kArenaGranule = 2u << 20;

thread_local std::string g_create_error;

struct HandleBlob {
  uint32_t magic;
  uint32_t version;
  int32_t rank, world, device, mem_kind;
  int64_t pid;
  uint64_t arena_bytes;
  uint64_t arena_ptr;    // valid inside the exporting process only
  uint64_t vmm_handle;   // CUmemGenericAllocationHandle, exporting process only
  int32_t fd;            // POSIX fd of the VMM allocation *in the importing process* (patched)
  int32_t pad;
  cudaIpcMemHandle_t ipc;
  uint64_t proc_nonce;   // random per process: equal pids in different pid namespaces / hosts must not look local
  unsigned char reserved[B2D_HANDLE_BYTES - 72 - sizeof(cudaIpcMemHandle_t)];
};
static_assert(sizeof(HandleBlob) == B2D_HANDLE_BYTES, "handle blob size is part of the ABI");

// ---- driver entry points (VMM + multicast), resolved lazily ------------------------------
struct Driver {
  bool tried = false, ok = false;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long);
  CUresult (*MemRelease)(CUmemGenericAllocationHandle);
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long);
  CUresult (*MemAddressFree)(CUdeviceptr, size_t);
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
  CUresult (*MemUnmap)(CUdeviceptr, size_t);
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t);
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags);
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long);
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType);
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*);
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice);
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long);
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t);
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags);
  CUresult (*DeviceGet)(CUdevice*, int);
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
  CUresult (*GetErrorString)(CUresult, const char**);
};
Driver g_drv;
std::mutex g_drv_mu;

template <typename F>
bool resolve(const char* name, F* fn) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || p == nullptr ||
      q != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    return false;
  }
  *fn = reinterpret_cast<F>(p);
  return true;
}

bool driver_ready() {
  std::lock_guard<std::mutex> lk(g_drv_mu);
  if (g_drv.tried) return g_drv.ok;
  g_drv.tried = true;
  bool ok = true;
  ok &= resolve("cuMemCreate", &g_drv.MemCreate);
  ok &= resolve("cuMemRelease", &g_drv.MemRelease);
  ok &= resolve("cuMemAddressReserve", &g_drv.MemAddressReserve);
  ok &= resolve("cuMemAddressFree", &g_drv.MemAddressFree);
  ok &= resolve("cuMemMap", &g_drv.MemMap);
  ok &= resolve("cuMemUnmap", &g_drv.MemUnmap);
  ok &= resolve("cuMemSetAccess", &g_drv.MemSetAccess);
  ok &= resolve("cuMemGetAllocationGranularity", &g_drv.MemGetAllocationGranularity);
  ok &= resolve("cuMemExportToShareableHandle", &g_drv.MemExportToShareableHandle);
  ok &= resolve("cuMemImportFromShareableHandle", &g_drv.MemImportFromShareableHandle);
  ok &= resolve("cuDeviceGet", &g_drv.DeviceGet);
  ok &= resolve("cuDeviceGetAttribute", &g_drv.DeviceGetAttribute);
  ok &= resolve("cuGetErrorString", &g_drv.GetErrorString);
  // multicast is optional
  if (!(resolve("cuMulticastCreate", &g_drv.MulticastCreate) &&
        resolve("cuMulticastAddDevice", &g_drv.MulticastAddDevice) &&
        resolve("cuMulticastBindMem", &g_drv.MulticastBindMem) &&
        resolve("cuMulticastUnbind", &g_drv.MulticastUnbind) &&
        resolve("cuMulticastGetGranularity", &g_drv.MulticastGetGranularity))) {
    g_drv.MulticastCreate = nullptr;
  }
  g_drv.ok = ok;
  return ok;
}

const char* cu_err(CUresult r) {
  const char* s = nullptr;
  if (g_drv.GetErrorString != nullptr && g_drv.GetErrorString(r, &s) == CUDA_SUCCESS && s) return s;
  return "unknown CUresult";
}

struct Slot {
  size_t off = 0;      // byte offset of the double buffer inside the arena
  size_t half = 0;     // bytes of one half
  size_t n = 0;
  int wire = -1, algo = -1, grid = 0;
  unsigned parity = 0;
  // staged exchange: the op whose phases are being issued (b2d_allreduce_bucket_phased) and, per half, the
  // event after which the half may be staged into again (its last write-back has finished)
  uint32_t op_epoch0 = 0;
  size_t op_stage_off = 0;
  cudaEvent_t reuse_ev[2] = {nullptr, nullptr};   // recorded on the write-back stream; owned by the slot (never the shared ring:
                                                  // a ring event may have been re-recorded on another stream by the time it is waited for)
};

uint64_t process_nonce() {
  static const uint64_t nonce = [] {
    uint64_t v = 0;
    FILE* f = fopen("/dev/urandom", "rb");
    if (f != nullptr) { if (fread(&v, sizeof(v), 1, f) != 1) v = 0; fclose(f); }
    if (v == 0) v = (static_cast<uint64_t>(getpid()) << 32) ^ static_cast<uint64_t>(reinterpret_cast<uintptr_t>(&v));
    return v;
  }();
  return nonce;
}

enum PeerMap { kMapNone = 0, kMapSelf, kMapDirect, kMapLegacyIpc, kMapVmm };

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); }
    if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};

}  // namespace

struct b2d_ctx {
  int rank = 0, world = 1, device = 0;
  unsigned flags = 0;
  int sm_count = 0;
  int mem_kind = 0;
  size_t arena_bytes = 0;
  unsigned char* arena = nullptr;
  CUmemGenericAllocationHandle vmm_handle = 0;
  int own_fd = -1;
  Peers peers{};
  PeerMap peer_map[B2D_MAX_WORLD] = {};
  CUmemGenericAllocationHandle peer_vmm[B2D_MAX_WORLD] = {};
  bool finalized = false;

  // multicast
  CUmemGenericAllocationHandle mc_handle = 0;
  bool mc_joined = false, mc_bound = false;
  size_t mc_size = 0;

  Diag* diag_host = nullptr;
  Diag* diag_dev = nullptr;

  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_free, ev_pending;
  uint64_t launches = 0, timed_launches = 0;
  double timed_ms = 0.0;

  std::map<int, Slot> slots;
  size_t slot_top = 0;     // slots grow up from just above the signal pad
  size_t user_bottom = 0;  // user allocations grow down from the end of the arena
  std::map<size_t, size_t> slot_free;   // offset -> bytes: regions given back by re-laid-out slots (first fit)

  // staged exchange (b2d_staged.cuh): three internal streams, a ring of ordering events (shared by every stream
  // join), the chunk epoch
  cudaStream_t s_stage = nullptr, s_xfer = nullptr, s_unstage = nullptr;
  std::vector<cudaEvent_t> ev_ring = std::vector<cudaEvent_t>(1024, nullptr);
  size_t ev_ring_idx = 0;
  cudaEvent_t last_unstage_ev = nullptr;   // own event, re-recorded after every write-back / parameter wait
  uint32_t epoch = 0;
  size_t chunk_bytes = 64u << 20;        // wire bytes per pipeline chunk (host launch cost grows with the chunk count)
  int exch_ctas = 64;                    // CTAs (256 threads) of the exchange kernel (the only one that waits for peers)
  int nvls_auto = 1;                     // AUTO may pick the in-switch reduction when a multicast object is bound
  int inplace = 1;                       // fp32 buckets that live in the arena are exchanged where they are
  uint64_t pool_allocs = 0, pool_digest = 1469598103934665603ull;   // FNV-1a over (offset, size) of pool allocations
  uint64_t exch_launches = 0, exch_timed = 0;
  double exch_ms = 0.0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> exch_pending;

  // sharded path: reduce buckets registered by the host (segment tables live in device memory)
  struct OwnerBucket {
    int nseg = 0, wire = 0;
    long long* d_flat_off = nullptr;
    unsigned* d_start = nullptr;
    unsigned owner_pack[B2D_MAX_WORLD + 1] = {};
    uint32_t op_epoch = 0;
  };
  std::map<int, OwnerBucket> owner_buckets;
  uint32_t push_epoch = 0;
  struct OptimBucket { int nseg = 0; size_t n = 0; float** d_ptr = nullptr; unsigned* d_start = nullptr; };   // d_ptr: [3][nseg] params | state1 | state2
  std::map<int, OptimBucket> optim_buckets;

  // synchronised BatchNorm (b2d_syncbn.cuh): one arena region per registered layer, laid out as
  // [forward gen 0 | forward gen 1 | backward gen 0 | backward gen 1], each generation W rows.  Index d: 0 forward,
  // 1 backward.  op_epoch[d] != 0 while a pushed exchange waits for its combine phase.
  struct BnLayer {
    int channels = 0;
    size_t off = 0;
    unsigned calls[2] = {0, 0};
    unsigned op_gen[2] = {0, 0};
    uint32_t op_epoch[2] = {0, 0};
  };
  std::map<int, BnLayer> bn_layers;
  uint32_t bn_epoch = 0;   // the BN exchanges' own epoch (Signal::bn), independent of the bucket exchanges' `epoch`

  // gradient clipping (b2d_clip.cuh): one arena region, [gen 0: W slots | gen 1: W slots | kClipGMax block sums],
  // taken by b2d_clip_register.  clip_op_epoch != 0 while a pushed partial waits for its combine phase.
  bool clip_registered = false;
  size_t clip_off = 0;
  unsigned clip_calls = 0, clip_gen = 0;
  uint32_t clip_epoch = 0, clip_op_epoch = 0;   // Signal::clip's own epoch, independent of `epoch` and `bn_epoch`

  unsigned long long* trace_dev = nullptr;   // debug: per-block phase stamps of the LAST allreduce launch
  int trace_grid = 0;

  // 64 CTAs: inside a training step a larger grid waits longer for SMs to drain from the backward kernels than
  // it gains, although it is faster in isolation.  b2d_ctx_set_max_ctas raises it.
  int max_ctas = 64;
  int tma_ctas = 48;        // CTAs of the TMA-staged kernel (b2d_ctx_set_max_ctas caps it too)
  int tma_ctas_user = 0;
  size_t one_shot_max_bytes = 1024 * 1024;
  bool one_shot_max_user = false;
  int auto_profile = B2D_PROFILE_OVERLAP;
  // peer watchdog: minutes, like a process-group timeout — a rank that is late because of a slow data loader,
  // rank-0 logging or a debugger pause must not poison the CUDA context (b2d_ctx_set_timeout; 0 = never trap)
  unsigned timeout_ms = 600000;
  int last_algo = 0, last_grid = 0, last_block = 0;

  std::string err;
  std::mutex mu;
};

namespace {

int fail(b2d_ctx* ctx, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx != nullptr) ctx->err = buf; else g_create_error = buf;
  return code;
}

#define B2D_CUDA(ctx, expr)                                                                  \
  do {                                                                                       \
    cudaError_t e__ = (expr);                                                                \
    if (e__ != cudaSuccess) {                                                                \
      cudaGetLastError();                                                                    \
      return fail((ctx), B2D_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                  __FILE__, __LINE__);                                                       \
    }                                                                                        \
  } while (0)

#define B2D_CU(ctx, expr)                                                                    \
  do {                                                                                       \
    CUresult r__ = (expr);                                                                   \
    if (r__ != CUDA_SUCCESS)                                                                 \
      return fail((ctx), B2D_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cu_err(r__), __FILE__, \
                  __LINE__);                                                                 \
  } while (0)

size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int vmm_map(b2d_ctx* ctx, CUmemGenericAllocationHandle h, size_t bytes, int device, unsigned char** out) {
  CUdeviceptr va = 0;
  B2D_CU(ctx, g_drv.MemAddressReserve(&va, bytes, kArenaGranule, 0, 0));
  CUresult r = g_drv.MemMap(va, bytes, 0, h, 0);
  if (r != CUDA_SUCCESS) {
    g_drv.MemAddressFree(va, bytes);
    return fail(ctx, B2D_ERR_CUDA, "cuMemMap failed: %s", cu_err(r));
  }
  CUmemAccessDesc desc{};
  desc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  desc.location.id = device;
  desc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = g_drv.MemSetAccess(va, bytes, &desc, 1);
  if (r != CUDA_SUCCESS) {
    g_drv.MemUnmap(va, bytes);
    g_drv.MemAddressFree(va, bytes);
    return fail(ctx, B2D_ERR_CUDA, "cuMemSetAccess failed: %s", cu_err(r));
  }
  *out = reinterpret_cast<unsigned char*>(va);
  return B2D_OK;
}

void vmm_unmap(unsigned char* p, size_t bytes) {
  if (p == nullptr) return;
  g_drv.MemUnmap(reinterpret_cast<CUdeviceptr>(p), bytes);
  g_drv.MemAddressFree(reinterpret_cast<CUdeviceptr>(p), bytes);
}

using TimingPair = std::pair<cudaEvent_t, cudaEvent_t>;

// Adds the finished pairs of `pending` to (count, ms) and returns them to the free list; `block` waits for all of them.
void resolve_pairs(b2d_ctx* ctx, std::vector<TimingPair>& pending, uint64_t& count, double& total_ms, bool block) {
  size_t keep = 0;
  for (size_t i = 0; i < pending.size(); ++i) {
    TimingPair& pr = pending[i];
    cudaError_t q = block ? cudaEventSynchronize(pr.second) : cudaEventQuery(pr.second);
    if (q == cudaSuccess) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) {
        total_ms += ms;
        count += 1;
      } else {
        cudaGetLastError();
      }
      ctx->ev_free.push_back(pr);
    } else {
      cudaGetLastError();
      pending[keep++] = pr;
    }
  }
  pending.resize(keep);
}

void resolve_timing(b2d_ctx* ctx, bool block) {
  resolve_pairs(ctx, ctx->ev_pending, ctx->timed_launches, ctx->timed_ms, block);
  resolve_pairs(ctx, ctx->exch_pending, ctx->exch_timed, ctx->exch_ms, block);
}

// A free pair of timing events.  Once 8192 pairs are unresolved, the work goes untimed rather than growing the pool.
bool take_timing_pair(b2d_ctx* ctx, TimingPair* out) {
  if (ctx->ev_free.empty() && ctx->ev_pending.size() + ctx->exch_pending.size() >= 8192) resolve_timing(ctx, false);
  if (ctx->ev_free.empty()) {
    if (ctx->ev_pending.size() + ctx->exch_pending.size() >= 8192) return false;
    cudaEvent_t a, b;
    if (cudaEventCreate(&a) != cudaSuccess) { cudaGetLastError(); return false; }
    if (cudaEventCreate(&b) != cudaSuccess) { cudaGetLastError(); cudaEventDestroy(a); return false; }
    ctx->ev_free.emplace_back(a, b);
  }
  *out = ctx->ev_free.back();
  ctx->ev_free.pop_back();
  return true;
}

// A span of work on one stream, timed into `pending` (ev_pending or exch_pending) when the context times its
// launches.  The pair is taken at construction; start() and stop() record its two events.
struct TimedSpan {
  b2d_ctx* ctx;
  std::vector<TimingPair>& pending;
  TimingPair ev{nullptr, nullptr};
  bool timing;
  TimedSpan(b2d_ctx* c, std::vector<TimingPair>& p)
      : ctx(c), pending(p), timing((c->flags & B2D_FLAG_TIMING) && take_timing_pair(c, &ev)) {}
  int start(cudaStream_t st) {
    if (timing) B2D_CUDA(ctx, cudaEventRecord(ev.first, st));
    return B2D_OK;
  }
  int stop(cudaStream_t st) {
    if (timing) {
      B2D_CUDA(ctx, cudaEventRecord(ev.second, st));
      pending.push_back(ev);
    }
    return B2D_OK;
  }
};

// The next event of the ring of ordering events (b2d_ctx_create makes them).
cudaEvent_t next_event(b2d_ctx* ctx) { return ctx->ev_ring[ctx->ev_ring_idx++ % ctx->ev_ring.size()]; }

// `waiter` runs what is issued to it next only after everything already issued to `waited`.
int join(b2d_ctx* ctx, cudaStream_t waiter, cudaStream_t waited) {
  cudaEvent_t e = next_event(ctx);
  B2D_CUDA(ctx, cudaEventRecord(e, waited));
  B2D_CUDA(ctx, cudaStreamWaitEvent(waiter, e, 0));
  return B2D_OK;
}

// Launches `kernel` and counts the launch.
template <typename Kernel, typename... Args>
void launch(b2d_ctx* ctx, Kernel kernel, int grid, int block, size_t smem, cudaStream_t st, const Args&... args) {
  kernel<<<grid, block, smem, st>>>(args...);
  ctx->launches += 1;
}

// The end of every entry point that launched: a launch that could not be enqueued is an error.
int launch_result(b2d_ctx* ctx, const char* what = "kernel") {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(ctx, B2D_ERR_CUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
  return B2D_OK;
}

// One timed kernel on `comm` behind `wait_stream` (K0-K6), recorded as the context's last launch.
template <typename Kernel, typename... Args>
int launch_timed(b2d_ctx* ctx, void* wait_stream, void* comm_stream, int algo, Kernel kernel, int grid, int block,
                 size_t smem, const Args&... args) {
  cudaStream_t ws = static_cast<cudaStream_t>(wait_stream), comm = static_cast<cudaStream_t>(comm_stream);
  int rc = ws != comm ? join(ctx, comm, ws) : B2D_OK;
  if (rc != B2D_OK) return rc;
  TimedSpan span(ctx, ctx->ev_pending);
  rc = span.start(comm);
  if (rc != B2D_OK) return rc;
  launch(ctx, kernel, grid, block, smem, comm, args...);
  ctx->last_algo = algo; ctx->last_grid = grid; ctx->last_block = kThreads;
  rc = launch_result(ctx);
  return rc != B2D_OK ? rc : span.stop(comm);
}

// The fields of a kernel's parameters that let it wait for peers, from the context.
template <typename Params>
void set_peer_wait(const b2d_ctx* ctx, Params* P) {
  set_peer_wait(P, ctx->rank, ctx->world, ctx->peers, static_cast<unsigned long long>(ctx->timeout_ms) * 1000000ull,
                ctx->diag_dev);
}

// ceil(work / per_cta) CTAs, at least one, at most cap
int clamp_grid(size_t work, size_t per_cta, size_t cap) {
  return static_cast<int>(std::min(std::max<size_t>((work + per_cta - 1) / per_cta, 1), cap));
}

int launch_barrier(b2d_ctx* ctx, cudaStream_t stream) {
  ArParams P{};
  set_peer_wait(ctx, &P);
  launch(ctx, barrier_kernel, B2D_MAX_BLOCKS, 32, 0, stream, P);
  return launch_result(ctx, "barrier");
}

bool is_staged(int algo) { return algo == B2D_ALGO_STAGED || algo == B2D_ALGO_NVLS; }

int pick_algo(b2d_ctx* ctx, size_t n, int wire, int algo) {
  if (ctx->world == 1) return B2D_ALGO_ONE_SHOT;
  if (algo == B2D_ALGO_TWO_SHOT_TMA && (wire != B2D_WIRE_BF16 || n % 8 != 0)) return B2D_ALGO_TWO_SHOT;
  if (algo != B2D_ALGO_AUTO) return algo;
  const size_t wire_bytes = n * (wire == B2D_WIRE_BF16 ? 2 : 4);
  const int W = ctx->world;
  const bool nvls = ctx->mc_bound && ctx->nvls_auto && W >= 4;
  // Small buckets: one kernel, one barrier, every rank reads everything.  Cross-over: 16 MiB at world 2 (the
  // same bytes as any two-shot scheme), 4 MiB at world 4, 1 MiB at world 8; b2d_ctx_set_one_shot_max_bytes
  // overrides it for a given fabric.
  size_t one_shot_max = ctx->one_shot_max_bytes;
  if (!ctx->one_shot_max_user) one_shot_max = W == 2 ? (16u << 20) : (W <= 4 ? (4u << 20) : (1u << 20));
  if (ctx->auto_profile == B2D_PROFILE_LATENCY) {
    // an isolated call, nothing to overlap with: the single-kernel algorithms are ahead of the staged pipeline's
    // four launches up to ~100 MiB; beyond that the chunk pipeline hides the cast passes behind the link
    if (wire_bytes <= one_shot_max) return B2D_ALGO_ONE_SHOT;
    if (nvls && W >= 8) return wire_bytes <= (96u << 20) ? B2D_ALGO_NVLS_FUSED : B2D_ALGO_NVLS;
    return B2D_ALGO_TWO_SHOT;
  }
  // B2D_PROFILE_OVERLAP (default; the DDP hook): the exchange shares the GPU with backward kernels.  The staged
  // pipeline's streaming kernels never spin and its exchange kernel holds a few half-SMs only, which is worth more
  // inside a training step than the few microseconds of extra launches it loses in isolation.
  if (wire_bytes <= (W == 2 ? one_shot_max : (one_shot_max < (1u << 20) ? one_shot_max : (1u << 20)))) return B2D_ALGO_ONE_SHOT;
  // the in-switch reduction pays from 4 ranks up ((1 + 1/W) N w bytes per direction instead of 2 (W-1)/W N w)
  return nvls ? B2D_ALGO_NVLS : B2D_ALGO_STAGED;
}

// macro-tile size (packs) of the TMA kernel for a given grid: spread the slice over the grid, 8..4096
int tma_mt(size_t slice, int grid) {
  size_t mt = (slice + grid - 1) / grid;
  mt = (mt + 7) / 8 * 8;
  if (mt < 8) mt = 8;
  if (mt > static_cast<size_t>(kTmaMaxMt)) mt = kTmaMaxMt;
  return static_cast<int>(mt);
}

// packs per pipeline chunk of the staged exchange: a multiple of the world size, at least one CTA's worth
size_t staged_chunk_packs(const b2d_ctx* ctx) {
  size_t cp = ctx->chunk_bytes / 16;
  const size_t unit = static_cast<size_t>(ctx->world) * 1024;
  cp = cp / unit * unit;
  return cp < unit ? unit : cp;
}

int exch_grid(const b2d_ctx* ctx, size_t chunk_packs, int algo) {
  const size_t slice = (chunk_packs + ctx->world - 1) / ctx->world;
  const size_t per_thread = algo == B2D_ALGO_NVLS ? 8 : (ctx->world <= 8 && kMaxLoadsInFlight / ctx->world > 1 ? kMaxLoadsInFlight / ctx->world : 1);
  // multimem keeps the link busy from fewer CTAs: NVLS uses half the P2P budget
  const size_t cap = algo == B2D_ALGO_NVLS ? static_cast<size_t>(ctx->exch_ctas > 1 ? ctx->exch_ctas / 2 : 1) : static_cast<size_t>(ctx->exch_ctas);
  return clamp_grid(slice, kExThreads * per_thread, cap);
}

// S / U: plain streaming kernels.  At most ONE wave (4 CTAs of 256 threads per SM, __launch_bounds__(256, 4)): a grid a
// few CTAs larger than the machine holds costs a whole second wave, which roughly doubles the pass.
int stream_grid(const b2d_ctx* ctx, size_t packs) {
  return clamp_grid(packs, kStThreads * 8, static_cast<size_t>(ctx->sm_count) * 4);
}

int pick_grid(b2d_ctx* ctx, size_t n, int wire, int algo) {
  const size_t epp = wire == B2D_WIRE_BF16 ? 8 : 4;
  const size_t npacks = (n + epp - 1) / epp;
  if (is_staged(algo)) {
    const size_t cp = staged_chunk_packs(ctx);
    return exch_grid(ctx, npacks < cp ? npacks : cp, algo);
  }
  if (algo == B2D_ALGO_TWO_SHOT_TMA) {
    const size_t slice = (npacks + ctx->world - 1) / ctx->world;
    return clamp_grid(slice, 256, ctx->tma_ctas);   // at least 4 KiB of wire per block and slice
  }
  size_t work = npacks;
  if (algo != B2D_ALGO_ONE_SHOT) work = (npacks + ctx->world - 1) / ctx->world;
  return clamp_grid(work, kThreads, ctx->max_ctas);
}

int ensure_streams(b2d_ctx* ctx) {
  if (ctx->s_stage != nullptr) return B2D_OK;
  int lo = 0, hi = 0;   // "greatest" priority is the numerically lowest
  if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess) { cudaGetLastError(); lo = hi = 0; }
  // the exchange stream outranks the two streaming ones: its few CTAs take the first half-SM that frees up, so
  // chunk c crosses NVLink while chunk c+1 is still being staged; all three outrank default-priority compute
  const int lower = hi < lo ? hi + 1 : hi;
  B2D_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->s_stage, cudaStreamNonBlocking, lower));
  B2D_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->s_xfer, cudaStreamNonBlocking, hi));
  B2D_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->s_unstage, cudaStreamNonBlocking, lower));
  return B2D_OK;
}

// The final join of the internal streams: `comm` waits for everything issued to s_unstage, and last_unstage_ev marks
// that point for get_slot's drain.
int join_unstage(b2d_ctx* ctx, cudaStream_t comm) {
  int rc = join(ctx, comm, ctx->s_unstage);
  if (rc != B2D_OK) return rc;
  if (ctx->last_unstage_ev == nullptr) B2D_CUDA(ctx, cudaEventCreateWithFlags(&ctx->last_unstage_ev, cudaEventDisableTiming));
  B2D_CUDA(ctx, cudaEventRecord(ctx->last_unstage_ev, ctx->s_unstage));
  return B2D_OK;
}

// first-fit region allocator for bucket slots (identical call sequence on every rank => identical offsets)
bool slot_region_alloc(b2d_ctx* ctx, size_t bytes, size_t* off) {
  for (auto it = ctx->slot_free.begin(); it != ctx->slot_free.end(); ++it) {
    if (it->second >= bytes) {
      *off = it->first;
      const size_t rest = it->second - bytes;
      const size_t rest_off = it->first + bytes;
      ctx->slot_free.erase(it);
      if (rest > 0) ctx->slot_free[rest_off] = rest;
      return true;
    }
  }
  if (ctx->slot_top + bytes > ctx->user_bottom) return false;
  *off = ctx->slot_top;
  ctx->slot_top += bytes;
  return true;
}

void slot_region_free(b2d_ctx* ctx, size_t off, size_t bytes) {
  if (bytes == 0) return;
  ctx->slot_free[off] = bytes;
  auto it = ctx->slot_free.find(off);
  auto nx = std::next(it);
  if (nx != ctx->slot_free.end() && it->first + it->second == nx->first) { it->second += nx->second; ctx->slot_free.erase(nx); }
  if (it != ctx->slot_free.begin()) {
    auto pv = std::prev(it);
    if (pv->first + pv->second == it->first) { pv->second += it->second; ctx->slot_free.erase(it); it = pv; }
  }
  if (it->first + it->second == ctx->slot_top) { ctx->slot_top = it->first; ctx->slot_free.erase(it); }
}

// Arena slot of a bucket: two halves used alternately, so that a rank may start staging
// step k+1 while a slow peer still reads step k's payload (see DESIGN.md §5).
int get_slot(b2d_ctx* ctx, int key, size_t half_bytes, size_t n, int wire, int algo, int grid,
             cudaStream_t stream, size_t* stage_off, Slot** slot_out = nullptr, int* half_out = nullptr,
             bool single = false) {
  half_bytes = round_up(half_bytes, kAlign);
  if (single) half_bytes = round_up((half_bytes + 1) / 2, kAlign);   // one buffer: two "halves" of half the size
  Slot& s = ctx->slots[key];
  const bool same = s.half >= half_bytes && s.n == n && s.wire == wire && s.algo == algo && s.grid == grid;
  if (!same) {
    if (s.half != 0) {
      // geometry changed (DDP rebuilt its buckets, reducer.hpp:125-151): peers may still read the old layout
      // of this region — drain the own staged pipeline into `stream`, then meet every peer, before anything
      // is re-mapped; the staging stream continues behind that barrier
      if (ctx->last_unstage_ev != nullptr) B2D_CUDA(ctx, cudaStreamWaitEvent(stream, ctx->last_unstage_ev, 0));
      int rc = launch_barrier(ctx, stream);
      if (rc != B2D_OK) return rc;
      if (ctx->s_stage != nullptr) {
        cudaEvent_t e = next_event(ctx);
        B2D_CUDA(ctx, cudaEventRecord(e, stream));
        B2D_CUDA(ctx, cudaStreamWaitEvent(ctx->s_stage, e, 0));
        B2D_CUDA(ctx, cudaStreamWaitEvent(ctx->s_xfer, e, 0));
      }
    }
    if (s.half < half_bytes) {
      const size_t old_off = s.off, old_bytes = 2 * s.half;
      slot_region_free(ctx, old_off, old_bytes);   // behind the barrier above
      size_t off = 0;
      if (!slot_region_alloc(ctx, 2 * half_bytes, &off)) {
        s.half = 0; s.off = 0; s.n = 0;
        return fail(ctx, B2D_ERR_NOMEM,
                    "symmetric arena exhausted: slot %d needs 2 x %zu bytes, %zu free of %zu", key,
                    half_bytes, ctx->user_bottom - ctx->slot_top, ctx->arena_bytes);
      }
      s.off = off;
      s.half = half_bytes;
    }
    s.n = n; s.wire = wire; s.algo = algo; s.grid = grid;
  }
  if (single) {   // the caller guarantees a fence between consecutive uses (sharded path: the parameter exchange)
    *stage_off = s.off;
    if (slot_out != nullptr) *slot_out = &s;
    if (half_out != nullptr) *half_out = 0;
    return B2D_OK;
  }
  *stage_off = s.off + (s.parity & 1u) * s.half;
  if (slot_out != nullptr) *slot_out = &s;
  if (half_out != nullptr) *half_out = static_cast<int>(s.parity & 1u);
  s.parity ^= 1u;
  return B2D_OK;
}

// K2T's selector (b2d_launch.cuh holds the others; the emulator does not compile b2d_tma.cuh)
auto select_k2t(int world) {
  return dispatch_world(world, [](auto w) { return &k2t_two_shot_tma_kernel<decltype(w)::value, true>; });
}

// CUDA loads kernels lazily; a load can serialise against running work, and these kernels spin on
// peers.  Load every kernel a selector can return up front (what NCCL does at communicator init).
template <typename K>
void preload_one(K kernel) {
  cudaFuncAttributes a;
  if (cudaFuncGetAttributes(&a, kernel) != cudaSuccess) cudaGetLastError();
}
void preload_kernels() {
  for (int w : {0, 2, 4, 8}) {
    if (cudaFuncSetAttribute(select_k2t(w), cudaFuncAttributeMaxDynamicSharedMemorySize, kTmaSmemBytes) != cudaSuccess)
      cudaGetLastError();
    preload_one(select_k2t(w));
    for (bool a : {false, true}) {
      preload_one(select_k1(w, a));
      preload_one(select_k456(w, a));
      for (bool b : {false, true}) {
        preload_one(select_k2(w, a, b));
        preload_one(select_seg_reduce(w, a, b));
        preload_one(select_adam_push(w, a, b));
        for (bool c : {false, true})
          if (!(a && c)) preload_one(select_exch(w, a, b, c));   // bf16 in place is the fp32 in-place kernel
      }
    }
  }
  for (bool a : {false, true}) {
    preload_one(select_k0(a));
    preload_one(select_stage(a));
    preload_one(select_unstage(a));
    preload_one(select_seg_stage(a));
    preload_one(select_bn_combine(a));
  }
  preload_one(barrier_kernel); preload_one(arrive_kernel); preload_one(wait_published_kernel); preload_one(peer_read_kernel);
  preload_one(bucket_optim_kernel); preload_one(bn_push_kernel); preload_one(sqnorm_partial_kernel); preload_one(clip_coef_kernel);
}

// The staged exchange of one bucket (b2d_staged.cuh): S on s_stage, X on s_xfer, W+U on s_unstage, chunk by
// chunk; `comm` only receives the final join.  `phases` (bit 0 S, bit 1 X, bit 2 W+U) lets single-process
// multi-rank drivers (loopback tests, smoke under ncu) issue the phases of ALL ranks in phase-major order.
int launch_staged(b2d_ctx* ctx, int key, float* grad, size_t n, int wire, float scale, int algo, unsigned phases,
                  cudaStream_t wait_s, cudaStream_t comm) {
  int rc = ensure_streams(ctx);
  if (rc != B2D_OK) return rc;
  const bool bf16 = wire == B2D_WIRE_BF16, nvls = algo == B2D_ALGO_NVLS;
  const size_t epp = bf16 ? 8 : 4;
  const size_t npacks = (n + epp - 1) / epp;
  const unsigned char* g8 = reinterpret_cast<const unsigned char*>(grad);
  const bool inplace = ctx->inplace && !bf16 && g8 >= ctx->arena + kSignalBytes && g8 + npacks * 16 <= ctx->arena + ctx->arena_bytes;
  const size_t cp = staged_chunk_packs(ctx);
  const int nchunks = static_cast<int>((npacks + cp - 1) / cp);

  Slot* slot = nullptr;
  int half = 0;
  size_t stage_off = 0;
  if (inplace) {
    slot = &ctx->slots[key];          // bookkeeping only (epoch of the op in flight); owns no arena bytes
    stage_off = static_cast<size_t>(g8 - ctx->arena);
    if (phases & 1u) slot->op_stage_off = stage_off;
  } else if (phases & 1u) {
    rc = get_slot(ctx, key, npacks * 16, n, wire, algo, 0, comm, &stage_off, &slot, &half);
    if (rc != B2D_OK) return rc;
    slot->op_stage_off = stage_off;
  } else {
    auto it = ctx->slots.find(key);
    if (it == ctx->slots.end() || it->second.op_epoch0 == 0) return fail(ctx, B2D_ERR_STATE, "phase issued before phase 0 of bucket %d", key);
    slot = &it->second;
    stage_off = slot->op_stage_off;
    half = static_cast<int>((slot->parity ^ 1u) & 1u);
  }
  if (phases & 1u) {
    slot->op_epoch0 = ctx->epoch + 1u;
    ctx->epoch += static_cast<uint32_t>(nchunks);
  }
  const uint32_t epoch0 = slot->op_epoch0;
  if (epoch0 == 0) return fail(ctx, B2D_ERR_STATE, "phase issued before phase 0 of bucket %d", key);

  StParams SP{};
  SP.scale = scale; SP.rank = ctx->rank; SP.world = ctx->world; SP.peers = ctx->peers;
  ExParams XP{};
  XP.scale = scale;
  set_peer_wait(ctx, &XP);

  std::vector<cudaEvent_t> ev_s(nchunks, nullptr), ev_x(nchunks, nullptr);
  if (phases & 1u) {
    rc = join(ctx, ctx->s_stage, wait_s);
    if (rc != B2D_OK) return rc;
    if (!inplace && slot->reuse_ev[half] != nullptr) B2D_CUDA(ctx, cudaStreamWaitEvent(ctx->s_stage, slot->reuse_ev[half], 0));
    if (inplace) {
      SP.epoch = epoch0 + static_cast<uint32_t>(nchunks) - 1u;   // the whole bucket is ready at once
      launch(ctx, arrive_kernel, 1, 32, 0, ctx->s_stage, SP);
      cudaEvent_t es = next_event(ctx);
      B2D_CUDA(ctx, cudaEventRecord(es, ctx->s_stage));
      for (int c = 0; c < nchunks; ++c) ev_s[c] = es;
    } else {
      for (int c = 0; c < nchunks; ++c) {
        const ChunkSpan cs = chunk_span(c, npacks, cp, n, epp);
        SP.grad = grad + cs.p0 * epp;
        SP.n = cs.n;
        SP.wire = reinterpret_cast<uint4*>(ctx->arena + stage_off) + cs.p0;
        SP.epoch = epoch0 + static_cast<uint32_t>(c);
        launch(ctx, select_stage(bf16), stream_grid(ctx, cs.packs), kStThreads, 0, ctx->s_stage, SP);
        ev_s[c] = next_event(ctx);
        B2D_CUDA(ctx, cudaEventRecord(ev_s[c], ctx->s_stage));
      }
    }
  }
  if (phases & 2u) {
    TimedSpan span(ctx, ctx->exch_pending);   // one pair around all the chunks
    for (int c = 0; c < nchunks; ++c) {
      const ChunkSpan cs = chunk_span(c, npacks, cp, n, epp);
      if (ev_s[c] != nullptr && (c == 0 || ev_s[c] != ev_s[c - 1])) B2D_CUDA(ctx, cudaStreamWaitEvent(ctx->s_xfer, ev_s[c], 0));
      if (c == 0 && (rc = span.start(ctx->s_xfer)) != B2D_OK) return rc;
      XP.wire_off = stage_off + cs.p0 * 16;
      XP.npacks = cs.packs;
      XP.n_valid = inplace ? cs.n_valid : 0;
      XP.epoch = epoch0 + static_cast<uint32_t>(c);
      const int grid = exch_grid(ctx, cs.packs, algo);
      launch(ctx, select_exch(ctx->world, bf16, nvls, inplace), grid, kExThreads, 0, ctx->s_xfer, XP);
      ctx->exch_launches += 1;
      ctx->last_grid = grid;
      ev_x[c] = next_event(ctx);
      B2D_CUDA(ctx, cudaEventRecord(ev_x[c], ctx->s_xfer));
    }
    rc = span.stop(ctx->s_xfer);
    if (rc != B2D_OK) return rc;
  }
  if (phases & 4u) {
    for (int c = 0; c < nchunks; ++c) {
      if (ev_x[c] != nullptr) B2D_CUDA(ctx, cudaStreamWaitEvent(ctx->s_unstage, ev_x[c], 0));
      XP.epoch = epoch0 + static_cast<uint32_t>(c);
      launch(ctx, wait_published_kernel, 1, 32, 0, ctx->s_unstage, XP);
      if (!inplace) {
        const ChunkSpan cs = chunk_span(c, npacks, cp, n, epp);
        SP.grad = grad + cs.p0 * epp;
        SP.n = cs.n;
        SP.wire = reinterpret_cast<uint4*>(ctx->arena + stage_off) + cs.p0;
        SP.epoch = epoch0 + static_cast<uint32_t>(c);
        launch(ctx, select_unstage(bf16), stream_grid(ctx, cs.packs), kStThreads, 0, ctx->s_unstage, SP);
      }
    }
    rc = join_unstage(ctx, comm);
    if (rc != B2D_OK) return rc;
    if (!inplace) {
      if (slot->reuse_ev[half] == nullptr) B2D_CUDA(ctx, cudaEventCreateWithFlags(&slot->reuse_ev[half], cudaEventDisableTiming));
      B2D_CUDA(ctx, cudaEventRecord(slot->reuse_ev[half], ctx->s_unstage));
    }
    slot->op_epoch0 = 0;
  }
  rc = launch_result(ctx);
  if (rc != B2D_OK) return rc;
  ctx->last_algo = algo; ctx->last_block = kExThreads;
  return B2D_OK;
}

void free_tables(b2d_ctx::OwnerBucket& b) { cudaFree(b.d_flat_off); cudaFree(b.d_start); }
void free_tables(b2d_ctx::OptimBucket& b) { cudaFree(b.d_ptr); cudaFree(b.d_start); }

// Copies a host table to a new device allocation.
template <typename T>
int upload_table(b2d_ctx* ctx, const std::vector<T>& v, T** out) {
  void* p = nullptr;
  B2D_CUDA(ctx, cudaMalloc(&p, v.size() * sizeof(T)));
  *out = static_cast<T*>(p);
  B2D_CUDA(ctx, cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return B2D_OK;
}

// Forgets bucket `id` of `buckets` before it is registered again.  Its device tables are freed once the device is idle:
// kernels still in flight may read them.
template <typename Bucket>
int drop_bucket(b2d_ctx* ctx, std::map<int, Bucket>& buckets, int id) {
  auto it = buckets.find(id);
  if (it == buckets.end()) return B2D_OK;
  B2D_CUDA(ctx, cudaDeviceSynchronize());
  free_tables(it->second);
  buckets.erase(it);
  return B2D_OK;
}

// shard_off[0 .. world]: the owner shards of [0, n), non-decreasing multiples of 8.  *max_len: the longest shard.
int check_shard_off(b2d_ctx* ctx, const int64_t* shard_off, size_t n, size_t* max_len) {
  if (shard_off[0] != 0 || static_cast<size_t>(shard_off[ctx->world]) != n)
    return fail(ctx, B2D_ERR_INVALID, "shard_off must start at 0 and end at n");
  *max_len = 0;
  for (int r = 0; r < ctx->world; ++r) {
    if (shard_off[r + 1] < shard_off[r] || shard_off[r] % 8 != 0 || shard_off[r + 1] % 8 != 0)
      return fail(ctx, B2D_ERR_INVALID, "shard offsets must be non-decreasing multiples of 8 (got %lld..%lld for rank %d)",
                  (long long)shard_off[r], (long long)shard_off[r + 1], r);
    *max_len = std::max(*max_len, static_cast<size_t>(shard_off[r + 1] - shard_off[r]));
  }
  return B2D_OK;
}

int check_ready(b2d_ctx* ctx) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (!ctx->finalized) return fail(ctx, B2D_ERR_STATE, "b2d_ctx_finalize() has not been called");
  if (ctx->diag_host != nullptr && ctx->diag_host->code != 0)
    return fail(ctx, B2D_ERR_PEER,
                "peer timeout recorded: rank %u block %u waited for peer %u (expected epoch %u, saw %u)",
                ctx->diag_host->rank, ctx->diag_host->block, ctx->diag_host->peer,
                ctx->diag_host->expect, ctx->diag_host->got);
  return B2D_OK;
}

// The way into an entry point: check_ready (`ready`) or only a NULL check, then the context's lock.  use_device()
// switches to the context's device until the entry point returns; an entry point that allocates or launches calls it
// after its argument checks.
struct Entry {
  b2d_ctx* ctx;
  int rc;
  std::unique_lock<std::mutex> lk;
  std::optional<DeviceGuard> guard;
  Entry(b2d_ctx* c, bool ready)
      : ctx(c), rc(ready ? check_ready(c) : c == nullptr ? fail(nullptr, B2D_ERR_INVALID, "ctx is NULL") : B2D_OK) {
    if (rc == B2D_OK) lk = std::unique_lock<std::mutex>(c->mu);
  }
  int use_device() {
    guard.emplace(ctx->device);
    return guard->ok ? B2D_OK : fail(ctx, B2D_ERR_CUDA, "cudaSetDevice(%d) failed", ctx->device);
  }
};

}  // namespace

// =========================================================================================
extern "C" {

int b2d_version(void) { return B2D_VERSION; }

const char* b2d_last_error(b2d_ctx* ctx) {
  return ctx != nullptr ? ctx->err.c_str() : g_create_error.c_str();
}

int b2d_ctx_create(int rank, int world, int device, size_t arena_bytes, unsigned flags, b2d_ctx** out) {
  if (out == nullptr) return fail(nullptr, B2D_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (world < 1 || world > B2D_MAX_WORLD || rank < 0 || rank >= world)
    return fail(nullptr, B2D_ERR_INVALID, "bad rank/world %d/%d (max world %d)", rank, world, B2D_MAX_WORLD);
  int ndev = 0;
  {
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(nullptr, B2D_ERR_CUDA, "no usable CUDA device: %s", cudaGetErrorString(e));
    }
  }
  if (device < 0 || device >= ndev) return fail(nullptr, B2D_ERR_INVALID, "device %d out of range (%d visible)", device, ndev);
  cudaDeviceProp prop;
  B2D_CUDA(nullptr, cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, B2D_ERR_UNSUPPORTED, "libb2d is built for sm_90a; device %d is sm_%d%d", device, prop.major, prop.minor);

  DeviceGuard guard(device);
  if (!guard.ok) return fail(nullptr, B2D_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  B2D_CUDA(nullptr, cudaFree(0));  // make sure the primary context exists

  b2d_ctx* ctx = new b2d_ctx();
  ctx->rank = rank; ctx->world = world; ctx->device = device; ctx->flags = flags;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->mem_kind = (flags & B2D_FLAG_MEM_VMM) ? 1 : 0;
  ctx->arena_bytes = round_up(arena_bytes + kSignalBytes, kArenaGranule);

  auto bail = [&](int code) { std::string m = ctx->err; b2d_ctx_destroy(ctx); g_create_error = m; return code; };

  if (ctx->mem_kind == 1) {
    if (!driver_ready()) return bail(fail(ctx, B2D_ERR_UNSUPPORTED, "CUDA VMM driver entry points not available"));
    CUmemAllocationProp ap{};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = device;
    ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gran = kArenaGranule;
    if (g_drv.MemGetAllocationGranularity(&gran, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && gran > 0)
      ctx->arena_bytes = round_up(ctx->arena_bytes, gran);
    if (g_drv.MulticastCreate != nullptr) {
      CUmulticastObjectProp mp{};
      mp.numDevices = world > 1 ? world : 2;
      mp.size = ctx->arena_bytes;
      mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      size_t mg = 0;
      if (g_drv.MulticastGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && mg > 0)
        ctx->arena_bytes = round_up(ctx->arena_bytes, mg);
    }
    CUresult r = g_drv.MemCreate(&ctx->vmm_handle, ctx->arena_bytes, &ap, 0);
    if (r != CUDA_SUCCESS) return bail(fail(ctx, B2D_ERR_CUDA, "cuMemCreate(%zu) failed: %s", ctx->arena_bytes, cu_err(r)));
    int rc = vmm_map(ctx, ctx->vmm_handle, ctx->arena_bytes, device, &ctx->arena);
    if (rc != B2D_OK) return bail(rc);
  } else {
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, ctx->arena_bytes);
    if (e != cudaSuccess) { cudaGetLastError(); return bail(fail(ctx, B2D_ERR_CUDA, "cudaMalloc(%zu) failed: %s", ctx->arena_bytes, cudaGetErrorString(e))); }
    ctx->arena = static_cast<unsigned char*>(p);
  }
  {
    // only the signal pad has to start at zero
    cudaError_t e = cudaMemset(ctx->arena, 0, kSignalBytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaGetLastError(); return bail(fail(ctx, B2D_ERR_CUDA, "arena memset failed: %s", cudaGetErrorString(e))); }
  }
  ctx->peers.arena[rank] = ctx->arena;
  ctx->peers.signal[rank] = reinterpret_cast<Signal*>(ctx->arena);
  ctx->peer_map[rank] = kMapSelf;
  ctx->slot_top = kSignalBytes;
  ctx->user_bottom = ctx->arena_bytes;

  {
    void* h = nullptr;
    cudaError_t e = cudaHostAlloc(&h, sizeof(Diag), cudaHostAllocMapped);
    if (e == cudaSuccess) {
      memset(h, 0, sizeof(Diag));
      ctx->diag_host = static_cast<Diag*>(h);
      void* d = nullptr;
      if (cudaHostGetDevicePointer(&d, h, 0) == cudaSuccess) ctx->diag_dev = static_cast<Diag*>(d);
      else cudaGetLastError();
    } else {
      cudaGetLastError();
    }
  }
  for (auto& e : ctx->ev_ring) {
    cudaError_t r = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    if (r != cudaSuccess) { cudaGetLastError(); return bail(fail(ctx, B2D_ERR_CUDA, "cudaEventCreate failed: %s", cudaGetErrorString(r))); }
  }
  preload_kernels();
  if (world == 1) ctx->finalized = true;
  *out = ctx;
  return B2D_OK;
}

int b2d_ctx_export(b2d_ctx* ctx, void* handle_buf, size_t* len) {
  if (ctx == nullptr || handle_buf == nullptr || len == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  if (*len < sizeof(HandleBlob)) return fail(ctx, B2D_ERR_INVALID, "handle buffer too small: %zu < %zu", *len, sizeof(HandleBlob));
  DeviceGuard guard(ctx->device);
  HandleBlob b;
  memset(&b, 0, sizeof(b));
  b.magic = kMagic; b.version = B2D_VERSION;
  b.rank = ctx->rank; b.world = ctx->world; b.device = ctx->device; b.mem_kind = ctx->mem_kind;
  b.pid = static_cast<int64_t>(getpid());
  b.proc_nonce = process_nonce();
  b.arena_bytes = ctx->arena_bytes;
  b.arena_ptr = reinterpret_cast<uint64_t>(ctx->arena);
  b.vmm_handle = static_cast<uint64_t>(ctx->vmm_handle);
  b.fd = -1;
  if (ctx->mem_kind == 0) B2D_CUDA(ctx, cudaIpcGetMemHandle(&b.ipc, ctx->arena));
  memcpy(handle_buf, &b, sizeof(b));
  *len = sizeof(b);
  return B2D_OK;
}

int b2d_ctx_export_fd(b2d_ctx* ctx, int* fd_out) {
  if (ctx == nullptr || fd_out == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  if (ctx->mem_kind != 1) return fail(ctx, B2D_ERR_STATE, "context was not created with B2D_FLAG_MEM_VMM");
  if (ctx->own_fd < 0) {
    int fd = -1;
    B2D_CU(ctx, g_drv.MemExportToShareableHandle(&fd, ctx->vmm_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    ctx->own_fd = fd;
  }
  *fd_out = ctx->own_fd;
  return B2D_OK;
}

int b2d_handle_set_fd(void* handle_buf, size_t len, int fd) {
  if (handle_buf == nullptr || len < sizeof(HandleBlob)) return fail(nullptr, B2D_ERR_INVALID, "bad handle buffer");
  HandleBlob* b = static_cast<HandleBlob*>(handle_buf);
  if (b->magic != kMagic) return fail(nullptr, B2D_ERR_INVALID, "not a b2d handle");
  b->fd = fd;
  return B2D_OK;
}

int b2d_ctx_import(b2d_ctx* ctx, int peer, const void* handle_buf, size_t len) {
  if (ctx == nullptr || handle_buf == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  if (len < sizeof(HandleBlob)) return fail(ctx, B2D_ERR_INVALID, "handle too short");
  if (peer < 0 || peer >= ctx->world || peer == ctx->rank) return fail(ctx, B2D_ERR_INVALID, "bad peer %d", peer);
  if (ctx->peer_map[peer] != kMapNone) return fail(ctx, B2D_ERR_STATE, "peer %d already imported", peer);
  HandleBlob b;
  memcpy(&b, handle_buf, sizeof(b));
  if (b.magic != kMagic || b.version != B2D_VERSION) return fail(ctx, B2D_ERR_INVALID, "handle magic/version mismatch");
  if (b.rank != peer || b.world != ctx->world) return fail(ctx, B2D_ERR_INVALID, "handle is from rank %d/%d, expected %d/%d", b.rank, b.world, peer, ctx->world);
  if (b.arena_bytes != ctx->arena_bytes) return fail(ctx, B2D_ERR_INVALID, "peer arena is %llu bytes, ours %zu: arenas must be symmetric", (unsigned long long)b.arena_bytes, ctx->arena_bytes);
  if (b.mem_kind != ctx->mem_kind) return fail(ctx, B2D_ERR_INVALID, "peer memory kind differs");
  DeviceGuard guard(ctx->device);
  unsigned char* mapped = nullptr;
  if (b.pid == static_cast<int64_t>(getpid()) && b.proc_nonce == process_nonce()) {
    // another rank of this very process (loopback ranks / single-process multi-GPU)
    mapped = reinterpret_cast<unsigned char*>(b.arena_ptr);
    if (b.device != ctx->device) {
      if (ctx->mem_kind == 1) {
        CUmemAccessDesc desc{};
        desc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        desc.location.id = ctx->device;
        desc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
        B2D_CU(ctx, g_drv.MemSetAccess(reinterpret_cast<CUdeviceptr>(mapped), b.arena_bytes, &desc, 1));
      } else {
        int can = 0;
        B2D_CUDA(ctx, cudaDeviceCanAccessPeer(&can, ctx->device, b.device));
        if (!can) return fail(ctx, B2D_ERR_PEER, "device %d cannot access device %d", ctx->device, b.device);
        cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
          cudaGetLastError();
          return fail(ctx, B2D_ERR_PEER, "cudaDeviceEnablePeerAccess(%d) failed: %s", b.device, cudaGetErrorString(e));
        }
        cudaGetLastError();
      }
    }
    ctx->peer_map[peer] = kMapDirect;
  } else if (ctx->mem_kind == 1) {
    if (b.fd < 0) return fail(ctx, B2D_ERR_INVALID, "VMM handle of peer %d carries no fd (pass it with SCM_RIGHTS, then b2d_handle_set_fd)", peer);
    CUmemGenericAllocationHandle h = 0;
    B2D_CU(ctx, g_drv.MemImportFromShareableHandle(&h, reinterpret_cast<void*>(static_cast<uintptr_t>(b.fd)), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    int rc = vmm_map(ctx, h, b.arena_bytes, ctx->device, &mapped);
    if (rc != B2D_OK) { g_drv.MemRelease(h); return rc; }
    ctx->peer_vmm[peer] = h;
    ctx->peer_map[peer] = kMapVmm;
  } else {
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, b.ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(ctx, B2D_ERR_PEER, "cudaIpcOpenMemHandle(peer %d) failed: %s", peer, cudaGetErrorString(e));
    }
    mapped = static_cast<unsigned char*>(p);
    ctx->peer_map[peer] = kMapLegacyIpc;
  }
  ctx->peers.arena[peer] = mapped;
  ctx->peers.signal[peer] = reinterpret_cast<Signal*>(mapped);
  return B2D_OK;
}

int b2d_ctx_finalize(b2d_ctx* ctx) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  for (int r = 0; r < ctx->world; ++r)
    if (ctx->peer_map[r] == kMapNone) return fail(ctx, B2D_ERR_STATE, "peer %d has not been imported", r);
  ctx->finalized = true;
  return B2D_OK;
}

// ---- NVLS -------------------------------------------------------------------------------
int b2d_mc_supported(b2d_ctx* ctx, int* supported) {
  if (ctx == nullptr || supported == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  *supported = 0;
  if (ctx->mem_kind != 1 || !driver_ready() || g_drv.MulticastCreate == nullptr) return B2D_OK;
  CUdevice dev;
  if (g_drv.DeviceGet(&dev, ctx->device) != CUDA_SUCCESS) return B2D_OK;
  int v = 0;
  if (g_drv.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) == CUDA_SUCCESS) *supported = v;
  return B2D_OK;
}

int b2d_mc_create(b2d_ctx* ctx, int* fd_out) {
  if (ctx == nullptr || fd_out == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  int sup = 0;
  b2d_mc_supported(ctx, &sup);
  if (!sup) return fail(ctx, B2D_ERR_UNSUPPORTED, "multicast not supported (needs B2D_FLAG_MEM_VMM and an NVSwitch fabric)");
  DeviceGuard guard(ctx->device);
  CUmulticastObjectProp mp{};
  mp.numDevices = ctx->world;
  mp.size = ctx->arena_bytes;
  mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUmemGenericAllocationHandle mc = 0;
  CUresult r = g_drv.MulticastCreate(&mc, &mp);
  if (r != CUDA_SUCCESS) return fail(ctx, B2D_ERR_UNSUPPORTED, "cuMulticastCreate failed: %s", cu_err(r));
  int fd = -1;
  r = g_drv.MemExportToShareableHandle(&fd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
  if (r != CUDA_SUCCESS) { g_drv.MemRelease(mc); return fail(ctx, B2D_ERR_CUDA, "multicast export failed: %s", cu_err(r)); }
  ctx->mc_handle = mc;
  ctx->mc_size = ctx->arena_bytes;
  *fd_out = fd;
  return B2D_OK;
}

int b2d_mc_join(b2d_ctx* ctx, int fd) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (ctx->mem_kind != 1 || !driver_ready() || g_drv.MulticastCreate == nullptr) return fail(ctx, B2D_ERR_UNSUPPORTED, "multicast unavailable");
  DeviceGuard guard(ctx->device);
  if (ctx->mc_handle == 0) {
    CUmemGenericAllocationHandle mc = 0;
    B2D_CU(ctx, g_drv.MemImportFromShareableHandle(&mc, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    ctx->mc_handle = mc;
    ctx->mc_size = ctx->arena_bytes;
  }
  CUdevice dev;
  B2D_CU(ctx, g_drv.DeviceGet(&dev, ctx->device));
  B2D_CU(ctx, g_drv.MulticastAddDevice(ctx->mc_handle, dev));
  ctx->mc_joined = true;
  return B2D_OK;
}

int b2d_mc_bind(b2d_ctx* ctx) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (!ctx->mc_joined) return fail(ctx, B2D_ERR_STATE, "b2d_mc_join() first");
  DeviceGuard guard(ctx->device);
  B2D_CU(ctx, g_drv.MulticastBindMem(ctx->mc_handle, 0, ctx->vmm_handle, 0, ctx->arena_bytes, 0));
  unsigned char* va = nullptr;
  int rc = vmm_map(ctx, ctx->mc_handle, ctx->arena_bytes, ctx->device, &va);
  if (rc != B2D_OK) return rc;
  ctx->peers.mc_arena = va;
  ctx->mc_bound = true;
  return B2D_OK;
}

int b2d_ctx_destroy(b2d_ctx* ctx) {
  if (ctx == nullptr) return B2D_OK;
  {
    DeviceGuard guard(ctx->device);
    cudaDeviceSynchronize();
    cudaGetLastError();
    for (auto& pr : ctx->ev_pending) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    for (auto& pr : ctx->ev_free) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    for (auto& pr : ctx->exch_pending) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    for (auto& kv : ctx->owner_buckets) free_tables(kv.second);
    for (auto& kv : ctx->optim_buckets) free_tables(kv.second);
    for (auto& e : ctx->ev_ring) if (e != nullptr) cudaEventDestroy(e);
    if (ctx->last_unstage_ev != nullptr) cudaEventDestroy(ctx->last_unstage_ev);
    for (auto& kv : ctx->slots) for (cudaEvent_t e : kv.second.reuse_ev) if (e != nullptr) cudaEventDestroy(e);
    for (cudaStream_t st : {ctx->s_stage, ctx->s_xfer, ctx->s_unstage}) if (st != nullptr) cudaStreamDestroy(st);
    if (ctx->peers.mc_arena != nullptr) vmm_unmap(ctx->peers.mc_arena, ctx->arena_bytes);
    if (ctx->mc_handle != 0) {
      if (ctx->mc_bound) {
        CUdevice dev;
        if (g_drv.DeviceGet(&dev, ctx->device) == CUDA_SUCCESS) g_drv.MulticastUnbind(ctx->mc_handle, dev, 0, ctx->arena_bytes);
      }
      g_drv.MemRelease(ctx->mc_handle);
    }
    for (int r = 0; r < ctx->world; ++r) {
      if (ctx->peer_map[r] == kMapLegacyIpc) cudaIpcCloseMemHandle(ctx->peers.arena[r]);
      if (ctx->peer_map[r] == kMapVmm) { vmm_unmap(ctx->peers.arena[r], ctx->arena_bytes); g_drv.MemRelease(ctx->peer_vmm[r]); }
    }
    if (ctx->arena != nullptr) {
      if (ctx->mem_kind == 1) { vmm_unmap(ctx->arena, ctx->arena_bytes); }
      else cudaFree(ctx->arena);
    }
    if (ctx->vmm_handle != 0) g_drv.MemRelease(ctx->vmm_handle);
    if (ctx->own_fd >= 0) close(ctx->own_fd);
    if (ctx->diag_host != nullptr) cudaFreeHost(ctx->diag_host);
    if (ctx->trace_dev != nullptr) cudaFree(ctx->trace_dev);
    cudaGetLastError();
  }
  delete ctx;
  return B2D_OK;
}

// ---- knobs -------------------------------------------------------------------------------
int b2d_ctx_set_timeout(b2d_ctx* ctx, unsigned timeout_ms) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  ctx->timeout_ms = timeout_ms;
  return B2D_OK;
}
int b2d_ctx_set_max_ctas(b2d_ctx* ctx, int max_ctas) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (max_ctas < 1 || max_ctas > B2D_MAX_BLOCKS) return fail(ctx, B2D_ERR_INVALID, "max_ctas must be in [1, %d]", B2D_MAX_BLOCKS);
  ctx->max_ctas = max_ctas;
  ctx->tma_ctas = max_ctas < 48 ? max_ctas : (ctx->tma_ctas_user > 0 ? ctx->tma_ctas_user : 48);
  return B2D_OK;
}
int b2d_ctx_set_tma_ctas(b2d_ctx* ctx, int ctas) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (ctas < 1 || ctas > B2D_MAX_BLOCKS) return fail(ctx, B2D_ERR_INVALID, "tma ctas must be in [1, %d]", B2D_MAX_BLOCKS);
  ctx->tma_ctas = ctas; ctx->tma_ctas_user = ctas;
  return B2D_OK;
}
int b2d_ctx_set_one_shot_max_bytes(b2d_ctx* ctx, size_t wire_bytes) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  ctx->one_shot_max_bytes = wire_bytes;
  ctx->one_shot_max_user = true;
  return B2D_OK;
}

int b2d_ctx_set_chunk_bytes(b2d_ctx* ctx, size_t wire_bytes) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (wire_bytes < (64u << 10)) return fail(ctx, B2D_ERR_INVALID, "chunk must be at least 64 KiB of wire payload");
  ctx->chunk_bytes = wire_bytes;
  return B2D_OK;
}
int b2d_ctx_set_exch_ctas(b2d_ctx* ctx, int ctas) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (ctas < 1 || ctas > B2D_MAX_BLOCKS) return fail(ctx, B2D_ERR_INVALID, "exchange ctas must be in [1, %d]", B2D_MAX_BLOCKS);
  ctx->exch_ctas = ctas;
  return B2D_OK;
}
int b2d_ctx_set_auto_profile(b2d_ctx* ctx, int profile) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (profile != B2D_PROFILE_OVERLAP && profile != B2D_PROFILE_LATENCY) return fail(ctx, B2D_ERR_INVALID, "bad profile %d", profile);
  ctx->auto_profile = profile;
  return B2D_OK;
}
int b2d_ctx_set_inplace(b2d_ctx* ctx, int enable) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  ctx->inplace = enable ? 1 : 0;
  return B2D_OK;
}
int b2d_ctx_set_nvls_auto(b2d_ctx* ctx, int enable) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  ctx->nvls_auto = enable ? 1 : 0;
  return B2D_OK;
}

int b2d_ctx_trace(b2d_ctx* ctx, int enable, double* phase_us, int* n_phases) {
  Entry en(ctx, false);
  if (en.rc != B2D_OK) return en.rc;
  int rc = en.use_device();
  if (rc != B2D_OK) return rc;
  if (enable && ctx->trace_dev == nullptr) {
    void* p = nullptr;
    B2D_CUDA(ctx, cudaMalloc(&p, sizeof(unsigned long long) * B2D_MAX_BLOCKS * kTraceSlots));
    B2D_CUDA(ctx, cudaMemset(p, 0, sizeof(unsigned long long) * B2D_MAX_BLOCKS * kTraceSlots));
    ctx->trace_dev = static_cast<unsigned long long*>(p);
  }
  if (phase_us != nullptr && n_phases != nullptr) {
    *n_phases = 0;
    if (ctx->trace_dev != nullptr && ctx->trace_grid > 0) {
      B2D_CUDA(ctx, cudaDeviceSynchronize());
      std::vector<unsigned long long> h(static_cast<size_t>(ctx->trace_grid) * kTraceSlots);
      B2D_CUDA(ctx, cudaMemcpy(h.data(), ctx->trace_dev, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      // phase k = mean over blocks of stamp[k+1] - stamp[k]; slot kTraceSlots-1 reports max(end) - min(start)
      unsigned long long t0 = ~0ull, t1 = 0;
      int used = 0;
      for (int k = 0; k + 1 < kTraceSlots; ++k) {
        double sum = 0; int cnt = 0;
        for (int b = 0; b < ctx->trace_grid; ++b) {
          const unsigned long long a = h[static_cast<size_t>(b) * kTraceSlots + k], e = h[static_cast<size_t>(b) * kTraceSlots + k + 1];
          if (a != 0 && e != 0 && e >= a) { sum += static_cast<double>(e - a); cnt++; t0 = a < t0 ? a : t0; t1 = e > t1 ? e : t1; }
        }
        if (cnt == 0) break;
        phase_us[k] = sum / cnt / 1e3;
        used = k + 1;
      }
      phase_us[used] = t1 > t0 ? static_cast<double>(t1 - t0) / 1e3 : 0.0;
      *n_phases = used + 1;
      B2D_CUDA(ctx, cudaMemset(ctx->trace_dev, 0, sizeof(unsigned long long) * B2D_MAX_BLOCKS * kTraceSlots));
    }
  }
  if (!enable && ctx->trace_dev != nullptr) { cudaFree(ctx->trace_dev); ctx->trace_dev = nullptr; }
  return B2D_OK;
}

int b2d_plan(b2d_ctx* ctx, size_t n, int wire, int algo, int* algo_out, int* grid_out, int* block_out) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  if (wire != B2D_WIRE_FP32 && wire != B2D_WIRE_BF16) return fail(ctx, B2D_ERR_INVALID, "bad wire %d", wire);
  const int a = pick_algo(ctx, n, wire, algo);
  int grid;
  if (ctx->world == 1) {
    grid = clamp_grid(n / 4, static_cast<size_t>(kThreads) * 4, static_cast<size_t>(ctx->sm_count) * 4);
  } else {
    grid = pick_grid(ctx, n, wire, a);
  }
  if (algo_out) *algo_out = a;
  if (grid_out) *grid_out = grid;
  if (block_out) *block_out = kThreads;
  return B2D_OK;
}

// ---- data path ---------------------------------------------------------------------------
int b2d_allreduce_bucket_phased(b2d_ctx* ctx, int bucket_idx, float* grad, size_t n, int wire, float scale,
                                int algo, unsigned phases, void* wait_stream, void* comm_stream) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (grad == nullptr && n != 0) return fail(ctx, B2D_ERR_INVALID, "grad is NULL");
  if (reinterpret_cast<uintptr_t>(grad) % 16 != 0) return fail(ctx, B2D_ERR_INVALID, "bucket buffer must be 16-byte aligned");
  if (wire != B2D_WIRE_FP32 && wire != B2D_WIRE_BF16) return fail(ctx, B2D_ERR_INVALID, "bad wire %d", wire);
  if (algo < B2D_ALGO_AUTO || algo > B2D_ALGO_NVLS_FUSED) return fail(ctx, B2D_ERR_INVALID, "bad algo %d", algo);
  if ((algo == B2D_ALGO_NVLS || algo == B2D_ALGO_NVLS_FUSED) && !ctx->mc_bound && ctx->world > 1)
    return fail(ctx, B2D_ERR_UNSUPPORTED, "NVLS requested but no multicast object is bound");
  if (phases == 0 || phases > 7u) return fail(ctx, B2D_ERR_INVALID, "bad phase mask %u", phases);
  if (n == 0) return B2D_OK;  // empty bucket: nothing to exchange, and every rank agrees on that
  int rc = en.use_device();
  if (rc != B2D_OK) return rc;
  cudaStream_t comm = static_cast<cudaStream_t>(comm_stream);

  int a = 0, grid = 0;
  b2d_plan(ctx, n, wire, algo, &a, &grid, nullptr);

  if (ctx->world > 1 && is_staged(a))
    return launch_staged(ctx, bucket_idx, grad, n, wire, scale, a, phases, static_cast<cudaStream_t>(wait_stream), comm);
  if (phases != 7u) return fail(ctx, B2D_ERR_INVALID, "only the staged algorithms can be issued phase by phase");

  const bool bf = wire == B2D_WIRE_BF16;
  if (ctx->world == 1)
    return launch_timed(ctx, wait_stream, comm_stream, 0, select_k0(bf), grid, kThreads, 0, grad, n, scale);

  const size_t epp = wire == B2D_WIRE_BF16 ? 8 : 4;
  const size_t npacks = (n + epp - 1) / epp;
  const size_t slice = (npacks + ctx->world - 1) / ctx->world;
  const size_t half = slice * ctx->world * 16;
  size_t stage_off = 0;
  rc = get_slot(ctx, bucket_idx, half, n, wire, a, grid, comm, &stage_off);
  if (rc != B2D_OK) return rc;

  ArParams P{};
  set_peer_wait(ctx, &P);
  P.grad = grad; P.n = n; P.stage_off = stage_off; P.scale = scale;
  P.trace = ctx->trace_dev;
  ctx->trace_grid = grid;
  // the remaining algorithms: B2D_ALGO_ONE_SHOT, B2D_ALGO_TWO_SHOT, B2D_ALGO_NVLS_FUSED, B2D_ALGO_TWO_SHOT_TMA
  if (a == B2D_ALGO_TWO_SHOT_TMA)
    return launch_timed(ctx, wait_stream, comm_stream, a, select_k2t(ctx->world), grid, kTmaThreads, kTmaSmemBytes, P,
                        tma_mt(slice, grid));
  if (a == B2D_ALGO_ONE_SHOT)
    return launch_timed(ctx, wait_stream, comm_stream, a, select_k1(ctx->world, bf), grid, kThreads, 0, P);
  return launch_timed(ctx, wait_stream, comm_stream, a, select_k2(ctx->world, bf, a == B2D_ALGO_NVLS_FUSED), grid, kThreads,
                      0, P);
}

int b2d_allreduce_bucket(b2d_ctx* ctx, int bucket_idx, float* grad, size_t n, int wire, float scale,
                         int algo, void* wait_stream, void* comm_stream) {
  return b2d_allreduce_bucket_phased(ctx, bucket_idx, grad, n, wire, scale, algo, 7u, wait_stream, comm_stream);
}

static int sharded_common(b2d_ctx* ctx, int slot, const float* grads, float* params, float* exp_avg,
                          float* exp_avg_sq, float* rs_out, size_t n, const int64_t* shard_off, int wire,
                          float scale, const b2d_adam64* adam, int do_sr, int do_gather, int end_barrier,
                          void* wait_stream, void* comm_stream) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (shard_off == nullptr) return fail(ctx, B2D_ERR_INVALID, "shard_off is NULL");
  if (wire != B2D_WIRE_FP32 && wire != B2D_WIRE_BF16) return fail(ctx, B2D_ERR_INVALID, "bad wire %d", wire);
  size_t max_len = 0;
  int rc = check_shard_off(ctx, shard_off, n, &max_len);
  if (rc != B2D_OK) return rc;
  if (n == 0) return B2D_OK;
  rc = en.use_device();
  if (rc != B2D_OK) return rc;
  cudaStream_t comm = static_cast<cudaStream_t>(comm_stream);

  ShParams P{};
  P.grads = grads; P.params = params; P.exp_avg = exp_avg; P.exp_avg_sq = exp_avg_sq; P.rs_out = rs_out;
  P.n = n; P.scale = scale;
  P.do_stage_reduce = do_sr; P.do_adam = adam != nullptr; P.do_gather = do_gather; P.end_barrier = end_barrier;
  for (int r = 0; r <= ctx->world; ++r) P.off[r] = shard_off[r];
  for (int r = ctx->world + 1; r <= B2D_MAX_WORLD; ++r) P.off[r] = shard_off[ctx->world];
  set_peer_wait(ctx, &P);

  if (do_gather) {
    const unsigned char* p8 = reinterpret_cast<const unsigned char*>(params);
    if (p8 < ctx->arena || p8 + n * 4 > ctx->arena + ctx->arena_bytes)
      return fail(ctx, B2D_ERR_INVALID, "the flat parameter buffer must live in the symmetric arena (b2d_arena_alloc)");
    P.param_off = static_cast<size_t>(p8 - ctx->arena);
  }
  if (do_sr) {
    if (grads == nullptr || reinterpret_cast<uintptr_t>(grads) % 16 != 0) return fail(ctx, B2D_ERR_INVALID, "grads must be a 16-byte aligned device pointer");
    if (adam != nullptr) {
      if (params == nullptr || exp_avg == nullptr || exp_avg_sq == nullptr) return fail(ctx, B2D_ERR_INVALID, "params/exp_avg/exp_avg_sq are NULL");
      if (adam->step < 1) return fail(ctx, B2D_ERR_INVALID, "adam.step must be >= 1");
      P.adam = adam_consts(*adam);
      if (adam->zero_grads) P.grads_rw = const_cast<float*>(grads);
    } else if (rs_out == nullptr) {
      return fail(ctx, B2D_ERR_INVALID, "reduce-scatter output is NULL");
    }
    const size_t half = n * (wire == B2D_WIRE_BF16 ? 2 : 4);
    const int grid = clamp_grid(max_len / (wire == B2D_WIRE_BF16 ? 8 : 4), kThreads, ctx->max_ctas);
    size_t stage_off = 0;
    rc = get_slot(ctx, 0x40000000 + slot, half, n, wire, 100 + do_gather, grid, comm, &stage_off);
    if (rc != B2D_OK) return rc;
    P.stage_off = stage_off;
    return launch_timed(ctx, wait_stream, comm_stream, 10, select_k456(ctx->world, wire == B2D_WIRE_BF16), grid, kThreads,
                        0, P);
  }
  // all-gather only
  const int grid = clamp_grid(max_len / 4, kThreads, ctx->max_ctas);
  return launch_timed(ctx, wait_stream, comm_stream, 11, select_k456(ctx->world, false), grid, kThreads, 0, P);
}

int b2d_sharded_step64(b2d_ctx* ctx, int slot, const float* grads, float* params, float* exp_avg,
                       float* exp_avg_sq, size_t n, const int64_t* shard_off, int wire, float scale,
                       const b2d_adam64* adam, void* wait_stream, void* comm_stream) {
  if (adam == nullptr) return fail(ctx, B2D_ERR_INVALID, "adam is NULL");
  return sharded_common(ctx, slot, grads, params, exp_avg, exp_avg_sq, nullptr, n, shard_off, wire, scale, adam,
                        1, 1, 0, wait_stream, comm_stream);
}

int b2d_sharded_step(b2d_ctx* ctx, int slot, const float* grads, float* params, float* exp_avg,
                     float* exp_avg_sq, size_t n, const int64_t* shard_off, int wire, float scale,
                     const b2d_adam* adam, void* wait_stream, void* comm_stream) {
  if (adam == nullptr) return fail(ctx, B2D_ERR_INVALID, "adam is NULL");
  const b2d_adam64 a = adam64(*adam);
  return b2d_sharded_step64(ctx, slot, grads, params, exp_avg, exp_avg_sq, n, shard_off, wire, scale, &a, wait_stream,
                            comm_stream);
}

int b2d_reduce_scatter(b2d_ctx* ctx, int slot, const float* grads, float* out, size_t n,
                       const int64_t* shard_off, int wire, float scale, void* wait_stream, void* comm_stream) {
  return sharded_common(ctx, slot, grads, nullptr, nullptr, nullptr, out, n, shard_off, wire, scale, nullptr,
                        1, 0, 0, wait_stream, comm_stream);
}

int b2d_allgather(b2d_ctx* ctx, float* buf, size_t n, const int64_t* shard_off, void* wait_stream, void* comm_stream) {
  return sharded_common(ctx, 0, nullptr, buf, nullptr, nullptr, nullptr, n, shard_off, B2D_WIRE_FP32, 1.f, nullptr,
                        0, 1, 1, wait_stream, comm_stream);
}

// ---- sharded path on the staged machinery (b2d_owner.cuh) ----------------------------------------------------
int b2d_bucket_register(b2d_ctx* ctx, int bucket_id, const b2d_seg* segs, int nseg, int wire) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (segs == nullptr || nseg < 1) return fail(ctx, B2D_ERR_INVALID, "a reduce bucket needs at least one segment");
  if (wire != B2D_WIRE_FP32 && wire != B2D_WIRE_BF16) return fail(ctx, B2D_ERR_INVALID, "bad wire %d", wire);
  OwnerTable t;
  const std::string bad = build_owner_table(segs, nseg, ctx->world, wire, &t);
  if (!bad.empty()) return fail(ctx, B2D_ERR_INVALID, "%s", bad.c_str());
  int rc = en.use_device();
  if (rc == B2D_OK) rc = drop_bucket(ctx, ctx->owner_buckets, bucket_id);
  if (rc != B2D_OK) return rc;
  b2d_ctx::OwnerBucket nb;
  nb.nseg = static_cast<int>(t.flat_off.size()); nb.wire = wire;
  std::copy(t.owner_pack, t.owner_pack + B2D_MAX_WORLD + 1, nb.owner_pack);
  rc = upload_table(ctx, t.flat_off, &nb.d_flat_off);
  if (rc == B2D_OK) rc = upload_table(ctx, t.start, &nb.d_start);
  if (rc != B2D_OK) return rc;
  ctx->owner_buckets[bucket_id] = nb;
  return B2D_OK;
}

int b2d_reduce_to_owner(b2d_ctx* ctx, int bucket_id, float* grads, float* reduced, const int64_t* shard_off, float scale,
                        unsigned flags, unsigned phases, void* wait_stream, void* comm_stream) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  auto it = ctx->owner_buckets.find(bucket_id);
  if (it == ctx->owner_buckets.end()) return fail(ctx, B2D_ERR_STATE, "reduce bucket %d has not been registered", bucket_id);
  if (grads == nullptr || reduced == nullptr || shard_off == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  if ((phases & 3u) == 0 || phases > 3u) return fail(ctx, B2D_ERR_INVALID, "bad phase mask %u (bit 0 stage, bit 1 reduce)", phases);
  const bool nvls = (flags & B2D_RTO_NVLS) != 0;
  if (nvls && !ctx->mc_bound) return fail(ctx, B2D_ERR_UNSUPPORTED, "NVLS requested but no multicast object is bound");
  b2d_ctx::OwnerBucket& ob = it->second;
  int rc = en.use_device();
  if (rc == B2D_OK) rc = ensure_streams(ctx);
  if (rc != B2D_OK) return rc;
  cudaStream_t comm = static_cast<cudaStream_t>(comm_stream);
  const bool bf16 = ob.wire == B2D_WIRE_BF16;
  const size_t total = ob.owner_pack[ctx->world];
  size_t stage_off = 0;
  Slot* slot = nullptr;
  rc = get_slot(ctx, 0x20000000 + bucket_id, total * 16 * 2, total, ob.wire, 200, 0, comm, &stage_off, &slot, nullptr, true);
  if (rc != B2D_OK) return rc;
  if (phases & 1u) ob.op_epoch = ++ctx->epoch;
  if (ob.op_epoch == 0) return fail(ctx, B2D_ERR_STATE, "reduce phase issued before the stage phase of bucket %d", bucket_id);

  SegParams P{};
  P.seg_flat_off = ob.d_flat_off; P.seg_start = ob.d_start; P.nseg = ob.nseg;
  for (int r = 0; r <= B2D_MAX_WORLD; ++r) P.owner_pack[r] = ob.owner_pack[r];
  P.grads = grads; P.reduced = reduced; P.shard_lo = shard_off[ctx->rank]; P.wire_off = stage_off; P.scale = scale;
  P.zero_grads = (flags & B2D_RTO_ZERO_GRADS) ? 1 : 0; P.accumulate = (flags & B2D_RTO_ACCUMULATE) ? 1 : 0;
  P.epoch = ob.op_epoch;
  set_peer_wait(ctx, &P);
  cudaEvent_t es = nullptr;
  if (phases & 1u) {
    rc = join(ctx, ctx->s_stage, static_cast<cudaStream_t>(wait_stream));
    if (rc != B2D_OK) return rc;
    launch(ctx, select_seg_stage(bf16), stream_grid(ctx, total), kStThreads, 0, ctx->s_stage, P);
    es = next_event(ctx);
    B2D_CUDA(ctx, cudaEventRecord(es, ctx->s_stage));
  }
  if (phases & 2u) {
    if (es != nullptr) B2D_CUDA(ctx, cudaStreamWaitEvent(ctx->s_xfer, es, 0));
    const size_t mine = ob.owner_pack[ctx->rank + 1] - ob.owner_pack[ctx->rank];
    const size_t per_thread = nvls ? 8 : (kMaxLoadsInFlight / ctx->world > 1 ? kMaxLoadsInFlight / ctx->world : 1);
    const int grid = clamp_grid(mine, kExThreads * per_thread, ctx->exch_ctas);
    TimedSpan span(ctx, ctx->exch_pending);
    if ((rc = span.start(ctx->s_xfer)) != B2D_OK) return rc;
    launch(ctx, select_seg_reduce(ctx->world, bf16, nvls), grid, kExThreads, 0, ctx->s_xfer, P);
    ctx->exch_launches += 1;
    if ((rc = span.stop(ctx->s_xfer)) != B2D_OK || (rc = join(ctx, comm, ctx->s_xfer)) != B2D_OK) return rc;
    ctx->last_grid = grid;
    ob.op_epoch = 0;
  }
  rc = launch_result(ctx);
  if (rc != B2D_OK) return rc;
  ctx->last_algo = 12; ctx->last_block = kExThreads;
  return B2D_OK;
}

// b2d_adam_push (grad_scale == NULL: K13) and b2d_adam_push_scaled (K13 with the gradients scaled on the device)
static int adam_push(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                     const int64_t* shard_off, const b2d_adam_group64* groups, int ngroups, unsigned flags, unsigned phases,
                     void* wait_stream, void* comm_stream, const float* grad_scale) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (params == nullptr || shard_off == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  if (ngroups < 0 || ngroups > kMaxAdamGroups) return fail(ctx, B2D_ERR_INVALID, "at most %d parameter groups", kMaxAdamGroups);
  if (ngroups > 0 && (groups == nullptr || exp_avg == nullptr || exp_avg_sq == nullptr || reduced == nullptr))
    return fail(ctx, B2D_ERR_INVALID, "groups / exp_avg / exp_avg_sq / reduced are NULL");
  if ((phases & 6u) == 0 || (phases & ~6u) != 0) return fail(ctx, B2D_ERR_INVALID, "bad phase mask %u (bit 1 step + push, bit 2 wait)", phases);
  size_t max_len = 0;
  int rc = check_shard_off(ctx, shard_off, n, &max_len);
  if (rc != B2D_OK) return rc;
  const bool nvls = (flags & B2D_RTO_NVLS) != 0;
  if (nvls && !ctx->mc_bound) return fail(ctx, B2D_ERR_UNSUPPORTED, "NVLS requested but no multicast object is bound");
  const unsigned char* p8 = reinterpret_cast<const unsigned char*>(params);
  if (p8 < ctx->arena || p8 + n * 4 > ctx->arena + ctx->arena_bytes)
    return fail(ctx, B2D_ERR_INVALID, "the flat parameter buffer must live in the symmetric arena (b2d_arena_alloc)");
  if (n == 0) return B2D_OK;
  rc = en.use_device();
  if (rc == B2D_OK) rc = ensure_streams(ctx);
  if (rc != B2D_OK) return rc;
  cudaStream_t comm = static_cast<cudaStream_t>(comm_stream);
  if (phases & 2u) ctx->push_epoch = ++ctx->epoch;
  if (ctx->push_epoch == 0) return fail(ctx, B2D_ERR_STATE, "wait phase issued before the push phase");
  if (phases & 2u) {
    PushParams P{};
    P.params = params; P.param_off = static_cast<size_t>(p8 - ctx->arena);
    P.exp_avg = exp_avg; P.exp_avg_sq = exp_avg_sq; P.reduced = reduced;
    P.lo = shard_off[ctx->rank]; P.hi = shard_off[ctx->rank + 1];
    P.ngroups = ngroups;
    for (int k = 0; k < ngroups; ++k) {
      if (groups[k].lo < 0 || groups[k].hi < groups[k].lo || groups[k].hi > P.hi - P.lo || groups[k].lo % 4 != 0 || groups[k].hi % 4 != 0)
        return fail(ctx, B2D_ERR_INVALID, "parameter group %d covers [%lld, %lld) of a shard of %lld elements", k, (long long)groups[k].lo, (long long)groups[k].hi, (long long)(P.hi - P.lo));
      if (groups[k].adam.step < 1) return fail(ctx, B2D_ERR_INVALID, "adam.step must be >= 1");
      P.group_lo[k] = groups[k].lo; P.group_hi[k] = groups[k].hi;
      P.group[k] = adam_consts(groups[k].adam);
    }
    P.rank = ctx->rank; P.world = ctx->world; P.epoch = ctx->push_epoch; P.peers = ctx->peers;
    P.grad_scale = grad_scale;
    rc = join(ctx, ctx->s_xfer, static_cast<cudaStream_t>(wait_stream));
    if (rc != B2D_OK) return rc;
    // the step is not overlapped with anything and moves 28 B of local HBM traffic per owned element: one full wave
    // (3 CTAs of 256 threads x 68 registers per SM on sm_90a); a 128-CTA grid leaves most warp slots idle
    const int grid = clamp_grid(static_cast<size_t>(P.hi - P.lo) / 4, kExThreads * 2, static_cast<size_t>(ctx->sm_count) * 3);
    TimedSpan span(ctx, ctx->ev_pending);
    if ((rc = span.start(ctx->s_xfer)) != B2D_OK) return rc;
    launch(ctx, select_adam_push(ctx->world, nvls, grad_scale != nullptr), grid, kExThreads, 0, ctx->s_xfer, P);
    if ((rc = span.stop(ctx->s_xfer)) != B2D_OK) return rc;
    ctx->last_grid = grid;
  }
  if (phases & 4u) {
    ExParams XP{};
    XP.epoch = ctx->push_epoch;
    set_peer_wait(ctx, &XP);
    rc = join(ctx, ctx->s_unstage, ctx->s_xfer);
    if (rc != B2D_OK) return rc;
    launch(ctx, wait_published_kernel, 1, 32, 0, ctx->s_unstage, XP);
    rc = join_unstage(ctx, comm);
    if (rc != B2D_OK) return rc;
    ctx->push_epoch = 0;
  }
  rc = launch_result(ctx);
  if (rc != B2D_OK) return rc;
  ctx->last_algo = 13; ctx->last_block = kExThreads;
  return B2D_OK;
}

// The fp32 groups of b2d_adam_push, widened; more than kMaxAdamGroups are refused by adam_push itself.
static std::vector<b2d_adam_group64> groups64(const b2d_adam_group* groups, int ngroups) {
  std::vector<b2d_adam_group64> g(groups != nullptr && ngroups > 0 ? ngroups : 0);
  for (size_t k = 0; k < g.size(); ++k) g[k] = b2d_adam_group64{groups[k].lo, groups[k].hi, adam64(groups[k].adam)};
  return g;
}

int b2d_adam_push64(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                    const int64_t* shard_off, const b2d_adam_group64* groups, int ngroups, unsigned flags, unsigned phases,
                    void* wait_stream, void* comm_stream) {
  return adam_push(ctx, params, exp_avg, exp_avg_sq, reduced, n, shard_off, groups, ngroups, flags, phases, wait_stream,
                   comm_stream, nullptr);
}

int b2d_adam_push_scaled64(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                           const int64_t* shard_off, const b2d_adam_group64* groups, int ngroups, unsigned flags,
                           unsigned phases, void* wait_stream, void* comm_stream, const float* grad_scale) {
  if (grad_scale == nullptr) return fail(ctx, B2D_ERR_INVALID, "grad_scale is NULL");
  return adam_push(ctx, params, exp_avg, exp_avg_sq, reduced, n, shard_off, groups, ngroups, flags, phases, wait_stream,
                   comm_stream, grad_scale);
}

int b2d_adam_push(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                  const int64_t* shard_off, const b2d_adam_group* groups, int ngroups, unsigned flags, unsigned phases,
                  void* wait_stream, void* comm_stream) {
  const std::vector<b2d_adam_group64> g = groups64(groups, ngroups);
  return adam_push(ctx, params, exp_avg, exp_avg_sq, reduced, n, shard_off, groups == nullptr ? nullptr : g.data(), ngroups,
                   flags, phases, wait_stream, comm_stream, nullptr);
}

int b2d_adam_push_scaled(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                         const int64_t* shard_off, const b2d_adam_group* groups, int ngroups, unsigned flags, unsigned phases,
                         void* wait_stream, void* comm_stream, const float* grad_scale) {
  if (grad_scale == nullptr) return fail(ctx, B2D_ERR_INVALID, "grad_scale is NULL");
  const std::vector<b2d_adam_group64> g = groups64(groups, ngroups);
  return adam_push(ctx, params, exp_avg, exp_avg_sq, reduced, n, shard_off, groups == nullptr ? nullptr : g.data(), ngroups,
                   flags, phases, wait_stream, comm_stream, grad_scale);
}

// ---- gradient clipping (b2d_clip.cuh) ------------------------------------------------------------------------------
static_assert(kClipGMax <= static_cast<unsigned>(kClipThreads), "K18's final tree combines at most kClipThreads block sums");

int b2d_clip_register(b2d_ctx* ctx, size_t* offset) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->clip_registered) {
    const size_t bytes = round_up(2 * static_cast<size_t>(ctx->world) * kClipSlotBytes + kClipGMax * sizeof(double), kAlign);
    size_t off = 0;
    if (!slot_region_alloc(ctx, bytes, &off))
      return fail(ctx, B2D_ERR_NOMEM, "symmetric arena exhausted: the clip region needs %zu bytes, %zu free of %zu", bytes,
                  ctx->user_bottom - ctx->slot_top, ctx->arena_bytes);
    ctx->clip_off = off;
    ctx->clip_registered = true;
  }
  if (offset != nullptr) *offset = ctx->clip_off;
  return B2D_OK;
}

int b2d_clip_norm(b2d_ctx* ctx, const float* x, size_t n, float max_norm, float* norm_out, float* coef_out, unsigned phases,
                  void* wait_stream, void* comm_stream) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (!ctx->clip_registered) return fail(ctx, B2D_ERR_STATE, "b2d_clip_norm before b2d_clip_register");
  if ((phases & 3u) == 0 || phases > 3u) return fail(ctx, B2D_ERR_INVALID, "bad phase mask %u (bit 0 partial, bit 1 coefficient)", phases);
  if (!(max_norm >= 0.f) || !isfinite(max_norm)) return fail(ctx, B2D_ERR_INVALID, "max_norm must be finite and >= 0 (got %g)", static_cast<double>(max_norm));
  if ((phases & 1u) && n > 0 && x == nullptr) return fail(ctx, B2D_ERR_INVALID, "x is NULL");
  if ((phases & 2u) && (norm_out == nullptr || coef_out == nullptr)) return fail(ctx, B2D_ERR_INVALID, "NULL output");
  if ((phases & 1u) && ctx->clip_op_epoch != 0) return fail(ctx, B2D_ERR_STATE, "clip partial issued again before the previous one was combined");
  if (!(phases & 1u) && ctx->clip_op_epoch == 0) return fail(ctx, B2D_ERR_STATE, "clip coefficient issued before the partial");
  int rc = en.use_device();
  if (rc == B2D_OK) rc = ensure_streams(ctx);
  if (rc != B2D_OK) return rc;
  // on s_xfer, behind the reduce buckets (K12) that wrote the shard
  const size_t gen_bytes = static_cast<size_t>(ctx->world) * kClipSlotBytes;
  if (phases & 1u) {
    rc = join(ctx, ctx->s_xfer, static_cast<cudaStream_t>(wait_stream));
    if (rc != B2D_OK) return rc;
    ctx->clip_gen = ctx->clip_calls++ & 1u;
    ctx->clip_op_epoch = ++ctx->clip_epoch;
    ClipPartialParams P{};
    P.x = x; P.n = n; P.vec = (reinterpret_cast<uintptr_t>(x) % 16) == 0;
    P.block_sums = reinterpret_cast<double*>(ctx->arena + ctx->clip_off + 2 * gen_bytes);
    P.region_off = ctx->clip_off + ctx->clip_gen * gen_bytes;
    P.rank = ctx->rank; P.world = ctx->world; P.epoch = ctx->clip_op_epoch; P.peers = ctx->peers;
    launch(ctx, sqnorm_partial_kernel, static_cast<int>(clip_grid(n, kClipGMax)), kClipThreads, 0, ctx->s_xfer, P);
  }
  if (phases & 2u) {
    ClipCoefParams P{};
    P.region_off = ctx->clip_off + ctx->clip_gen * gen_bytes;
    P.max_norm = max_norm; P.norm_out = norm_out; P.coef_out = coef_out;
    set_peer_wait(ctx, &P);
    P.epoch = ctx->clip_op_epoch;
    launch(ctx, clip_coef_kernel, 1, 32, 0, ctx->s_xfer, P);
    rc = join(ctx, static_cast<cudaStream_t>(comm_stream), ctx->s_xfer);
    if (rc != B2D_OK) return rc;
    ctx->clip_op_epoch = 0;
  }
  return launch_result(ctx);
}

// ---- optimizer in backward (f-2) ----------------------------------------------------------------------------------
int b2d_optim_register(b2d_ctx* ctx, int bucket_id, float* const* params, float* const* state1, float* const* state2,
                       const int64_t* bucket_off, const int64_t* numel, int nparam) {
  Entry en(ctx, false);
  if (en.rc != B2D_OK) return en.rc;
  if (params == nullptr || bucket_off == nullptr || numel == nullptr || nparam < 1) return fail(ctx, B2D_ERR_INVALID, "bad parameter table");
  std::vector<float*> ptr(3 * static_cast<size_t>(nparam), nullptr);
  std::vector<unsigned> start(nparam + 1);
  long long cur = 0;
  for (int i = 0; i < nparam; ++i) {
    if (bucket_off[i] != cur || numel[i] <= 0 || params[i] == nullptr)
      return fail(ctx, B2D_ERR_INVALID, "parameters must tile the bucket in order (parameter %d at %lld, expected %lld)", i, (long long)bucket_off[i], cur);
    ptr[i] = params[i]; start[i] = static_cast<unsigned>(cur);
    if (state1 != nullptr) ptr[nparam + i] = state1[i];
    if (state2 != nullptr) ptr[2 * nparam + i] = state2[i];
    cur += numel[i];
    if (cur > 0xffffffffll) return fail(ctx, B2D_ERR_INVALID, "bucket too large");
  }
  start[nparam] = static_cast<unsigned>(cur);
  int rc = en.use_device();
  if (rc == B2D_OK) rc = drop_bucket(ctx, ctx->optim_buckets, bucket_id);
  if (rc != B2D_OK) return rc;
  b2d_ctx::OptimBucket ob;
  ob.nseg = nparam; ob.n = static_cast<size_t>(cur);
  rc = upload_table(ctx, ptr, &ob.d_ptr);
  if (rc == B2D_OK) rc = upload_table(ctx, start, &ob.d_start);
  if (rc != B2D_OK) return rc;
  ctx->optim_buckets[bucket_id] = ob;
  return B2D_OK;
}

int b2d_bucket_optim(b2d_ctx* ctx, int bucket_id, const float* grads, size_t n, int kind, const b2d_adam* hp, float momentum,
                     void* stream) {
  if (hp == nullptr) return b2d_bucket_optim64(ctx, bucket_id, grads, n, kind, nullptr, momentum, stream);
  const b2d_adam64 a = adam64(*hp);
  return b2d_bucket_optim64(ctx, bucket_id, grads, n, kind, &a, momentum, stream);
}

int b2d_bucket_optim64(b2d_ctx* ctx, int bucket_id, const float* grads, size_t n, int kind, const b2d_adam64* hp,
                       float momentum, void* stream) {
  Entry en(ctx, false);
  if (en.rc != B2D_OK) return en.rc;
  auto it = ctx->optim_buckets.find(bucket_id);
  if (it == ctx->optim_buckets.end()) return fail(ctx, B2D_ERR_STATE, "bucket %d has no parameter table (b2d_optim_register)", bucket_id);
  if (it->second.n != n) return fail(ctx, B2D_ERR_INVALID, "bucket %d has %zu elements, its parameter table covers %zu", bucket_id, n, it->second.n);
  if (grads == nullptr || hp == nullptr || (kind != 0 && kind != 1)) return fail(ctx, B2D_ERR_INVALID, "bad argument");
  if (kind == 1 && hp->step < 1) return fail(ctx, B2D_ERR_INVALID, "Adam needs step >= 1");
  const int rc = en.use_device();
  if (rc != B2D_OK) return rc;
  OptimParams P{};
  P.param_ptr = it->second.d_ptr; P.seg_start = it->second.d_start; P.nseg = it->second.nseg;
  P.state1_ptr = it->second.d_ptr + it->second.nseg; P.state2_ptr = it->second.d_ptr + 2 * it->second.nseg;
  P.grads = grads; P.n = n; P.kind = kind;
  P.lr = static_cast<float>(hp->lr); P.momentum = momentum; P.weight_decay = static_cast<float>(hp->weight_decay);
  P.first_step = hp->step <= 1;
  if (kind == 1) P.adam = adam_consts(*hp);
  const int grid = clamp_grid(n, kStThreads * 4, static_cast<size_t>(ctx->sm_count) * 2);
  launch(ctx, bucket_optim_kernel, grid, kStThreads, 0, static_cast<cudaStream_t>(stream), P);
  return launch_result(ctx);
}

int b2d_barrier(b2d_ctx* ctx, void* stream) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (ctx->world == 1) return B2D_OK;
  const int rc = en.use_device();
  return rc != B2D_OK ? rc : launch_barrier(ctx, static_cast<cudaStream_t>(stream));
}

// ---- synchronised BatchNorm (b2d_syncbn.cuh) -----------------------------------------------
int b2d_bn_register(b2d_ctx* ctx, int layer_id, int channels, size_t* offset) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (channels < 1) return fail(ctx, B2D_ERR_INVALID, "a BatchNorm layer needs at least one channel (got %d)", channels);
  auto it = ctx->bn_layers.find(layer_id);
  if (it != ctx->bn_layers.end()) {
    if (it->second.channels != channels)
      return fail(ctx, B2D_ERR_INVALID, "BatchNorm layer %d is registered with %d channels, not %d", layer_id, it->second.channels, channels);
  } else {
    const size_t W = static_cast<size_t>(ctx->world);
    const size_t bytes = round_up(2 * W * (bn_fwd_row(channels) + bn_bwd_row(channels)) * 4, kAlign);
    size_t off = 0;
    if (!slot_region_alloc(ctx, bytes, &off))
      return fail(ctx, B2D_ERR_NOMEM, "symmetric arena exhausted: BatchNorm layer %d needs %zu bytes, %zu free of %zu", layer_id,
                  bytes, ctx->user_bottom - ctx->slot_top, ctx->arena_bytes);
    b2d_ctx::BnLayer L;
    L.channels = channels;
    L.off = off;
    it = ctx->bn_layers.emplace(layer_id, L).first;
  }
  if (offset != nullptr) *offset = it->second.off;
  return B2D_OK;
}

// One BN exchange: K15 (phase bit 0) and K16 / K17 (bit 1) on `stream`.  a / b: this rank's two halves of the row.
static int bn_exchange(b2d_ctx* ctx, int layer_id, bool fwd, const float* a, const float* b, float count, float eps,
                       float momentum, float* out_a, float* out_b, int32_t* counts, float* running_mean, float* running_var,
                       unsigned phases, void* stream) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  auto it = ctx->bn_layers.find(layer_id);
  if (it == ctx->bn_layers.end()) return fail(ctx, B2D_ERR_STATE, "BatchNorm layer %d has not been registered", layer_id);
  if ((phases & 3u) == 0 || phases > 3u) return fail(ctx, B2D_ERR_INVALID, "bad phase mask %u (bit 0 push, bit 1 combine)", phases);
  if ((phases & 1u) && fwd && !(count >= 0.f)) return fail(ctx, B2D_ERR_INVALID, "count must be >= 0");
  if ((phases & 1u) && fwd && count > 0.f && (a == nullptr || b == nullptr))
    return fail(ctx, B2D_ERR_INVALID, "a rank with count > 0 must pass its mean and invstd");
  if ((phases & 2u) && (out_a == nullptr || out_b == nullptr || (fwd && counts == nullptr)))
    return fail(ctx, B2D_ERR_INVALID, "NULL output");
  b2d_ctx::BnLayer& L = it->second;
  const int d = fwd ? 0 : 1;
  if ((phases & 1u) && L.op_epoch[d] != 0)
    return fail(ctx, B2D_ERR_STATE, "BatchNorm layer %d: push issued again before the previous exchange was combined", layer_id);
  if (!(phases & 1u) && L.op_epoch[d] == 0)
    return fail(ctx, B2D_ERR_STATE, "BatchNorm layer %d: combine issued before the push", layer_id);
  const int rc = en.use_device();
  if (rc != B2D_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int C = L.channels;
  const size_t W = static_cast<size_t>(ctx->world);
  const size_t gen_bytes = W * (fwd ? bn_fwd_row(C) : bn_bwd_row(C)) * 4;
  const size_t base = L.off + (fwd ? 0 : 2 * W * bn_fwd_row(C) * 4);
  if (phases & 1u) {
    L.op_gen[d] = L.calls[d]++ & 1u;
    L.op_epoch[d] = ++ctx->bn_epoch;
    BnPushParams P{};
    P.a = a; P.b = b; P.count = fwd ? count : 0.f; P.channels = C; P.fwd = fwd ? 1 : 0;
    P.region_off = base + L.op_gen[d] * gen_bytes;
    P.rank = ctx->rank; P.world = ctx->world; P.epoch = L.op_epoch[d]; P.peers = ctx->peers;
    launch(ctx, bn_push_kernel, 1, kBnThreads, 0, st, P);
  }
  if (phases & 2u) {
    BnCombineParams P{};
    P.region_off = base + L.op_gen[d] * gen_bytes;
    P.channels = C; P.eps = eps; P.momentum = momentum;
    P.out_a = out_a; P.out_b = out_b; P.counts = counts;
    P.running_mean = fwd ? running_mean : nullptr; P.running_var = fwd ? running_var : nullptr;
    set_peer_wait(ctx, &P);
    P.epoch = L.op_epoch[d];
    const int grid = clamp_grid(static_cast<size_t>(C), kBnThreads, static_cast<size_t>(ctx->sm_count));
    launch(ctx, select_bn_combine(fwd), grid, kBnThreads, 0, st, P);
    L.op_epoch[d] = 0;
  }
  return launch_result(ctx);
}

int b2d_bn_stats_exchange(b2d_ctx* ctx, int layer_id, const float* mean, const float* invstd, float count, float eps,
                          float momentum, float* mean_out, float* invstd_out, int32_t* counts_out, float* running_mean,
                          float* running_var, unsigned phases, void* stream) {
  return bn_exchange(ctx, layer_id, true, mean, invstd, count, eps, momentum, mean_out, invstd_out, counts_out, running_mean,
                     running_var, phases, stream);
}

int b2d_bn_grad_exchange(b2d_ctx* ctx, int layer_id, const float* sum_dy, const float* sum_dy_xmu, float* sum_dy_out,
                         float* sum_dy_xmu_out, unsigned phases, void* stream) {
  return bn_exchange(ctx, layer_id, false, sum_dy, sum_dy_xmu, 0.f, 0.f, 0.f, sum_dy_out, sum_dy_xmu_out, nullptr, nullptr,
                     nullptr, phases, stream);
}

// ---- arena -------------------------------------------------------------------------------
int b2d_arena_alloc(b2d_ctx* ctx, size_t bytes, void** dev_ptr, size_t* offset) {
  if (ctx == nullptr || dev_ptr == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  bytes = round_up(bytes, kAlign);
  if (bytes > ctx->user_bottom || ctx->user_bottom - bytes < ctx->slot_top)
    return fail(ctx, B2D_ERR_NOMEM, "symmetric arena exhausted: %zu bytes requested, %zu free", bytes, ctx->user_bottom - ctx->slot_top);
  ctx->user_bottom -= bytes;
  *dev_ptr = ctx->arena + ctx->user_bottom;
  if (offset) *offset = ctx->user_bottom;
  return B2D_OK;
}

int b2d_arena_reset(b2d_ctx* ctx) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (auto& kv : ctx->slots) for (cudaEvent_t e : kv.second.reuse_ev) if (e != nullptr) cudaEventDestroy(e);
  ctx->slots.clear();
  ctx->bn_layers.clear();
  ctx->clip_registered = false;
  ctx->clip_op_epoch = 0;
  ctx->slot_free.clear();
  ctx->slot_top = kSignalBytes;
  ctx->user_bottom = ctx->arena_bytes;
  return B2D_OK;
}

// ---- link probe ----------------------------------------------------------------------------
int b2d_peer_bw(b2d_ctx* ctx, int peer, size_t bytes, int iters, int mode, double* gbps) {
  Entry en(ctx, true);
  if (en.rc != B2D_OK) return en.rc;
  if (gbps == nullptr || peer < 0 || peer >= ctx->world) return fail(ctx, B2D_ERR_INVALID, "bad peer/gbps");
  if (iters < 1) iters = 1;
  const int rc = en.use_device();
  if (rc != B2D_OK) return rc;
  bytes = bytes / 16 * 16;
  if (bytes == 0 || kSignalBytes + bytes > ctx->arena_bytes) return fail(ctx, B2D_ERR_INVALID, "probe size must fit the arena");
  void* dst = nullptr;
  B2D_CUDA(ctx, cudaMalloc(&dst, bytes));
  const unsigned char* src = ctx->peers.arena[peer] + kSignalBytes;   // content is irrelevant
  cudaStream_t st = nullptr;
  cudaEvent_t a = nullptr, b = nullptr;
  cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&a);
  if (e == cudaSuccess) e = cudaEventCreate(&b);
  float ms = 0.f;
  if (e == cudaSuccess) {
    for (int i = -2; i < iters && e == cudaSuccess; ++i) {
      if (i == 0) e = cudaEventRecord(a, st);
      if (e != cudaSuccess) break;
      if (mode == 0) e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
      else { peer_read_kernel<<<64, kExThreads, 0, st>>>(reinterpret_cast<const uint4*>(src), static_cast<uint4*>(dst), bytes / 16); e = cudaGetLastError(); }
    }
    if (e == cudaSuccess) e = cudaEventRecord(b, st);
    if (e == cudaSuccess) e = cudaEventSynchronize(b);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, a, b);
  }
  if (a) cudaEventDestroy(a);
  if (b) cudaEventDestroy(b);
  if (st) cudaStreamDestroy(st);
  cudaFree(dst);
  if (e != cudaSuccess) { cudaGetLastError(); return fail(ctx, B2D_ERR_CUDA, "link probe failed: %s", cudaGetErrorString(e)); }
  *gbps = static_cast<double>(bytes) * iters / (static_cast<double>(ms) * 1e6);
  return B2D_OK;
}

// ---- the arena as a torch memory pool (SURVEY §8 f-1) ---------------------------------------
// torch.cuda.memory.CUDAPluggableAllocator(libb2d.so, "b2d_pool_alloc", "b2d_pool_free") + torch.cuda.MemPool:
// whatever torch allocates while that pool is active (DDP's flat bucket tensors, reducer.hpp:347-406) comes
// out of the bound context's symmetric arena, so peers can reach it and the fp32 exchange runs in place.
static std::mutex g_pool_mu;
static b2d_ctx* g_pool_ctx = nullptr;

int b2d_pool_bind(b2d_ctx* ctx) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  g_pool_ctx = ctx;
  return B2D_OK;
}

// Allocations the arena could not take (exhausted, or no context bound): ordinary device memory, so torch sees no
// out-of-memory.  A bucket that ends up there is simply not exchanged in place (the hook stages it like any tensor).
static std::map<void*, size_t> g_pool_plain;

void* b2d_pool_alloc(size_t size, int device, void* stream) {
  (void)stream;
  b2d_ctx* ctx;
  { std::lock_guard<std::mutex> lk(g_pool_mu); ctx = g_pool_ctx; }
  void* p = nullptr;
  size_t off = ~static_cast<size_t>(0);
  if (ctx != nullptr && ctx->device == device && b2d_arena_alloc(ctx, size, &p, &off) != B2D_OK) p = nullptr;
  if (p == nullptr) {
    int prev = -1;
    cudaGetDevice(&prev);
    if (prev != device) cudaSetDevice(device);
    if (cudaMalloc(&p, size) != cudaSuccess) { cudaGetLastError(); p = nullptr; }
    if (prev >= 0 && prev != device) cudaSetDevice(prev);
    if (p == nullptr) return nullptr;
    std::lock_guard<std::mutex> lk(g_pool_mu);
    g_pool_plain[p] = size;
    off = ~static_cast<size_t>(0);
  }
  if (ctx != nullptr) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->pool_allocs += 1;
    for (uint64_t v : {static_cast<uint64_t>(off), static_cast<uint64_t>(size)})
      for (int i = 0; i < 8; ++i) { ctx->pool_digest ^= (v >> (8 * i)) & 0xffu; ctx->pool_digest *= 1099511628211ull; }
  }
  return p;
}

void b2d_pool_free(void* ptr, size_t size, int device, void* stream) {
  (void)size; (void)device; (void)stream;
  {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    auto it = g_pool_plain.find(ptr);
    if (it == g_pool_plain.end()) return;   // arena memory lives as long as its context (bump-allocated)
    g_pool_plain.erase(it);
  }
  cudaFree(ptr);
}

// ---- introspection -----------------------------------------------------------------------
int b2d_ctx_stats(b2d_ctx* ctx, b2d_stats* out) {
  if (ctx == nullptr || out == nullptr) return fail(ctx, B2D_ERR_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  {
    DeviceGuard guard(ctx->device);
    resolve_timing(ctx, false);
  }
  memset(out, 0, sizeof(*out));
  out->exch_launches = ctx->exch_launches; out->exch_timed = ctx->exch_timed; out->exch_ms = ctx->exch_ms;
  out->pool_allocs = ctx->pool_allocs; out->pool_digest = ctx->pool_digest;
  out->launches = ctx->launches;
  out->timed_launches = ctx->timed_launches;
  out->timed_ms = ctx->timed_ms;
  out->arena_bytes = ctx->arena_bytes;
  out->arena_used = (ctx->slot_top) + (ctx->arena_bytes - ctx->user_bottom);
  out->world = ctx->world; out->rank = ctx->rank; out->device = ctx->device; out->sm_count = ctx->sm_count;
  out->mem_kind = ctx->mem_kind; out->mc_bound = ctx->mc_bound ? 1 : 0;
  out->last_algo = ctx->last_algo; out->last_grid = ctx->last_grid; out->last_block = ctx->last_block;
  return B2D_OK;
}

int b2d_ctx_reset_stats(b2d_ctx* ctx) {
  if (ctx == nullptr) return fail(nullptr, B2D_ERR_INVALID, "ctx is NULL");
  std::lock_guard<std::mutex> lk(ctx->mu);
  {
    DeviceGuard guard(ctx->device);
    resolve_timing(ctx, true);
  }
  ctx->launches = 0; ctx->timed_launches = 0; ctx->timed_ms = 0.0;
  ctx->exch_launches = 0; ctx->exch_timed = 0; ctx->exch_ms = 0.0;
  return B2D_OK;
}

}  // extern "C"
