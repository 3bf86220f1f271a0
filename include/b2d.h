/*
 * b2d.h — C ABI of libb2d: the H100-native (sm_90a) DDP gradient-sync data path.
 *
 * This is the drop-in boundary of the repo (DESIGN.md §2, SURVEY.md §8b).  The
 * library replaces, for one 8xH100 NVSwitch box, the collectives that the
 * reference's strategies reach through torch DDP / FairScale:
 *
 *   reference seam                                   replaced by
 *   ------------------------------------------------ ---------------------------
 *   ray_lightning/ray_ddp.py:112-116  (**ddp_kwargs  b2d_allreduce_bucket()
 *     -> DistributedDataParallel -> c10d::Reducer      (one call per DDP bucket,
 *     -> ncclAllReduce per bucket; with                 fp32->bf16 cast, 1/W scale,
 *     bf16_compress_hook: cast, div, allreduce, copy)    P2P reduce, fp32 write-back
 *                                                       fused in ONE kernel)
 *   ray_lightning/ray_ddp.py:192-196  (process group  b2d_ctx_create/export/import
 *     init; peers become addressable)                   /finalize (peer mapping)
 *   ray_lightning/ray_ddp_sharded.py:12-13            b2d_sharded_step()
 *     (FairScale ShardedDataParallel reduce-to-owner    (reduce-scatter to owner +
 *      + OSS.step + OSS._broadcast_params)               partitioned Adam + param
 *                                                       all-gather, one kernel),
 *                                                     b2d_reduce_scatter(),
 *                                                     b2d_allgather()
 *   ray_lightning/launchers/ray_launcher.py:177-219   (precondition: every worker
 *     (_share_cuda_visible_devices)                    sees every GPU of its node)
 *
 * Conventions
 *   - plain C, no torch / pybind types; loadable with ctypes / cgo / JNI.
 *   - every entry point returns 0 on success, a negative b2d_status otherwise;
 *     never throws; b2d_last_error() gives the message (per ctx, or the
 *     thread-local creation error when ctx == NULL).
 *   - data-path entry points only ENQUEUE work on `comm_stream` (after making
 *     it wait for `wait_stream`); they never synchronise the device.
 *   - streams are passed as `void*` holding a cudaStream_t (0 = legacy default).
 *   - the caller owns every tensor pointer; the library owns the symmetric
 *     arena, the signal pads, the peer mappings and the multicast object.
 *   - all ranks of a job must issue the same sequence of data-path calls with
 *     the same sizes (DDP guarantees this for buckets: reducer.hpp:282,524).
 *   - a peer that never arrives makes the kernel trap after `timeout_ms`
 *     (b2d_ctx_set_timeout); the next CUDA call then returns a sticky error.
 */
#ifndef B2D_H_
#define B2D_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2D_VERSION 110          /* 0.1.10 */
#define B2D_MAX_WORLD 8          /* one NVSwitch domain: 8 x H100 */
#define B2D_MAX_BLOCKS 264       /* 2 x 132 SMs (H100 SXM) */
#define B2D_HANDLE_BYTES 256     /* size of the blob b2d_ctx_export() writes */

typedef struct b2d_ctx b2d_ctx;

typedef enum b2d_status {
  B2D_OK = 0,
  B2D_ERR_INVALID = -1,      /* bad argument */
  B2D_ERR_CUDA = -2,         /* a CUDA runtime/driver call failed */
  B2D_ERR_STATE = -3,        /* call made in the wrong phase (e.g. before finalize) */
  B2D_ERR_NOMEM = -4,        /* symmetric arena exhausted */
  B2D_ERR_UNSUPPORTED = -5,  /* feature not available on this box (e.g. multicast) */
  B2D_ERR_PEER = -6          /* peer mapping failed / peer timeout recorded */
} b2d_status;

/* wire formats of the exchange */
typedef enum b2d_wire {
  B2D_WIRE_FP32 = 0,  /* peers exchange fp32: matches DDP's default allreduce
                         (default_comm_hooks.hpp:36-51): out = sum_r g_r * scale */
  B2D_WIRE_BF16 = 1   /* peers exchange bf16: matches bf16_compress_hook
                         (default_hooks.py:57-93,116-134):
                         c_r = bf16(bf16(g_r) * scale); s = bf16(sum_r c_r); out = fp32(s) */
} b2d_wire;

typedef enum b2d_algo {
  B2D_ALGO_AUTO = 0,
  B2D_ALGO_ONE_SHOT = 1,   /* every rank reads every peer's whole staged bucket */
  B2D_ALGO_TWO_SHOT = 2,   /* reduce-scatter of 1/W slices + all-gather, both by peer reads */
  B2D_ALGO_NVLS = 3,       /* staged exchange, reduce + broadcast inside the NVSwitch
                              (multimem.ld_reduce / multimem.st); sums in switch order: tolerance contract */
  B2D_ALGO_TWO_SHOT_TMA = 4, /* two-shot with every load a TMA bulk copy into a shared-memory ring (bf16 wire,
                               n % 8 == 0; other shapes fall back to B2D_ALGO_TWO_SHOT) */
  B2D_ALGO_STAGED = 5,     /* staged exchange over peer loads/stores: stage | reduce own slice + push | write back
                              as separate short kernels on three streams, chunk-pipelined; rank-ordered fp32
                              sums, bit-identical to ONE_SHOT / TWO_SHOT */
  B2D_ALGO_NVLS_FUSED = 6  /* round-1 single-kernel NVLS two-shot (kept for A/B sweeps) */
} b2d_algo;

/* b2d_ctx_create flags */
#define B2D_FLAG_MEM_LEGACY_IPC 0x0u /* arena = cudaMalloc, shared by cudaIpc handles (default) */
#define B2D_FLAG_MEM_VMM        0x1u /* arena = cuMemCreate (POSIX fd handles); needed for NVLS */
#define B2D_FLAG_TIMING         0x2u /* record a CUDA-event pair around every kernel launch */

/* ---- lifecycle ------------------------------------------------------------------------- */

int b2d_version(void);

/* Replaces: the NCCL communicator bring-up hidden behind init_process_group("nccl") at
 * ray_lightning/ray_ddp.py:192-196 (the process group itself stays, as control plane).
 * Create the per-rank context on CUDA device `device` (index inside the process's
 * CUDA_VISIBLE_DEVICES, i.e. RayStrategy.root_device.index, ray_ddp.py:259-304) and
 * allocate its symmetric arena (`arena_bytes`, rounded up to 2 MiB) and signal pad.
 * Several contexts may live in one process (also on the same device: "loopback"
 * ranks used by the single-GPU tests). */
int b2d_ctx_create(int rank, int world, int device, size_t arena_bytes,
                   unsigned flags, b2d_ctx** out);

/* Replaces: NCCL's out-of-band ncclUniqueId / peer discovery, done for the reference inside
 * init_process_group (ray_ddp.py:192-196); needs every worker to see its node's GPUs, which
 * ray_lightning/launchers/ray_launcher.py:177-219 (_share_cuda_visible_devices) provides.
 * Write this rank's B2D_HANDLE_BYTES-byte handle blob.  The blob travels to the peers
 * over whatever control plane the host already has (torch.distributed
 * all_gather_object, the Ray object store, ...).  For B2D_FLAG_MEM_VMM contexts the
 * blob additionally names a POSIX file descriptor (b2d_ctx_export_fd) that the host
 * must pass with SCM_RIGHTS and patch in with b2d_handle_set_fd() on the receiver. */
int b2d_ctx_export(b2d_ctx* ctx, void* handle_buf, size_t* len);
int b2d_ctx_export_fd(b2d_ctx* ctx, int* fd_out);
int b2d_handle_set_fd(void* handle_buf, size_t len, int fd);

/* Map peer `peer`'s arena + signal pad into this process / device. */
int b2d_ctx_import(b2d_ctx* ctx, int peer, const void* handle_buf, size_t len);

/* After all world-1 imports: upload the peer pointer tables.  Host must run a
 * control-plane barrier between the last b2d_ctx_finalize() and the first data call. */
int b2d_ctx_finalize(b2d_ctx* ctx);

/* Replaces: NCCL's own NVLS set-up (no reference line: NCCL decides it internally).
 * NVLS (NVLink-SHARP multicast), optional: rank 0 creates the multicast object and
 * exports its fd; every rank (rank 0 included) joins with the fd, then — after a
 * control-plane barrier — binds its arena.  Returns B2D_ERR_UNSUPPORTED when the
 * device or driver does not expose multicast. */
int b2d_mc_supported(b2d_ctx* ctx, int* supported);
int b2d_mc_create(b2d_ctx* ctx, int* fd_out);
int b2d_mc_join(b2d_ctx* ctx, int fd);
int b2d_mc_bind(b2d_ctx* ctx);

int b2d_ctx_destroy(b2d_ctx* ctx);
const char* b2d_last_error(b2d_ctx* ctx);

/* ---- knobs ----------------------------------------------------------------------------- */

int b2d_ctx_set_timeout(b2d_ctx* ctx, unsigned timeout_ms);  /* peer-flag watchdog; default 600000 (10 min), 0 = never */
int b2d_ctx_set_max_ctas(b2d_ctx* ctx, int max_ctas);        /* CTAs per comm kernel; default 64 */
int b2d_ctx_set_tma_ctas(b2d_ctx* ctx, int ctas);            /* CTAs of the TMA-staged kernel; default 48 */
int b2d_ctx_set_one_shot_max_bytes(b2d_ctx* ctx, size_t wire_bytes); /* AUTO: one-shot at or below (default: 16 / 4 / 1 MiB at world 2 / 4 / 8) */
int b2d_ctx_set_chunk_bytes(b2d_ctx* ctx, size_t wire_bytes);  /* staged exchange: wire bytes per pipeline chunk; default 64 MiB */
int b2d_ctx_set_exch_ctas(b2d_ctx* ctx, int ctas);             /* CTAs (256 threads) of the exchange kernel; default 64 (NVLS: half) */
#define B2D_PROFILE_OVERLAP 0   /* AUTO assumes the exchange overlaps compute (the DDP hook): staged pipeline above the one-shot range */
#define B2D_PROFILE_LATENCY 1   /* AUTO assumes an isolated call: single-kernel algorithms up to ~100 MiB */
int b2d_ctx_set_auto_profile(b2d_ctx* ctx, int profile);       /* default B2D_PROFILE_OVERLAP */
int b2d_ctx_set_inplace(b2d_ctx* ctx, int enable);             /* exchange arena-resident fp32 buckets in place? default 1 */
int b2d_ctx_set_nvls_auto(b2d_ctx* ctx, int enable);           /* may AUTO pick B2D_ALGO_NVLS when multicast is bound? default 1 */

/* ---- data path ------------------------------------------------------------------------- */

/* Replaces: the per-bucket collective torch DDP issues for RayStrategy(**ddp_kwargs)
 * (ray_lightning/ray_ddp.py:75,112-116) — with B2D_WIRE_BF16 the whole bf16_compress_hook
 * (torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py:57-93,116-134: cast, div,
 * ncclAllReduce, copy_), with B2D_WIRE_FP32 the default divide + allreduce
 * (default_hooks.py:18-54, default_comm_hooks.hpp:36-51).  Called from the DDP comm hook
 * (torch/nn/parallel/distributed.py:1987-2067).
 * In-place allreduce of one DDP gradient bucket (K0/K1/K2/K2T/K3).
 *   grad_inout : this rank's flat fp32 bucket (GradBucket.buffer(), comm.hpp:20-98), n elements
 *   bucket_idx : GradBucket.index(); selects the arena slot (double-buffered, so no
 *                trailing barrier is needed between consecutive steps)
 *   scale      : 1/world for DDP averaging (applied before the wire cast)
 * world == 1 degenerates to the cast/scale round trip (K0) with no peer access. */
int b2d_allreduce_bucket(b2d_ctx* ctx, int bucket_idx, float* grad_inout, size_t n,
                         int wire, float scale, int algo,
                         void* wait_stream, void* comm_stream);

/* The same call issued phase by phase (bit 0: stage, bit 1: exchange, bit 2: wait + write back; 7 = all, which
 * is what b2d_allreduce_bucket does).  Only the staged algorithms (B2D_ALGO_STAGED / B2D_ALGO_NVLS, or AUTO
 * resolving to them) accept a partial mask.  For hosts that drive SEVERAL ranks from one thread (the loopback
 * tests, smoke() under a serialising profiler): issue phase 1 for every rank, then 2, then 4 — no kernel then
 * ever waits for a kernel launched after it.  Replaces nothing in the reference (NCCL has no such seam). */
int b2d_allreduce_bucket_phased(b2d_ctx* ctx, int bucket_idx, float* grad_inout, size_t n,
                                int wire, float scale, int algo, unsigned phases,
                                void* wait_stream, void* comm_stream);

/* Hyper-parameters of the partitioned Adam (torch/optim/adam.py semantics, non-amsgrad, non-maximize).  `step` is the
 * 1-based step count AFTER increment.  The values are fp32: the library derives the kernel constants from them as if
 * they were the Python floats, so a value that fp32 does not hold exactly (beta2 = 0.999) gives constants that differ
 * from torch's in the last bits.  b2d_adam64 and the *64 entry points carry the Python floats themselves. */
typedef struct b2d_adam {
  float lr, beta1, beta2, eps, weight_decay;
  int32_t step;
  int32_t adamw;      /* 0: L2 (grad += wd*p) like torch.optim.Adam; 1: decoupled like AdamW */
  int32_t zero_grads; /* 1: overwrite the local flat grads with 0 once they are staged */
} b2d_adam;

/* b2d_adam with the floating-point hyper-parameters as doubles: the Python floats themselves.  The library forms
 * `1 - beta2`, `beta ** step`, `lr / bias_correction1`, `bias_correction2 ** 0.5` and `1 - lr * weight_decay` from them
 * in double, as torch does, and casts each to fp32 once: the update is then bit-exact against torch.optim.Adam / AdamW
 * on CUDA (default foreach path). */
typedef struct b2d_adam64 {
  double lr, beta1, beta2, eps, weight_decay;
  int32_t step;
  int32_t adamw;
  int32_t zero_grads;
  int32_t pad_;
} b2d_adam64;

/* Replaces: what RayShardedStrategy (ray_lightning/ray_ddp_sharded.py:12-13) reaches through PL's
 * DDPSpawnShardedStrategy: FairScale ShardedDataParallel's reduce-to-owner of every gradient,
 * OSS.step() on the owned shard and OSS._broadcast_params() (torch analogue:
 * torch/distributed/optim/zero_redundancy_optimizer.py:759-825,1038-1142).
 * Sharded optimizer step (K4+K5+K6 fused): the flat fp32 gradient space [0, n) is cut
 * into `world` contiguous owner shards shard_off[r] .. shard_off[r+1] (element offsets,
 * world+1 entries, multiples of 8, parameter aligned — FairScale OSS.partition_parameters
 * ownership).  Rank r: reduces its shard from all peers (x scale), applies Adam to
 * params/exp_avg/exp_avg_sq of that shard, and every rank then gathers the updated
 * shards so that `params` is whole again.
 *   grads, params : flat fp32 [n]; `params` MUST live in the arena (b2d_arena_alloc)
 *   exp_avg, exp_avg_sq : fp32 [shard_off[rank+1]-shard_off[rank]], local */
int b2d_sharded_step(b2d_ctx* ctx, int slot, const float* grads, float* params,
                     float* exp_avg, float* exp_avg_sq, size_t n,
                     const int64_t* shard_off, int wire, float scale,
                     const b2d_adam* adam, void* wait_stream, void* comm_stream);
/* b2d_sharded_step with double hyper-parameters (b2d_adam64). */
int b2d_sharded_step64(b2d_ctx* ctx, int slot, const float* grads, float* params,
                       float* exp_avg, float* exp_avg_sq, size_t n,
                       const int64_t* shard_off, int wire, float scale,
                       const b2d_adam64* adam, void* wait_stream, void* comm_stream);

/* Replaces: FairScale's dist.reduce(grad, dst=owner) stream for optimizers other than Adam/AdamW.
 * K4 alone: out[0 .. len_r) = sum_r grads_r[shard_off[rank] ..) * scale  (fp32 out, local). */
int b2d_reduce_scatter(b2d_ctx* ctx, int slot, const float* grads, float* out, size_t n,
                       const int64_t* shard_off, int wire, float scale,
                       void* wait_stream, void* comm_stream);

/* Replaces: OSS._broadcast_params (one broadcast per owner) after a local optimizer step.
 * K6 alone: `buf` (flat fp32 [n], in the arena) holds this rank's valid shard; pull every
 * other shard from its owner. */
int b2d_allgather(b2d_ctx* ctx, float* buf, size_t n, const int64_t* shard_off,
                  void* wait_stream, void* comm_stream);

/* ---- sharded path, overlapped with backward (b2d_owner.cuh) -------------------------------- */

/* One run of the flat gradient space (8-element aligned) and the rank that owns it. */
typedef struct b2d_seg {
  int64_t flat_off, len;   /* elements; multiples of 8 */
  int32_t owner;
  int32_t pad_;
} b2d_seg;

#define B2D_RTO_ZERO_GRADS 0x1u  /* overwrite the local gradient segments with 0 once they are staged */
#define B2D_RTO_ACCUMULATE 0x2u  /* reduced += sum  (gradient accumulation over several backward passes) */
#define B2D_RTO_NVLS       0x4u  /* sum inside the NVSwitch (multimem.ld_reduce / multimem.st); needs a bound multicast object */

/* Replaces: FairScale ShardedDataParallel's bucket set-up (reduce_buffer_size grouping of parameters that become
 * ready together), reached through ray_lightning/ray_ddp_sharded.py:12.  Declare reduce bucket `bucket_id` as a set
 * of segments of the flat gradient space.  The library sorts them by owner, merges touching runs and keeps the
 * tables in device memory; the bucket's staging region (sum of lengths x wire width) is taken from the arena on
 * first use.  Same call, same arguments, on every rank. */
int b2d_bucket_register(b2d_ctx* ctx, int bucket_id, const b2d_seg* segs, int nseg, int wire);

/* Replaces: FairScale's per-bucket `grad *= 1/W; dist.reduce(bucket, dst=owner)` issued from the autograd hooks
 * while backward runs (ShardedDataParallel._get_reduce_fn, recalled; torch analogue: reduce_scatter of a
 * ZeroRedundancyOptimizer bucket).  Every rank stages its copy of the bucket's segments (cast + scale); every owner
 * then reads ITS segments from all ranks, adds them in rank order in fp32 and writes
 *     reduced[flat_off - shard_off[rank] ...]  (fp32, local, the owner's shard of the flat space).
 * `grads`: base of the flat fp32 gradient buffer.  Asynchronous on the library's internal streams after
 * `wait_stream`; `comm_stream` waits for the result.  phases: bit 0 stage, bit 1 reduce (3 = both). */
int b2d_reduce_to_owner(b2d_ctx* ctx, int bucket_id, float* grads, float* reduced, const int64_t* shard_off,
                        float scale, unsigned flags, unsigned phases, void* wait_stream, void* comm_stream);

/* One parameter group's Adam constants and the part of the OWN shard it covers (elements relative to shard start). */
typedef struct b2d_adam_group {
  int64_t lo, hi;
  b2d_adam adam;
  int32_t pad_;
} b2d_adam_group;
typedef struct b2d_adam_group64 {
  int64_t lo, hi;
  b2d_adam64 adam;
} b2d_adam_group64;

/* Replaces: OSS.step() on the owned shard + OSS._broadcast_params() (one broadcast per owner).  Applies Adam /
 * AdamW (torch/optim/adam.py:530-547 arithmetic) to the own shard using `reduced` — per parameter group — and
 * PUSHES the new fp32 parameters into every rank's flat parameter buffer (`params`, in the arena); when it has
 * completed in `comm_stream` order, every rank's parameters are whole.  ngroups == 0: push only (the caller's own
 * optimizer has updated the shard).  flags: B2D_RTO_NVLS.  phases: bit 1 step + push, bit 2 wait (6 = both). */
int b2d_adam_push(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                  const int64_t* shard_off, const b2d_adam_group* groups, int ngroups, unsigned flags,
                  unsigned phases, void* wait_stream, void* comm_stream);
/* b2d_adam_push with double hyper-parameters (b2d_adam_group64). */
int b2d_adam_push64(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                    const int64_t* shard_off, const b2d_adam_group64* groups, int ngroups, unsigned flags,
                    unsigned phases, void* wait_stream, void* comm_stream);

/* ---- optimizer step inside backward, per DDP bucket (f-2) ----------------------------------- */

/* Replaces: torch's `_hook_then_optimizer` (torch/distributed/algorithms/ddp_comm_hooks/optimizer_overlap_hooks.py:
 * 131-163), the optional overlapped-optimizer companion of the comm hook reached through
 * ray_lightning/ray_ddp.py:112-116 (ddp_comm_hook / ddp_comm_wrapper).  Declare which parameters (device pointers,
 * fp32) tile DDP bucket `bucket_id` (GradBucket.parameters() / gradients(): first bucket element and element count
 * of each, in bucket order), and where each parameter's optimizer state lives (one tensor per parameter, the caller's:
 * state1 = momentum buffer | exp_avg, state2 = exp_avg_sq; NULL arrays when the optimizer keeps none). */
int b2d_optim_register(b2d_ctx* ctx, int bucket_id, float* const* params, float* const* state1, float* const* state2,
                       const int64_t* bucket_off, const int64_t* numel, int nparam);

/* Apply one optimizer step to the bucket's parameters from its (already averaged) gradients `grads` on `stream`:
 * kind 0 = torch.optim.SGD (hp->lr, hp->weight_decay, `momentum`; dampening 0, no nesterov; at hp->step <= 1 the
 * momentum buffers are written with the gradient, as torch clones it, afterwards they are read), kind 1 =
 * torch.optim.Adam / AdamW (all of *hp).  Issue it behind b2d_allreduce_bucket on the
 * same comm stream. */
int b2d_bucket_optim(b2d_ctx* ctx, int bucket_id, const float* grads, size_t n, int kind, const b2d_adam* hp,
                     float momentum, void* stream);
/* b2d_bucket_optim with double hyper-parameters (b2d_adam64); `momentum` is cast to fp32 as torch casts it. */
int b2d_bucket_optim64(b2d_ctx* ctx, int bucket_id, const float* grads, size_t n, int kind, const b2d_adam64* hp,
                       float momentum, void* stream);

/* Replaces: nothing in the reference (dist.barrier is host side); device-side fence of this library.
 * All-ranks barrier enqueued on `stream` (also quiesces the arena before slots are re-laid out). */
int b2d_barrier(b2d_ctx* ctx, void* stream);

/* ---- synchronised BatchNorm (b2d_syncbn.cuh) ---------------------------------------------- */

/* Declare BatchNorm layer `layer_id` with `channels` channels: takes its exchange region (two generations of
 * W forward rows and two of W backward rows, about 32 x W x channels bytes) from the arena and writes the region's
 * arena offset to *offset (may be NULL).  Every rank must register the same layers in the same order, so that the
 * offsets agree; registering a layer again with the same channel count is a no-op.  Host only. */
int b2d_bn_register(b2d_ctx* ctx, int layer_id, int channels, size_t* offset);

/* Replaces: torch.nn.SyncBatchNorm's forward statistics exchange (torch/nn/modules/_functions.py:65-115: cat,
 * all_gather_into_tensor, the host-side mask of empty ranks, batch_norm_gather_stats_with_counts).
 * mean / invstd: this rank's batch_norm_stats (fp32 [C]); count: its elements per channel.  A rank with count == 0
 * passes NULL mean / invstd and pushes a zero row.  Writes the statistics of the whole batch over every rank with
 * count > 0 (rank-ordered merge, fp32) to mean_out / invstd_out (fp32 [C]), every rank's count to counts_out
 * (int32 [W], zeros kept) and, when non-NULL, updates running_mean / running_var (fp32 [C]) in place with
 * `momentum` and the unbiased variance.  Enqueued on `stream`; no host synchronisation.
 * phases: bit 0 push, bit 1 wait + combine (3 = both); hosts that drive several ranks from one thread issue bit 0 for
 * every rank, then bit 1. */
int b2d_bn_stats_exchange(b2d_ctx* ctx, int layer_id, const float* mean, const float* invstd, float count,
                          float eps, float momentum, float* mean_out, float* invstd_out, int32_t* counts_out,
                          float* running_mean, float* running_var, unsigned phases, void* stream);

/* Replaces: torch.nn.SyncBatchNorm's backward exchange (torch/nn/modules/_functions.py:155-165: cat, all_reduce
 * SUM, split).  sum_dy / sum_dy_xmu: this rank's batch_norm_backward_reduce outputs (fp32 [C]; NULL: zeros).
 * Writes their rank-ordered fp32 sums over every rank to sum_dy_out / sum_dy_xmu_out.  phases as above. */
int b2d_bn_grad_exchange(b2d_ctx* ctx, int layer_id, const float* sum_dy, const float* sum_dy_xmu,
                         float* sum_dy_out, float* sum_dy_xmu_out, unsigned phases, void* stream);

/* Replaces: the gradient multiply of OSS.clip_grad_norm / torch.nn.utils.clip_grad_norm_ (`grad.mul_(clip_coef)`, a
 * separate pass over the gradients).  b2d_adam_push with every gradient of the own shard multiplied by *grad_scale
 * (device fp32, non-NULL; one rounding) before the Adam update: the coefficient b2d_clip_norm wrote, read on the
 * device, so the step needs no host synchronisation. */
int b2d_adam_push_scaled(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced, size_t n,
                         const int64_t* shard_off, const b2d_adam_group* groups, int ngroups, unsigned flags,
                         unsigned phases, void* wait_stream, void* comm_stream, const float* grad_scale);
/* b2d_adam_push_scaled with double hyper-parameters (b2d_adam_group64). */
int b2d_adam_push_scaled64(b2d_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, const float* reduced,
                           size_t n, const int64_t* shard_off, const b2d_adam_group64* groups, int ngroups,
                           unsigned flags, unsigned phases, void* wait_stream, void* comm_stream,
                           const float* grad_scale);

/* ---- gradient clipping (b2d_clip.cuh) ------------------------------------------------------ */

/* Takes the clip exchange's region (two generations of W slots plus the per-block partials, a few KiB) from the arena
 * and writes its arena offset to *offset (may be NULL).  Collective in the sense that every rank must call it at the
 * same point, so that the offsets agree; calling it again is a no-op.  A context that never registers allocates and
 * launches nothing for clipping.  Host only. */
int b2d_clip_register(b2d_ctx* ctx, size_t* offset);

/* Replaces: FairScale OSS.clip_grad_norm's local norm + NCCL all_reduce of its square (torch analogue:
 * torch.nn.utils.clip_grad_norm_ with norm_type 2 over the whole gradient).  x: this rank's n fp32 elements (its
 * reduced-gradient shard; n may be 0).  Every rank's sum of squares (fp64, an order fixed by n) reaches every rank;
 * each combines them in rank order and writes, with identical bits on every rank,
 *     norm_out[0] = fp32(sqrt(sum))    coef_out[0] = min(max_norm * (1 / (norm + 1e-6)), 1)   (NaN kept)
 * (device fp32).  max_norm must be finite and >= 0.  Asynchronous on the library's internal stream behind the reduce
 * buckets, after `wait_stream`; `comm_stream` waits for the result.  phases: bit 0 partial + push, bit 1 wait +
 * coefficient (3 = both); hosts that drive several ranks from one thread issue bit 0 for every rank, then bit 1. */
int b2d_clip_norm(b2d_ctx* ctx, const float* x, size_t n, float max_norm, float* norm_out, float* coef_out,
                  unsigned phases, void* wait_stream, void* comm_stream);

/* ---- symmetric arena ------------------------------------------------------------------- */

/* Bump-allocate `bytes` (256-byte aligned) of caller-visible symmetric memory.  Every rank
 * must make the same sequence of calls, so that offsets agree.  Never freed. */
int b2d_arena_alloc(b2d_ctx* ctx, size_t bytes, void** dev_ptr, size_t* offset);
/* Forget every bucket slot and arena allocation (host must have quiesced all ranks). */
int b2d_arena_reset(b2d_ctx* ctx);

/* ---- torch memory pool over the arena (f-1: zero-copy stage-in) ----------------------- */

/* Replaces: the cudaMalloc behind at::empty() for DDP's flat bucket tensors (reducer.hpp:347-406,
 * initialize_buckets), reached from ray_lightning/ray_ddp.py:75,112-116 with gradient_as_bucket_view=True.
 * b2d_pool_alloc / b2d_pool_free have the signature torch.cuda.memory.CUDAPluggableAllocator expects; while a
 * context is bound (b2d_pool_bind; NULL unbinds) allocations of its device are bump-allocated from its
 * symmetric arena; what the arena cannot take is served by cudaMalloc (and freed again), so torch never sees an
 * out-of-memory from this pool.  A bucket that lives in the arena is exchanged IN PLACE by the fp32-wire staged
 * algorithms; one that does not is staged like any other tensor. */
int b2d_pool_bind(b2d_ctx* ctx);
void* b2d_pool_alloc(size_t size, int device, void* stream);
void b2d_pool_free(void* ptr, size_t size, int device, void* stream);

/* ---- link probe ------------------------------------------------------------------------ */

/* Replaces: nothing (measurement aid).  Pull `bytes` from peer `peer`'s arena `iters` times and report GB/s:
 * mode 0 = cudaMemcpyAsync, mode 1 = a 16-byte-vector peer-read kernel (this library's access pattern).
 * Synchronises its own private stream only. */
int b2d_peer_bw(b2d_ctx* ctx, int peer, size_t bytes, int iters, int mode, double* gbps);

/* ---- introspection --------------------------------------------------------------------- */

typedef struct b2d_stats {
  uint64_t launches;       /* kernels launched by this ctx since creation */
  uint64_t timed_launches; /* launches bracketed by events (B2D_FLAG_TIMING) and resolved */
  double timed_ms;         /* sum of their device durations */
  uint64_t arena_bytes, arena_used;
  int32_t world, rank, device, sm_count;
  int32_t mem_kind;        /* 0 legacy IPC, 1 VMM */
  int32_t mc_bound;        /* 1 when NVLS is usable */
  int32_t last_algo, last_grid, last_block;
  int32_t pad_;
  uint64_t exch_launches;  /* exchange kernels (staged algorithms) launched */
  uint64_t exch_timed;     /* bucket exchanges bracketed by events (B2D_FLAG_TIMING) and resolved */
  double exch_ms;          /* sum of their device durations (first exchange kernel start .. last end) */
  uint64_t pool_allocs;    /* b2d_pool_alloc calls served */
  uint64_t pool_digest;    /* FNV-1a over their (offset, size): equal on every rank <=> bucket storage is symmetric */
} b2d_stats;

int b2d_ctx_stats(b2d_ctx* ctx, b2d_stats* out);   /* resolves finished timing events */
int b2d_ctx_reset_stats(b2d_ctx* ctx);
/* Debug: per-phase device times of the LAST allreduce launch.  enable=1 allocates the stamp buffer;
 * phase_us (>= 8 doubles) receives the mean over blocks of each interval between consecutive stamps
 * (two-shot: stage, barrier, reduce, barrier, gather) followed by max(end)-min(start); synchronises. */
int b2d_ctx_trace(b2d_ctx* ctx, int enable, double* phase_us, int* n_phases);
/* The algorithm AUTO would pick and the grid it would launch, without launching. */
int b2d_plan(b2d_ctx* ctx, size_t n, int wire, int algo, int* algo_out, int* grid_out, int* block_out);

#ifdef __cplusplus
}
#endif
#endif /* B2D_H_ */
