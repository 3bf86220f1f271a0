"""RayStrategy — DDP on actor-spawned workers, with the gradient allreduce done by libb2d.

Drop-in for ``ray_lightning.RayStrategy`` (ray_lightning/ray_ddp.py:22-333): same constructor,
attributes, properties and overridden hooks, so ``Trainer(strategy=RayStrategy(...))`` reads the
same.  What differs is underneath the ``**ddp_kwargs`` pass-through (reference :75,112-116): when
``use_gpu`` is set and the caller did not bring a comm hook of their own, the strategy registers
``b200_allreduce_hook`` through the SAME seam PL offers for ``ddp_comm_hook`` — so every bucket
the Reducer finishes goes to one fused sm_90a kernel instead of cast + div + ncclAllReduce +
copy.  New knobs ride in as keyword arguments prefixed ``b200_`` and never reach
``DistributedDataParallel``:

    b200_wire="fp32"|"bf16"   arithmetic contract.  Default "fp32": DDP's default divide + fp32 SUM allreduce, what the
                              reference computes when no comm hook is given.  "bf16" is torch's ``bf16_compress_hook``
                              (bf16 on the wire, fp32 accumulate); passing ``ddp_comm_hook=default_hooks.
                              bf16_compress_hook`` — the reference's own way to ask for it — selects it too.
    b200_algo="auto"|"one_shot"|"two_shot"|"staged"|"nvls"
    b200_mem="vmm"|"ipc"      how arenas are shared between the worker processes
    b200_timeout_ms           peer watchdog (default: the process group's timeout; 0 = never trap)
    b200_max_ctas, b200_one_shot_max_bytes, b200_chunk_bytes, b200_exch_ctas, b200_timing, b200_nvls,
    b200_arena_buckets=True   (with gradient_as_bucket_view=True and the fp32 wire) let DDP's flat bucket tensors live
                              in the symmetric arena so that buckets are exchanged in place — no stage-in copy
    b200_buffer_sync=True     module buffers (BatchNorm statistics) live in the arena; DDP's per-forward broadcast from
                              rank 0 becomes one peer-store kernel instead of a coalesced ncclBroadcast
    b200_optimizer_in_backward=False   SGD / Adam / AdamW applied per DDP bucket right behind its allreduce, on the comm
                              stream, while backward continues (torch's `_hook_then_optimizer`, fused); one backward
                              per step, one parameter group
    b200_enable=True

``Trainer(gradient_clip_val=...)`` clips the averaged gradients after DDP's backward with torch's own
``clip_grad_norm_`` / ``clip_grad_value_`` (they are whole and identical on every rank); it cannot be combined with
``b200_optimizer_in_backward``.

``Trainer(sync_batchnorm=True)`` on the libb2d path converts every BatchNorm to ``syncbn.B200SyncBatchNorm``, whose
statistics cross ranks through the arena; elsewhere it is torch's ``SyncBatchNorm``.

There is no CPU implementation of that hook: with ``use_gpu=False`` the strategy is the
reference's own CPU configuration (torch DDP over gloo), and with ``use_gpu=True`` a missing
libb2d.so or GPU is an error, not a fallback.
"""
import os
import warnings
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch

from ._compat import DDPSpawnStrategy, rank_zero_info, rank_zero_only, ray, reset_seed
from .launchers.ray_launcher import RayLauncher

_B200_DEFAULTS = dict(enable=True, wire="fp32", algo="auto", mem="vmm", max_ctas=None, one_shot_max_bytes=None,
                      timing=False, nvls="auto", arena_bytes=None, timeout_ms=None, chunk_bytes=None, exch_ctas=None,
                      arena_buckets=True, reduce_bucket_mb=None, arena_extra_bytes=0, buffer_sync=True, optimizer_in_backward=False)


def _is_torch_bf16_hook(hook) -> bool:
    try:
        from torch.distributed.algorithms.ddp_comm_hooks import default_hooks
        return hook is default_hooks.bf16_compress_hook
    except Exception:  # pragma: no cover
        return False


def _split_b200_kwargs(kwargs: Dict[str, Any]) -> Dict[str, Any]:
    opts = dict(_B200_DEFAULTS)
    for k in list(kwargs):
        if k.startswith("b200_"):
            name = k[len("b200_"):]
            if name not in opts:
                raise TypeError("unknown RayStrategy option %r (known: %s)"
                                % (k, ", ".join("b200_" + n for n in sorted(opts))))
            opts[name] = kwargs.pop(k)
    return opts


class RayStrategy(DDPSpawnStrategy):
    """PyTorch-Lightning strategy for DDP training on actor workers, one GPU each.

    Args mirror ray_lightning/ray_ddp.py:69-75:
        num_workers, num_cpus_per_worker, use_gpu, init_hook, resources_per_worker
        (``"CPU"`` / ``"GPU"`` keys override the per-worker CPU / GPU counts), ``**ddp_kwargs``
        forwarded to ``DistributedDataParallel`` (``bucket_cap_mb``, ``find_unused_parameters``,
        ``gradient_as_bucket_view``, ``ddp_comm_hook`` ...).
    """

    strategy_name = "ddp_ray"

    def __init__(self,
                 num_workers: int = 1,
                 num_cpus_per_worker: int = 1,
                 use_gpu: bool = False,
                 init_hook: Optional[Callable] = None,
                 resources_per_worker: Optional[Dict] = None,
                 **ddp_kwargs: Union[Any, Dict[str, Any]]):
        resources = dict(resources_per_worker) if resources_per_worker else {}
        self.nickname = "ddp_ray"
        self.num_workers = int(num_workers)
        self.num_cpus_per_worker = resources.pop("CPU", num_cpus_per_worker)
        self.num_gpus_per_worker = resources.pop("GPU") if "GPU" in resources else int(use_gpu)
        self.use_gpu = self.num_gpus_per_worker > 0
        if self.use_gpu and self.num_gpus_per_worker < 1 and num_workers > 1:
            warnings.warn("Identified less than 1 GPU being set per worker. GPU devices cannot be shared across "
                          "NCCL workers; libb2d's peer mapping works with shared devices, but the control-plane "
                          "process group must then be gloo: set PL_TORCH_DISTRIBUTED_BACKEND=gloo.")
        self.additional_resources_per_worker = resources
        self.init_hook = init_hook

        self._local_rank = 0
        self._global_rank = 0
        self._node_rank = 0
        self._is_remote = False
        self._device = None
        self.global_to_local = None

        self._b200 = _split_b200_kwargs(ddp_kwargs)
        if self.use_gpu and self._b200["enable"] and _is_torch_bf16_hook(ddp_kwargs.get("ddp_comm_hook")) \
                and ddp_kwargs.get("ddp_comm_state") is None and ddp_kwargs.get("ddp_comm_wrapper") is None:
            # the reference's way to ask for bf16 gradient compression: same arithmetic contract, fused kernel
            ddp_kwargs.pop("ddp_comm_hook")
            self._b200["wire"] = "bf16"
        if self.use_gpu and self._b200["enable"] and ddp_kwargs.get("ddp_comm_hook") is None:
            # Installed through PL's own ddp_comm_hook seam.  The state object holds no CUDA handle
            # yet (this strategy is pickled to every actor, reference ray_launcher.py:240-245).
            from .comm import B200HookState, b200_allreduce_hook
            o = self._b200
            ddp_kwargs["ddp_comm_state"] = B200HookState(
                wire=o["wire"], algo=o["algo"], mem=o["mem"], timing=o["timing"], max_ctas=o["max_ctas"],
                one_shot_max_bytes=o["one_shot_max_bytes"], nvls=o["nvls"], arena_bytes=o["arena_bytes"],
                timeout_ms=o["timeout_ms"], chunk_bytes=o["chunk_bytes"], exch_ctas=o["exch_ctas"],
                arena_buckets=o["arena_buckets"] and o["wire"] == "fp32", arena_extra_bytes=o["arena_extra_bytes"])
            ddp_kwargs["ddp_comm_hook"] = b200_allreduce_hook

        super().__init__(accelerator="_gpu" if use_gpu else "cpu", parallel_devices=[], cluster_environment=None,
                         **ddp_kwargs)

    # ---- driver side --------------------------------------------------------------------------
    def _configure_launcher(self):
        """Driver: the launcher owns the actors (reference :118-126)."""
        self._launcher = RayLauncher(self)

    # ---- worker side --------------------------------------------------------------------------
    def set_remote(self, remote: bool):
        self._is_remote = remote

    def set_global_to_local(self, global_to_local: List[Optional[Tuple[int, int]]]):
        self.global_to_local = global_to_local

    def set_world_ranks(self, process_idx: int = 0):
        """Ranks exist only once the actors do; on the driver this is a no-op (reference :145-159)."""
        if self._is_remote:
            self._global_rank = process_idx
            self._local_rank, self._node_rank = self.global_to_local[self.global_rank]

    def _worker_setup(self, process_idx: int):
        """Join the control-plane process group (``env://``) — reference :161-203.  libb2d's arena
        handles are exchanged over this group on the first bucket; gradients never use it."""
        reset_seed()
        self.set_world_ranks(process_idx)
        rank_zero_only.rank = self.global_rank
        self._process_group_backend = self._get_process_group_backend()
        if not torch.distributed.is_available():
            raise RuntimeError("torch.distributed is not available. Cannot initialize distributed process group")
        if torch.distributed.is_initialized():
            return
        backend = self.torch_distributed_backend
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(self.root_device)
            kw["device_id"] = self.root_device
        torch.distributed.init_process_group(backend, rank=self.global_rank, world_size=self.world_size,
                                             init_method="env://", **kw)
        rank_zero_info("distributed_backend=%s: all %d processes registered" % (backend, self.world_size))

    def configure_ddp(self) -> None:
        """DDP construction (reference :112-116 via PL), with DDP's flat bucket tensors placed in libb2d's symmetric
        arena when the fp32 wire is used (SURVEY §8 f-1): the hook then exchanges every bucket where it lies."""
        st = self.b200_state
        self.b200_arena_buckets_active = False
        self._b200_rebuilt = False
        self._b200_steps = 0
        if st is not None and self.root_device.type == "cuda" and self.world_size > 1:
            self._setup_sync_batchnorm(st)
        if (st is None or not self._b200["arena_buckets"] or st.wire != "fp32" or self.root_device.type != "cuda"
                or self.world_size < 2 or self._ddp_comm_wrapper is not None):
            return super().configure_ddp()
        if st.total_grad_elems is None:
            st.total_grad_elems = sum(p.numel() for p in self.model.parameters() if p.requires_grad)
        st.ensure(self.root_device)          # collective: every worker is here
        with st.allocate_in_arena():
            super().configure_ddp()
        self.b200_arena_buckets_active = st.verify_symmetric_buckets()

    def configure_sync_batchnorm(self, model):
        """``Trainer(sync_batchnorm=True)``: PL converts every BatchNorm before DDP wraps the model.  On the libb2d path
        the layers become ``B200SyncBatchNorm`` (statistics exchanged by peer stores); otherwise — ``b200_enable=False``,
        ``use_gpu=False`` or a comm hook of the user's — torch's ``SyncBatchNorm``, as in the reference."""
        st = self.b200_state
        if st is None or self.root_device.type != "cuda":
            return super().configure_sync_batchnorm(model)
        from .syncbn import convert_sync_batchnorm
        return convert_sync_batchnorm(model, lambda: st.comm)

    def _setup_sync_batchnorm(self, st):
        """Collective, before the first forward: the communicator must exist with room for every layer's exchange
        region, and the regions must be registered in the same order on every rank."""
        from .syncbn import register_sync_batchnorm, sync_batchnorm_layers, syncbn_arena_bytes
        layers = sync_batchnorm_layers(self.lightning_module)
        if not layers:
            return
        if st.comm is None:
            st.arena_extra_bytes += syncbn_arena_bytes([m.num_features for m in layers], self.world_size)
        if st.total_grad_elems is None:
            st.total_grad_elems = sum(p.numel() for p in self.model.parameters() if p.requires_grad)
        st.ensure(self.root_device)
        register_sync_batchnorm(self.lightning_module, st.comm)

    def training_step(self, *args):
        st = self.b200_state
        if getattr(self, "b200_arena_buckets_active", False) and not self._b200_rebuilt:
            if self._b200_steps >= 1 and torch.is_grad_enabled():
                # DDP lays its buckets out anew once, in the forward of the second iteration (reducer.hpp:125-151,
                # distributed.py `_pre_forward`).  Do it here, with the arena as the allocator; DDP's own call is
                # then a no-op.
                with st.allocate_in_arena():
                    self.model.reducer._rebuild_buckets()
                self._b200_rebuilt = True
                self.b200_arena_buckets_active = st.verify_symmetric_buckets()
            self._b200_steps += 1
        return super().training_step(*args)

    def setup_optimizers(self, trainer) -> None:
        if self._b200["optimizer_in_backward"] and (getattr(trainer, "gradient_clip_val", None) or 0) > 0:
            raise ValueError("b200_optimizer_in_backward=True cannot be combined with gradient_clip_val: the step runs "
                             "inside backward, before the gradient norm is known")
        super().setup_optimizers(trainer)
        st = self.b200_state
        if st is not None and self._b200["optimizer_in_backward"] and self.root_device.type == "cuda":
            from .comm import InBackwardOptimizer
            if len(self.optimizers) != 1:
                raise ValueError("b200_optimizer_in_backward needs exactly one optimizer")
            base = self.optimizers[0]
            wrapped = InBackwardOptimizer(base, st)
            for sch in self.lr_schedulers:
                if getattr(sch, "optimizer", None) is base:
                    sch.optimizer = wrapped
            self.optimizers = [wrapped]

    def _register_ddp_hooks(self) -> None:
        """Size the symmetric arena from the wrapped module, then let the base class register the hook."""
        state = getattr(self, "_ddp_comm_state", None)
        if state is not None and hasattr(state, "total_grad_elems") and state.total_grad_elems is None:
            state.total_grad_elems = sum(p.numel() for p in self.model.parameters() if p.requires_grad)
        if state is not None and hasattr(state, "ensure") and self.root_device.type != "cuda" and self.use_gpu:
            raise RuntimeError("RayStrategy(use_gpu=True) needs a CUDA device in the worker: the H100 gradient-sync "
                               "path has no CPU fallback")
        super()._register_ddp_hooks()
        # f-3: the per-forward buffer broadcast (BatchNorm statistics ...) goes through the arena too
        ddp = self.model
        if (state is not None and hasattr(state, "ensure") and self._b200["buffer_sync"] and self.world_size > 1
                and self.root_device.type == "cuda" and hasattr(ddp, "_register_buffer_comm_hook")
                and getattr(ddp, "broadcast_buffers", True) and any(True for _ in ddp.module.buffers())):
            from torch.nn.parallel.distributed import _BufferCommHookLocation
            from .comm import ArenaBufferSync, b200_buffer_hook
            self._b200_buffer_state = ArenaBufferSync(state)
            ddp._register_buffer_comm_hook(self._b200_buffer_state, b200_buffer_hook,
                                           comm_hook_location=_BufferCommHookLocation.PRE_FORWARD)   # where DDP's own sync sits

    @property
    def b200_state(self):
        """The hook state (communicator, side stream, counters) of this worker, or None."""
        st = getattr(self, "_ddp_comm_state", None)
        return st if hasattr(st, "ensure") else None

    def teardown_worker(self) -> None:
        """Worker: release the communicator before the process group goes away."""
        st = self.b200_state
        bst = getattr(self, "_b200_buffer_state", None)
        if bst is not None and bst.flat is not None and self.lightning_module is not None:
            for b in self.lightning_module.buffers():        # give the buffers ordinary storage back
                if st.comm is not None and st.comm.owns(b):
                    b.data = b.data.clone()
            self._b200_buffer_state = None
        self.model = None          # the Reducer's arena-backed buckets go before the arena does
        if st is not None:
            import gc
            gc.collect()
            st.close()
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.destroy_process_group()

    @property
    def world_size(self) -> int:
        return self.num_workers

    @property
    def local_rank(self) -> int:
        return self._local_rank

    @local_rank.setter
    def local_rank(self, value: int):
        self._local_rank = value

    @property
    def global_rank(self) -> int:
        return self._global_rank

    @global_rank.setter
    def global_rank(self, value: int):
        self._global_rank = value

    @property
    def node_rank(self) -> int:
        return self._node_rank

    @property
    def root_device(self):
        """cuda:<position of this worker's GPU id inside the shared CUDA_VISIBLE_DEVICES>
        (reference :259-304; the index libb2d receives as ``device``)."""
        if self._device:
            return self._device
        if not (self.use_gpu and torch.cuda.is_available()):
            return torch.device("cpu")
        if not self._is_remote:
            return torch.device("cuda:0")  # asked on the driver: any device will do
        device_id = 0
        gpu_ids = [str(g) for g in ray.get_gpu_ids()]  # ints or strings, depending on the runtime
        if gpu_ids:
            gpu_id = gpu_ids[0]  # first one if several; fractional GPUs may be shared between workers
            visible = os.environ.get("CUDA_VISIBLE_DEVICES", "")
            if not visible or visible == "NoDevFiles" or gpu_id not in visible.split(","):
                raise RuntimeError("CUDA_VISIBLE_DEVICES set incorrectly. Got %s, expected to include %s. "
                                   "Did you override the `CUDA_VISIBLE_DEVICES` environment variable?"
                                   % (visible, gpu_id))
            device_id = visible.split(",").index(gpu_id)
        return torch.device("cuda:%d" % device_id)

    @root_device.setter
    def root_device(self, device):
        self._device = device

    @property
    def distributed_sampler_kwargs(self):
        """(reference :315-324; pinned by ray_lightning/tests/test_ddp.py:179-211)"""
        return dict(num_replicas=self.num_workers, rank=self.global_rank)

    def teardown(self) -> None:
        """Driver-side teardown (reference :326-333)."""
        self.accelerator = None
        super().teardown()
