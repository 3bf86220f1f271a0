"""RayShardedStrategy — optimizer-state + gradient sharding on actor workers.

Drop-in for ``ray_lightning.RayShardedStrategy`` (ray_lightning/ray_ddp_sharded.py:8-13: pure
composition of RayStrategy and PL's DDPSpawnShardedStrategy, whose FairScale machinery does the
work).  Here ``configure_ddp`` builds ``sharded.FlatShards`` + ``sharded.ShardedOptimizer``
instead of FairScale's ShardedDataParallel + OSS: same observable behaviour — whole parameters
after every step, optimizer state for the owned shard only, consolidated checkpoints — through
libb2d's reduce-scatter / partitioned-Adam / all-gather kernels.

``use_gpu=False`` keeps the reference's CPU semantics with what torch itself ships (FairScale is
not installable here): DDP over gloo + ``ZeroRedundancyOptimizer`` — same sharded-state,
consolidate-before-save behaviour.
"""
import torch

from ._compat import DDPSpawnShardedStrategy
from .ray_ddp import RayStrategy


# C3 linearisation visits RayStrategy before DDPSpawnShardedStrategy; both share DDPSpawnStrategy.
class RayShardedStrategy(RayStrategy, DDPSpawnShardedStrategy):
    strategy_name = "ddp_sharded_ray"

    def __init__(self, *args, **kwargs):
        kwargs.setdefault("b200_enable", True)
        # wire format of the reduce-to-owner: like PL's sharded plugin (reduce_fp16 only under 16-bit precision) fp32
        # unless the trainer runs at 16-bit / bf16 precision; b200_wire="bf16" | "fp32" forces it
        kwargs.setdefault("b200_wire", None)
        super().__init__(*args, **kwargs)
        self._shards = None
        self._sharded_ready = False

    def configure_ddp(self):
        if self.root_device.type != "cuda":
            if self.use_gpu:
                raise RuntimeError("RayShardedStrategy(use_gpu=True) needs a CUDA device in the worker")
            return self._configure_cpu_reference()
        # GPU: no DDP wrapper at all — autograd hooks send every reduce bucket to its owners while backward runs
        from .comm import Communicator
        o = self._b200
        total = sum(p.numel() for p in self.lightning_module.parameters() if p.requires_grad)
        # flat fp32 parameters (4 B/element) + one single-buffered staging copy at wire width + a gather buffer for
        # consolidated checkpoints (4 B/element)
        wire = o["wire"] or ("bf16" if str(getattr(self, "precision", 32)) in ("16", "bf16") else "fp32")
        wire_w = 2 if wire == "bf16" else 4
        from .syncbn import register_sync_batchnorm, sync_batchnorm_layers, syncbn_arena_bytes
        bn_layers = sync_batchnorm_layers(self.lightning_module) if self.world_size > 1 else []
        bn_bytes = syncbn_arena_bytes([m.num_features for m in bn_layers], self.world_size)
        nbytes = o["arena_bytes"] or int((8 + wire_w) * total + (128 << 20) + o["arena_extra_bytes"] + bn_bytes)
        self._comm = Communicator(self.global_rank, self.world_size, self.root_device.index, nbytes, mem=o["mem"],
                                  timing=o["timing"], max_ctas=o["max_ctas"], nvls=o["nvls"], timeout_ms=o["timeout_ms"],
                                  exch_ctas=o["exch_ctas"])
        if bn_layers:
            # no DDP wrapper broadcasts buffers here: synchronised statistics keep the running statistics equal
            register_sync_batchnorm(self.lightning_module, self._comm)
        # the flat layout follows the optimizer's parameter groups: built in setup_optimizers, once they are known
        self.model = self.lightning_module
        self._sharded_wire = wire
        self._sharded_ready = True

    def configure_sync_batchnorm(self, model):
        """On the GPU the sharded path always has a libb2d communicator (created in configure_ddp): the layers become
        ``B200SyncBatchNorm`` over it.  On the CPU reference path, torch's ``SyncBatchNorm``."""
        if self.root_device.type != "cuda":
            return DDPSpawnShardedStrategy.configure_sync_batchnorm(self, model)
        from .syncbn import convert_sync_batchnorm
        return convert_sync_batchnorm(model, lambda: getattr(self, "_comm", None))

    def _configure_cpu_reference(self):
        super().configure_ddp()

    def setup_optimizers(self, trainer):
        super().setup_optimizers(trainer)
        if getattr(self, "_sharded_ready", False):
            from .sharded import FlatShards, ShardedOptimizer, group_index_of
            if len(self.optimizers) != 1:
                raise ValueError("RayShardedStrategy(use_gpu=True) shards ONE optimizer over all trainable parameters; "
                                 "got %d" % len(self.optimizers))
            params = [p for p in self.lightning_module.parameters() if p.requires_grad]
            self._shards = FlatShards(self.lightning_module, self._comm, wire=self._sharded_wire,
                                      group_of=group_index_of(params, self.optimizers[0]),
                                      reduce_bucket_mb=self._b200.get("reduce_bucket_mb") or 25.0)
            side = torch.cuda.Stream(device=self.root_device, priority=-1)
            wrapped = []
            for opt in self.optimizers:
                sopt = ShardedOptimizer(opt, self._shards, wire=self._sharded_wire, stream=side,
                                        nvls=bool(self._comm.nvls) and self.world_size >= 4)
                for sch in self.lr_schedulers:
                    if getattr(sch, "optimizer", None) is opt:
                        sch.optimizer = sopt
                wrapped.append(sopt)
            self.optimizers = wrapped
        elif torch.distributed.is_available() and torch.distributed.is_initialized() and self.world_size > 1:
            from torch.distributed.optim import ZeroRedundancyOptimizer
            wrapped = []
            for opt in self.optimizers:
                g = {k: v for k, v in opt.param_groups[0].items() if k != "params"}
                z = ZeroRedundancyOptimizer(opt.param_groups[0]["params"], optimizer_class=type(opt), **g)
                for sch in self.lr_schedulers:
                    if getattr(sch, "optimizer", None) is opt:
                        sch.optimizer = z
                wrapped.append(z)
            self.optimizers = wrapped

    def clip_gradients(self, optimizer, clip_val, algorithm="norm"):
        """On the GPU the gradients exist only as every owner's shard of the averaged gradient (``param.grad`` are zero
        by now): the ``ShardedOptimizer`` clips there, with a global norm over every rank.  On the CPU reference path DDP
        leaves whole gradients and torch's own clipping applies."""
        from .sharded import ShardedOptimizer
        if not isinstance(optimizer, ShardedOptimizer):
            return super().clip_gradients(optimizer, clip_val, algorithm)
        if algorithm == "value":
            optimizer.clip_grad_value(clip_val)
        else:
            optimizer.clip_grad_norm(clip_val)

    def training_step(self, *args):
        if self._shards is None:
            return super().training_step(*args)
        with self._autocast():
            return self.lightning_module.training_step(*args)

    def optimizer_state_for_checkpoint(self, trainer):
        """Collective: consolidate the sharded state to the stock layout (what PL does with
        ``OSS.consolidate_state_dict`` before saving)."""
        out = []
        for opt in self.optimizers:
            if hasattr(opt, "consolidate_state_dict"):  # ZeroRedundancyOptimizer
                opt.consolidate_state_dict(to=0)
                out.append(opt.state_dict() if self.global_rank == 0 else {})
            else:
                out.append(opt.state_dict())
        return out

    def teardown_worker(self) -> None:
        comm = getattr(self, "_comm", None)
        if comm is not None:
            torch.cuda.synchronize()
            if self._shards is not None:
                for p in self._shards.params:        # parameters were views of the arena: give them ordinary storage back
                    p.data = p.data.clone()
                    p.grad = None
            self._shards = None
            self.optimizers = []
            comm.close()
            self._comm = None
        super().teardown_worker()
