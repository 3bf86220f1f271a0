"""Synchronised BatchNorm over libb2d peer memory: what ``Trainer(sync_batchnorm=True)`` gives RayStrategy and
RayShardedStrategy on the GPU.

``B200SyncBatchNorm`` is a ``torch.nn.SyncBatchNorm`` (same parameters, buffers, state-dict keys and ``isinstance``
answers; checkpoints interchange with torch's module) whose cross-rank exchange is libb2d's instead of torch's:

    forward   torch.batch_norm_stats -> b2d_bn_stats_exchange -> torch.batch_norm_elemt
    backward  torch.batch_norm_backward_reduce -> b2d_bn_grad_exchange -> torch.batch_norm_backward_elemt

The per-rank arithmetic is torch's own; the exchange replaces the cat + all_gather_into_tensor + host-side mask +
batch_norm_gather_stats_with_counts of torch/nn/modules/_functions.py:65-115 and the cat + all_reduce + split of
:155-165 with one peer-store kernel and one combine kernel each, on the compute stream, without host
synchronisation.  Whole world only: a module with a ``process_group`` other than the whole world is refused.
"""
import torch
import torch.nn.functional as F

__all__ = ["B200SyncBatchNorm", "convert_sync_batchnorm", "sync_batchnorm_layers", "register_sync_batchnorm",
           "syncbn_arena_bytes"]


def _row_floats(channels):
    """Floats of a forward and of a backward row (b2d_syncbn.cuh: both padded to 16 bytes)."""
    return (2 * channels + 1 + 3) // 4 * 4, (2 * channels + 3) // 4 * 4


def syncbn_arena_bytes(channels, world):
    """Arena bytes that b2d_bn_register takes for layers of these channel counts at this world size: two generations of
    W forward and W backward rows per layer, each region 256-byte aligned (b2d.cu)."""
    total = 0
    for c in channels:
        f, b = _row_floats(int(c))
        total += -(-(2 * world * (f + b) * 4) // 256) * 256
    return total


def _channels_last(t):
    return t.is_contiguous(memory_format=torch.channels_last) or t.is_contiguous(memory_format=torch.channels_last_3d)


class _SyncBatchNormFunction(torch.autograd.Function):
    """torch's ``SyncBatchNorm`` autograd function (torch/nn/modules/_functions.py) with libb2d as the exchange."""

    @staticmethod
    def forward(ctx, input, weight, bias, running_mean, running_var, eps, momentum, comm, layer_id):
        if not _channels_last(input):
            input = input.contiguous()
        if weight is not None:
            weight = weight.contiguous()
        channels = input.shape[1]
        dev = input.device
        mean = torch.empty(channels, dtype=torch.float32, device=dev)
        invstd = torch.empty(channels, dtype=torch.float32, device=dev)
        counts = torch.empty(comm.world, dtype=torch.int32, device=dev)
        if input.numel() > 0:
            local_mean, local_invstd = torch.batch_norm_stats(input, eps)
            count = float(input.numel() // channels)
        else:
            local_mean = local_invstd = None          # an empty rank pushes a zero row and is skipped by every peer
            count = 0.0
        comm.bn_stats_exchange(layer_id, local_mean, local_invstd, count, eps, momentum, mean, invstd, counts,
                               running_mean, running_var)
        ctx.save_for_backward(input, weight, mean, invstd, counts)
        ctx.comm, ctx.layer_id = comm, layer_id
        if input.numel() > 0:
            return torch.batch_norm_elemt(input, weight, bias, mean, invstd, eps)
        return torch.empty_like(input)

    @staticmethod
    def backward(ctx, grad_output):
        if not _channels_last(grad_output):
            grad_output = grad_output.contiguous()
        saved_input, weight, mean, invstd, counts = ctx.saved_tensors
        comm, layer_id = ctx.comm, ctx.layer_id
        grad_input = grad_weight = grad_bias = None
        sum_dy_all = torch.empty_like(mean)
        sum_dy_xmu_all = torch.empty_like(mean)
        if saved_input.numel() > 0:
            sum_dy, sum_dy_xmu, grad_weight, grad_bias = torch.batch_norm_backward_reduce(
                grad_output, saved_input, mean, invstd, weight,
                ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2])
            if ctx.needs_input_grad[0]:
                comm.bn_grad_exchange(layer_id, sum_dy, sum_dy_xmu, sum_dy_all, sum_dy_xmu_all)
                if weight is not None and weight.dtype != mean.dtype:
                    weight = weight.to(mean.dtype)
                grad_input = torch.batch_norm_backward_elemt(grad_output, saved_input, mean, invstd, weight, sum_dy_all,
                                                             sum_dy_xmu_all, counts)
            # grad_weight / grad_bias are local: DDP (or the sharded reduce) averages them like any other gradient
            if weight is None or not ctx.needs_input_grad[1]:
                grad_weight = None
            if weight is None or not ctx.needs_input_grad[2]:
                grad_bias = None
        elif ctx.needs_input_grad[0]:
            # this rank had no samples: it still takes part in the exchange, with a zero row
            comm.bn_grad_exchange(layer_id, None, None, sum_dy_all, sum_dy_xmu_all)
        return grad_input, grad_weight, grad_bias, None, None, None, None, None, None


class B200SyncBatchNorm(torch.nn.SyncBatchNorm):
    """``torch.nn.SyncBatchNorm`` with libb2d's exchange.  ``comm_getter()`` returns the rank's libb2d communicator (or
    None); it is asked on every training forward, because the strategy creates the communicator after conversion.
    ``layer_id`` names the layer's exchange region (``register_sync_batchnorm``)."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, layer_id=0,
                 comm_getter=None, device=None, dtype=None):
        super().__init__(num_features, eps, momentum, affine, track_running_stats, None, device, dtype)
        self.layer_id = int(layer_id)
        self._comm_getter = comm_getter

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_comm_getter"] = None      # a communicator belongs to one worker process
        return d

    def forward(self, input):
        self._check_input_dim(input)
        self._check_non_zero_input_channels(input)
        # torch.nn.SyncBatchNorm.forward's preamble
        exponential_average_factor = 0.0 if self.momentum is None else self.momentum
        if self.training and self.track_running_stats:
            self.num_batches_tracked.add_(1)
            if self.momentum is None:
                exponential_average_factor = 1.0 / self.num_batches_tracked.item()
            else:
                exponential_average_factor = self.momentum
        bn_training = True if self.training else (self.running_mean is None and self.running_var is None)
        comm = self._comm_getter() if (bn_training and self.training and self._comm_getter is not None) else None
        need_sync = comm is not None and comm.world > 1
        running_mean = self.running_mean if not self.training or self.track_running_stats else None
        running_var = self.running_var if not self.training or self.track_running_stats else None
        if not need_sync:
            return F.batch_norm(input, running_mean, running_var, self.weight, self.bias, bn_training,
                                exponential_average_factor, self.eps)
        # the buffers are read here on every call: ArenaBufferSync.adopt may have moved them into the arena
        return _SyncBatchNormFunction.apply(input, self.weight, self.bias, running_mean, running_var, self.eps,
                                            exponential_average_factor, comm, self.layer_id)


def convert_sync_batchnorm(module, comm_getter):
    """``torch.nn.SyncBatchNorm.convert_sync_batchnorm`` with ``B200SyncBatchNorm``: every BatchNorm*D (and every
    torch SyncBatchNorm over the whole world) becomes a ``B200SyncBatchNorm`` that keeps the same Parameter and buffer
    objects.  Layers are numbered in traversal order, which is the same on every rank."""
    counter = [0]

    def convert(m):
        out = m
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            pg = getattr(m, "process_group", None)
            if pg is not None and not _is_world(pg):
                raise ValueError("B200SyncBatchNorm synchronises over the whole world only; %s has a process_group "
                                 "that is a subgroup" % type(m).__name__)
            for name in ("running_mean", "running_var"):
                buf = getattr(m, name)
                if buf is not None and buf.dtype != torch.float32:
                    raise ValueError("B200SyncBatchNorm keeps running statistics in float32; %s.%s is %s"
                                     % (type(m).__name__, name, buf.dtype))
            out = B200SyncBatchNorm(m.num_features, m.eps, m.momentum, m.affine, m.track_running_stats,
                                    layer_id=counter[0], comm_getter=comm_getter)
            counter[0] += 1
            if m.affine:
                with torch.no_grad():
                    out.weight = m.weight
                    out.bias = m.bias
            out.running_mean = m.running_mean
            out.running_var = m.running_var
            out.num_batches_tracked = m.num_batches_tracked
            out.training = m.training
            if hasattr(m, "qconfig"):
                out.qconfig = m.qconfig
        for name, child in m.named_children():
            out.add_module(name, convert(child))
        return out

    return convert(module)


def _is_world(pg):
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return False
    return pg is dist.group.WORLD or dist.get_world_size(pg) == dist.get_world_size()


def sync_batchnorm_layers(module):
    """The ``B200SyncBatchNorm`` modules of ``module``, each once, in traversal order."""
    return [m for m in module.modules() if isinstance(m, B200SyncBatchNorm)]


def register_sync_batchnorm(module, comm):
    """Collective: give every ``B200SyncBatchNorm`` of ``module`` its exchange region in ``comm``'s arena.  Must run
    before the first training forward, on every rank, with the same module structure."""
    layers = sync_batchnorm_layers(module)
    return comm.bn_register_all([(m.layer_id, m.num_features) for m in layers])
