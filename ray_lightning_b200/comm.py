"""Tensor-level host side of the H100 gradient-sync path.

* ``Communicator``   — one rank of a one-process-per-GPU job (the Ray-actor model of
  ray_lightning/launchers/ray_launcher.py:105-114): creates the libb2d context, exchanges the
  arena handles over the torch process group that ``RayStrategy._worker_setup`` already made
  (ray_lightning/ray_ddp.py:192-196) and exposes allreduce / sharded-step calls on tensors.
* ``LoopbackGroup``  — W ranks inside ONE process on ONE device (separate arenas, separate
  streams).  Exercises the whole inter-rank protocol (barriers, slicing, double buffering)
  on a single GPU; used by the parity tests and by ``bench.py`` at ``--gpus 1``.
* ``B200HookState`` / ``b200_allreduce_hook`` — the torch DDP communication hook
  (torch/nn/parallel/distributed.py:1987-2067) that replaces ``bf16_compress_hook`` /
  the default allreduce with one fused kernel per bucket.

No function here has a CPU implementation: tensors must be CUDA tensors and libb2d must load.
"""
import contextlib
import os
import socket
import struct
import uuid

import torch
import torch.distributed as dist

from . import _b2d
from ._b2d import ALGO_NAMES, FLAG_MEM_VMM, FLAG_TIMING, WIRE_NAMES, AdamParams, B2DError
from ._optim import kernel_args

__all__ = ["Communicator", "LoopbackGroup", "B200HookState", "b200_allreduce_hook", "arena_bytes_for",
           "arena_tensor", "ArenaBufferSync", "b200_buffer_hook", "InBackwardOptimizer"]


def _wire(w):
    return WIRE_NAMES[w] if isinstance(w, str) else int(w)


def _algo(a):
    return ALGO_NAMES[a] if isinstance(a, str) else int(a)


def arena_bytes_for(total_grad_elems, extra_bytes=0, wire="fp32", arena_buckets=False):
    """Arena size for a model with that many gradient elements.
      bf16 wire : a double-buffered staging copy at 2 B/element; DDP lays its buckets out anew once after the first
                  iteration (reducer.hpp:125-151) and the regions of the old layout are recycled (first fit), so
                  6 B/element covers the transient;
      fp32 wire : the same at 4 B/element -> 12 B/element — or, when DDP's bucket tensors themselves live in the
                  arena (exchanged in place, no staging): the two generations of bucket storage, 8 B/element, plus
                  256 MiB for the one coalescing buffer DDP's initial parameter broadcast allocates under the same
                  pool (torch caches and re-uses it; anything the arena cannot take falls back to cudaMalloc);
    plus 64 MiB for the signal pad, alignment and small buckets."""
    if wire != "bf16" and arena_buckets:
        return int(8 * total_grad_elems + (320 << 20) + extra_bytes)
    per = 6 if wire == "bf16" else 12
    return int(per * total_grad_elems + (64 << 20) + extra_bytes)


class _DevMem:
    """Exposes a raw device range through __cuda_array_interface__ so torch can view it."""

    def __init__(self, ptr, nbytes, owner):
        self._owner = owner  # keeps the libb2d context (and so the arena) alive
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1",
                                         "data": (int(ptr), False), "version": 2}


def arena_tensor(ctx, numel, dtype, device):
    """Allocate ``numel`` elements of ``dtype`` in the symmetric arena and view them as a tensor."""
    nbytes = numel * torch.empty((), dtype=dtype).element_size()
    ptr, off = ctx.arena_alloc(max(nbytes, 16))
    t = torch.as_tensor(_DevMem(ptr, max(nbytes, 16), ctx), device=device)
    return t[:nbytes].view(dtype), off


def _check_tensor(t, device_index):
    if not t.is_cuda:
        raise ValueError("libb2d works on CUDA tensors only (got %s)" % t.device)
    if t.device.index != device_index:
        raise ValueError("tensor is on %s, communicator on cuda:%d" % (t.device, device_index))
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise ValueError("expected a contiguous float32 tensor")


def _boot_id():
    try:
        with open("/proc/sys/kernel/random/boot_id") as f:
            return f.read().strip()
    except OSError:
        return ""


# ---- fd passing for VMM handles (SCM_RIGHTS over abstract unix sockets) -------------------
def _sock_name(token, rank):
    return "\0b2d-%s-%d" % (token, rank)


def _exchange_fds(group, rank, world, token, my_fd, senders=None):
    """Every rank in ``senders`` (default: all) gives ``my_fd`` to every other rank.
    Returns {sender_rank: received_fd}."""
    senders = list(range(world)) if senders is None else list(senders)
    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    srv.bind(_sock_name(token, rank))
    srv.listen(world + 1)
    dist.barrier(group=group)  # everyone is listening
    if rank in senders:
        for p in range(world):
            if p == rank:
                continue
            c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            c.connect(_sock_name(token, p))
            socket.send_fds(c, [struct.pack("i", rank)], [my_fd])
            c.close()
    got = {}
    expect = len([s for s in senders if s != rank])
    srv.settimeout(60.0)
    for _ in range(expect):
        conn, _addr = srv.accept()
        msg, fds, _flags, _a = socket.recv_fds(conn, 4, 1)
        conn.close()
        got[struct.unpack("i", msg)[0]] = fds[0]
    srv.close()
    dist.barrier(group=group)
    return got


class _Base:
    """Tensor-level calls shared by Communicator and the ranks of a LoopbackGroup."""

    ctx = None
    rank = 0
    world = 1
    device_index = 0

    def allreduce_(self, buf, bucket_idx=0, wire="bf16", scale=None, algo="auto", wait_stream=None,
                   comm_stream=None, phases=_b2d.PHASE_ALL):
        """In-place allreduce of one flat fp32 bucket: buf <- sum_r buf_r * scale (see b2d.h)."""
        _check_tensor(buf, self.device_index)
        scale = (1.0 / self.world) if scale is None else scale
        ws = torch.cuda.current_stream(buf.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        self.ctx.allreduce_bucket(bucket_idx, buf.data_ptr(), buf.numel(), _wire(wire), scale, _algo(algo), ws, cs,
                                  phases)
        return buf

    def sharded_step_(self, grads, params, exp_avg, exp_avg_sq, shard_off, step, lr, betas=(0.9, 0.999),
                      eps=1e-8, weight_decay=0.0, adamw=False, zero_grads=False, wire="bf16", scale=None,
                      slot=0, wait_stream=None, comm_stream=None):
        """reduce-scatter -> partitioned Adam -> parameter all-gather, one kernel (b2d_sharded_step)."""
        for t in (grads, params, exp_avg, exp_avg_sq):
            _check_tensor(t, self.device_index)
        scale = (1.0 / self.world) if scale is None else scale
        ws = torch.cuda.current_stream(grads.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        adam = AdamParams(lr=lr, beta1=betas[0], beta2=betas[1], eps=eps, weight_decay=weight_decay,
                          step=int(step), adamw=int(bool(adamw)), zero_grads=int(bool(zero_grads)))
        self.ctx.sharded_step(slot, grads.data_ptr(), params.data_ptr(), exp_avg.data_ptr(),
                              exp_avg_sq.data_ptr(), grads.numel(), shard_off, _wire(wire), scale, adam, ws, cs)

    def reduce_scatter(self, grads, out, shard_off, wire="fp32", scale=None, slot=0, wait_stream=None,
                       comm_stream=None):
        _check_tensor(grads, self.device_index)
        _check_tensor(out, self.device_index)
        scale = (1.0 / self.world) if scale is None else scale
        ws = torch.cuda.current_stream(grads.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        self.ctx.reduce_scatter(slot, grads.data_ptr(), out.data_ptr(), grads.numel(), shard_off,
                                _wire(wire), scale, ws, cs)
        return out

    # ---- sharded path, overlapped with backward (b2d_owner.cuh) ------------------------------------------
    def register_bucket(self, bucket_id, segs, wire="bf16"):
        """Declare a reduce bucket: ``segs`` = [(flat_off, len, owner_rank)] runs of the flat gradient space."""
        self.ctx.bucket_register(bucket_id, segs, _wire(wire))

    def reduce_to_owner(self, bucket_id, grads, reduced, shard_off, scale=None, zero_grads=True, accumulate=False,
                        nvls=False, wait_stream=None, comm_stream=None, phases=3):
        _check_tensor(grads, self.device_index)
        _check_tensor(reduced, self.device_index)
        scale = (1.0 / self.world) if scale is None else scale
        ws = torch.cuda.current_stream(grads.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        flags = (_b2d.RTO_ZERO_GRADS if zero_grads else 0) | (_b2d.RTO_ACCUMULATE if accumulate else 0) | \
                (_b2d.RTO_NVLS if nvls else 0)
        self.ctx.reduce_to_owner(bucket_id, grads.data_ptr(), reduced.data_ptr(), shard_off, scale, flags, ws, cs, phases)

    def adam_push_(self, params, exp_avg, exp_avg_sq, reduced, shard_off, groups, nvls=False, wait_stream=None,
                   comm_stream=None, phases=6, grad_scale=None):
        """Adam / AdamW on the own shard per parameter group, new parameters pushed into every rank's flat buffer
        (``groups`` = [(lo, hi, dict(lr, beta1, beta2, eps, weight_decay, step, adamw))], empty: push only).
        ``grad_scale``: a one-element fp32 device tensor every gradient is multiplied by first (the clip coefficient
        of ``clip_norm_``; b2d_adam_push_scaled)."""
        _check_tensor(params, self.device_index)
        if grad_scale is not None:
            _check_tensor(grad_scale, self.device_index)
        ws = torch.cuda.current_stream(params.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        gs = [(lo, hi, AdamParams(lr=a["lr"], beta1=a["beta1"], beta2=a["beta2"], eps=a["eps"],
                                  weight_decay=a["weight_decay"], step=int(a["step"]), adamw=int(a["adamw"]), zero_grads=0))
              for lo, hi, a in groups]
        ptr = lambda t: 0 if t is None else t.data_ptr()
        if grad_scale is None:
            self.ctx.adam_push(params.data_ptr(), ptr(exp_avg), ptr(exp_avg_sq), ptr(reduced), params.numel(), shard_off, gs,
                               _b2d.RTO_NVLS if nvls else 0, ws, cs, phases)
        else:
            self.ctx.adam_push(params.data_ptr(), ptr(exp_avg), ptr(exp_avg_sq), ptr(reduced), params.numel(), shard_off, gs,
                               _b2d.RTO_NVLS if nvls else 0, ws, cs, phases, grad_scale_ptr=grad_scale.data_ptr())

    # ---- gradient clipping (b2d_clip.cuh) --------------------------------------------------------------------
    def clip_register(self):
        """Give the clip exchange its region in the arena (once; later calls return the same offset)."""
        return self.ctx.clip_register()

    def clip_norm_(self, x, max_norm, norm_out, coef_out, wait_stream=None, comm_stream=None, phases=3):
        """Global 2-norm of every rank's ``x`` (its reduced-gradient shard; may be empty) into ``norm_out`` and torch's
        clip coefficient ``min(max_norm / (norm + 1e-6), 1)`` into ``coef_out`` (one-element fp32 device tensors), with
        identical bits on every rank.  Asynchronous after ``wait_stream``; ``comm_stream`` waits for the result."""
        _check_tensor(x, self.device_index)
        _check_tensor(norm_out, self.device_index)
        _check_tensor(coef_out, self.device_index)
        ws = torch.cuda.current_stream(x.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        self.ctx.clip_norm(x.data_ptr(), x.numel(), float(max_norm), norm_out.data_ptr(), coef_out.data_ptr(), phases, ws, cs)

    def allgather_(self, buf, shard_off, wait_stream=None, comm_stream=None):
        _check_tensor(buf, self.device_index)
        ws = torch.cuda.current_stream(buf.device) if wait_stream is None else wait_stream
        cs = ws if comm_stream is None else comm_stream
        self.ctx.allgather(buf.data_ptr(), buf.numel(), shard_off, ws, cs)
        return buf

    # ---- synchronised BatchNorm (b2d_syncbn.cuh) -------------------------------------------------------------
    def bn_register(self, layer_id, channels):
        """Give BatchNorm layer ``layer_id`` its exchange region in the arena; returns the region's arena offset.
        Every rank registers the same layers in the same order."""
        off = self.ctx.bn_register(layer_id, channels)
        if getattr(self, "_bn_channels", None) is None:
            self._bn_channels = {}
        self._bn_channels[layer_id] = int(channels)
        return off

    def bn_register_all(self, layers):
        """``layers``: [(layer_id, channels)]; returns their arena offsets."""
        return [self.bn_register(i, c) for i, c in layers]

    def _bn_check(self, layer_id, tensors, dtype=torch.float32):
        c = (getattr(self, "_bn_channels", None) or {}).get(layer_id)
        if c is None:
            raise ValueError("BatchNorm layer %d has not been registered (bn_register)" % layer_id)
        for t in tensors:
            if t is None:
                continue
            if not t.is_cuda or t.device.index != self.device_index:
                raise ValueError("tensor is on %s, communicator on cuda:%d" % (t.device, self.device_index))
            if t.dtype != dtype or not t.is_contiguous() or t.numel() != c:
                raise ValueError("expected a contiguous %s tensor of %d elements, got %s %s" % (dtype, c, t.dtype, tuple(t.shape)))

    def bn_stats_exchange(self, layer_id, mean, invstd, count, eps, momentum, mean_out, invstd_out, counts_out,
                          running_mean=None, running_var=None, stream=None, phases=3):
        """Synchronised BatchNorm statistics (b2d_bn_stats_exchange): this rank's ``mean`` / ``invstd`` over ``count``
        elements per channel (None and 0 for an empty rank) -> the whole batch's ``mean_out`` / ``invstd_out``, every
        rank's count in ``counts_out`` (int32 [W]) and the running statistics updated in place.  On ``stream``
        (default: the current one), without host synchronisation."""
        self._bn_check(layer_id, (mean, invstd, mean_out, invstd_out, running_mean, running_var))
        if counts_out.dtype != torch.int32 or counts_out.numel() != self.world or not counts_out.is_cuda:
            raise ValueError("counts_out must be a CUDA int32 tensor of %d elements" % self.world)
        st = torch.cuda.current_stream(mean_out.device) if stream is None else stream
        ptr = lambda t: 0 if t is None else t.data_ptr()
        self.ctx.bn_stats_exchange(layer_id, ptr(mean), ptr(invstd), count, eps, momentum, ptr(mean_out), ptr(invstd_out),
                                   ptr(counts_out), ptr(running_mean), ptr(running_var), phases, st)

    def bn_grad_exchange(self, layer_id, sum_dy, sum_dy_xmu, sum_dy_out, sum_dy_xmu_out, stream=None, phases=3):
        """Rank-ordered fp32 sums of every rank's ``sum_dy`` / ``sum_dy_xmu`` (None: zeros) into the outputs
        (b2d_bn_grad_exchange)."""
        self._bn_check(layer_id, (sum_dy, sum_dy_xmu, sum_dy_out, sum_dy_xmu_out))
        st = torch.cuda.current_stream(sum_dy_out.device) if stream is None else stream
        ptr = lambda t: 0 if t is None else t.data_ptr()
        self.ctx.bn_grad_exchange(layer_id, ptr(sum_dy), ptr(sum_dy_xmu), ptr(sum_dy_out), ptr(sum_dy_xmu_out), phases, st)

    def arena_tensor(self, numel, dtype=torch.float32):
        t, _ = arena_tensor(self.ctx, numel, dtype, torch.device("cuda", self.device_index))
        return t

    def owns(self, t):
        """Does tensor ``t`` live inside this rank's symmetric arena?"""
        base = getattr(self, "_arena_base", None)
        if base is None:
            p, off = self.ctx.arena_alloc(16)
            self._arena_base = base = p - off
            self._arena_bytes = int(self.ctx.stats()["arena_bytes"])
        return base <= t.data_ptr() and t.data_ptr() + t.numel() * t.element_size() <= base + self._arena_bytes

    def device_barrier(self, stream=None):
        st = torch.cuda.current_stream(torch.device("cuda", self.device_index)) if stream is None else stream
        self.ctx.barrier(st)

    def stats(self):
        return self.ctx.stats()


class Communicator(_Base):
    """One rank of a one-process-per-GPU job.

    ``group`` is an initialised torch.distributed group (gloo or nccl) used ONLY as control
    plane: handle exchange and host barriers.  No gradient byte ever goes through it.
    """

    def __init__(self, rank, world, device_index, arena_bytes, group=None, mem="ipc", timing=False,
                 nvls="auto", timeout_ms=None, max_ctas=None, one_shot_max_bytes=None, chunk_bytes=None,
                 exch_ctas=None):
        if not torch.cuda.is_available():
            raise _b2d.B2DUnavailableError("CUDA is not available: the H100 gradient-sync path has no CPU fallback")
        self.rank, self.world, self.device_index = rank, world, device_index
        self.group = group
        self.mem = mem
        flags = (FLAG_MEM_VMM if mem == "vmm" else 0) | (FLAG_TIMING if timing else 0)
        self.ctx = _b2d.Context(rank, world, device_index, arena_bytes, flags)
        self.nvls = False
        if timeout_ms is not None:
            self.ctx.set_timeout_ms(timeout_ms)
        if max_ctas is not None:
            self.ctx.set_max_ctas(max_ctas)
        if one_shot_max_bytes is not None:
            self.ctx.set_one_shot_max_bytes(one_shot_max_bytes)
        if chunk_bytes is not None:
            self.ctx.set_chunk_bytes(chunk_bytes)
        if exch_ctas is not None:
            self.ctx.set_exch_ctas(exch_ctas)
        if world > 1:
            self._check_single_box()
            self._connect(nvls)

    def _check_single_box(self):
        """The peer mapping is CUDA IPC / VMM fds inside ONE NVSwitch box: say so early (the reference's NCCL
        path would go multi-node; this one cannot)."""
        if self.world > _b2d.MAX_WORLD:
            raise RuntimeError("libb2d drives one NVSwitch domain of at most %d GPUs; got world size %d"
                               % (_b2d.MAX_WORLD, self.world))
        if dist.is_initialized():
            hosts = [None] * self.world
            dist.all_gather_object(hosts, (socket.gethostname(), _boot_id()), group=self.group)
            if len(set(hosts)) != 1:
                raise RuntimeError("libb2d workers must share one host (got %s): multi-node is out of scope"
                                   % sorted(set(h for h, _ in hosts)))

    def _connect(self, nvls):
        if not dist.is_initialized():
            raise RuntimeError("Communicator needs an initialised torch.distributed process group "
                               "(RayStrategy._worker_setup creates it)")
        blobs = [None] * self.world
        dist.all_gather_object(blobs, self.ctx.export_handle(), group=self.group)
        fds = {}
        token = None
        if self.mem == "vmm":
            tok = [uuid.uuid4().hex[:12] if self.rank == 0 else None]
            dist.broadcast_object_list(tok, src=0, group=self.group)
            token = tok[0]
            fds = _exchange_fds(self.group, self.rank, self.world, token + "a", self.ctx.export_fd())
        for p in range(self.world):
            if p != self.rank:
                self.ctx.import_handle(p, blobs[p], fds.get(p))
        for fd in fds.values():
            os.close(fd)
        self.ctx.finalize()
        dist.barrier(group=self.group)
        if self.mem == "vmm" and nvls in ("auto", True, "on"):
            self._try_nvls(token, required=nvls in (True, "on"))

    def _try_nvls(self, token, required):
        flags = [None] * self.world
        dist.all_gather_object(flags, bool(self.ctx.mc_supported()), group=self.group)
        ok = all(flags)
        err = None
        fd = -1
        if ok and self.rank == 0:
            try:
                fd = self.ctx.mc_create()
            except B2DError as e:
                err = str(e)
        st = [err is None and ok]
        dist.broadcast_object_list(st, src=0, group=self.group)
        if not st[0]:
            if required:
                raise RuntimeError("NVLS multicast is not available on this box: %s" % (err or "unsupported"))
            return
        got = _exchange_fds(self.group, self.rank, self.world, token + "m", fd if self.rank == 0 else -1, senders=[0])
        try:
            self.ctx.mc_join(fd if self.rank == 0 else got[0])
            joined = True
        except B2DError as e:
            joined, err = False, str(e)
        allj = [None] * self.world
        dist.all_gather_object(allj, joined, group=self.group)  # also: every device has been added
        if all(allj):
            try:
                self.ctx.mc_bind()
                bound = True
            except B2DError as e:
                bound, err = False, str(e)
            allb = [None] * self.world
            dist.all_gather_object(allb, bound, group=self.group)
            self.nvls = all(allb)
        for f in ([fd] if self.rank == 0 else list(got.values())):
            if f is not None and f >= 0:
                os.close(f)
        if required and not self.nvls:
            raise RuntimeError("NVLS multicast setup failed: %s" % err)

    def bn_register_all(self, layers):
        """Collective: register ``layers`` ([(layer_id, channels)], the same list in the same order on every rank) and
        check over the control plane that every rank placed them at the same arena offsets."""
        offs = super().bn_register_all(layers)
        if self.world > 1 and dist.is_initialized():
            allv = [None] * self.world
            dist.all_gather_object(allv, offs, group=self.group)
            if any(v != offs for v in allv):
                raise RuntimeError("SyncBatchNorm regions landed at different arena offsets on different ranks: every "
                                   "rank must register the same layers in the same order")
        return offs

    def clip_register(self):
        """Collective: register the clip region and check over the control plane that it sits at the same arena offset
        on every rank."""
        off = super().clip_register()
        if self.world > 1 and dist.is_initialized():
            allv = [None] * self.world
            dist.all_gather_object(allv, off, group=self.group)
            if any(v != off for v in allv):
                raise RuntimeError("the clip region landed at different arena offsets on different ranks (%s): every rank "
                                   "must clip at the same step" % allv)
        return off

    def close(self):
        if self.ctx is not None:
            if self.world > 1 and dist.is_initialized():
                try:
                    torch.cuda.synchronize(self.device_index)
                    dist.barrier(group=self.group)
                except Exception:
                    pass
            self.ctx.destroy()
            self.ctx = None


class _LoopRank(_Base):
    def __init__(self, ctx, rank, world, device_index, stream):
        self.ctx, self.rank, self.world, self.device_index, self.stream = ctx, rank, world, device_index, stream


class LoopbackGroup:
    """``world`` ranks in this process; rank r launches on its own stream.  By default all on ``device_index``
    (the whole inter-rank protocol on ONE GPU); ``devices=[...]`` spreads them over several GPUs of the box, and
    with ``mem="vmm"`` + ``nvls=True`` binds an NVLS multicast object over them (needs distinct devices).

    Co-residency: the single-kernel algorithms (one_shot / two_shot) spin on each other, so W ranks x grid CTAs
    x 512 threads must fit the device at once: their per-kernel CTA budget is 128 // W.  The staged algorithms
    never wait for a later launch when their phases are issued phase-major, which is what ``allreduce_`` does."""

    def __init__(self, world, device_index=0, arena_bytes=64 << 20, timing=False, timeout_ms=5000,
                 max_ctas=None, devices=None, mem="ipc", nvls=False):
        if not torch.cuda.is_available():
            raise _b2d.B2DUnavailableError("CUDA is not available")
        self.world = world
        devices = [device_index] * world if devices is None else list(devices)
        flags = (FLAG_TIMING if timing else 0) | (FLAG_MEM_VMM if mem == "vmm" else 0)
        self.ranks = []
        self.nvls = False
        for r in range(world):
            with torch.cuda.device(devices[r]):
                ctx = _b2d.Context(r, world, devices[r], arena_bytes, flags)
                ctx.set_timeout_ms(timeout_ms)
                same_dev = len(set(devices)) == 1
                ctx.set_max_ctas(max_ctas if max_ctas is not None else (max(1, 128 // world) if same_dev else 64))
                self.ranks.append(_LoopRank(ctx, r, world, devices[r], torch.cuda.Stream(device=devices[r])))
        blobs = [rk.ctx.export_handle() for rk in self.ranks]
        for rk in self.ranks:
            for p in range(world):
                if p != rk.rank:
                    rk.ctx.import_handle(p, blobs[p])
            rk.ctx.finalize()
        if nvls:
            if mem != "vmm" or len(set(devices)) != world:
                raise ValueError("NVLS needs mem='vmm' and one distinct device per rank")
            fd = self.ranks[0].ctx.mc_create()
            try:
                for rk in self.ranks:
                    rk.ctx.mc_join(fd)
                for rk in self.ranks:
                    rk.ctx.mc_bind()
            finally:
                os.close(fd)
            self.nvls = True

    def allreduce_(self, bufs, bucket_idx=0, wire="bf16", scale=None, algo="auto", wait_streams=None):
        """bufs[r] is rank r's bucket; all are reduced in place. Asynchronous.  ``wait_streams[r]`` (default: the
        current stream) is the stream whose work produced rank r's bucket."""
        a = self.ranks[0].ctx.plan(bufs[0].numel(), _wire(wire), _algo(algo))[0]
        phase_sets = ((_b2d.PHASE_STAGE, _b2d.PHASE_EXCHANGE, _b2d.PHASE_WRITEBACK)
                      if a in (_b2d.ALGO_STAGED, _b2d.ALGO_NVLS) and self.world > 1 else (_b2d.PHASE_ALL,))
        for ph in phase_sets:      # phase-major: no kernel ever waits for one launched after it
            for r, (rk, b) in enumerate(zip(self.ranks, bufs)):
                ws = torch.cuda.current_stream(b.device) if wait_streams is None else wait_streams[r]
                rk.allreduce_(b, bucket_idx, wire, scale, algo, wait_stream=ws, comm_stream=rk.stream, phases=ph)
        return bufs

    def sharded_step_(self, grads, params, exp_avg, exp_avg_sq, shard_off, **kw):
        for r, rk in enumerate(self.ranks):
            rk.sharded_step_(grads[r], params[r], exp_avg[r], exp_avg_sq[r], shard_off,
                             wait_stream=torch.cuda.current_stream(grads[r].device), comm_stream=rk.stream, **kw)

    def register_bucket(self, bucket_id, segs, wire="bf16"):
        for rk in self.ranks:
            rk.register_bucket(bucket_id, segs, wire)

    def reduce_to_owner(self, bucket_id, grads, reduced, shard_off, **kw):
        """Phase-major over the loopback ranks: stage everywhere, then reduce everywhere."""
        for ph in (1, 2):
            for r, rk in enumerate(self.ranks):
                rk.reduce_to_owner(bucket_id, grads[r], reduced[r], shard_off, phases=ph,
                                   wait_stream=torch.cuda.current_stream(grads[r].device), comm_stream=rk.stream, **kw)

    def adam_push_(self, params, exp_avg, exp_avg_sq, reduced, shard_off, groups, grad_scale=None, **kw):
        """groups[r]: rank r's parameter-group list; grad_scale[r] (optional): rank r's gradient factor.  Phase-major:
        step + push everywhere, then wait everywhere."""
        for ph in (2, 4):
            for r, rk in enumerate(self.ranks):
                rk.adam_push_(params[r], None if exp_avg is None else exp_avg[r], None if exp_avg_sq is None else exp_avg_sq[r],
                              None if reduced is None else reduced[r], shard_off, groups[r], phases=ph,
                              wait_stream=torch.cuda.current_stream(params[r].device), comm_stream=rk.stream,
                              grad_scale=None if grad_scale is None else grad_scale[r], **kw)

    def clip_register(self):
        offs = [rk.clip_register() for rk in self.ranks]
        if len(set(offs)) != 1:
            raise RuntimeError("clip region at different arena offsets: %s" % offs)
        return offs[0]

    def clip_norm_(self, xs, max_norm, norm_outs, coef_outs):
        """Rank r's shard is xs[r].  Phase-major on the ranks' own streams (after the current stream): every partial,
        then every coefficient."""
        for ph in (1, 2):
            for r, rk in enumerate(self.ranks):
                rk.clip_norm_(xs[r], max_norm, norm_outs[r], coef_outs[r], phases=ph,
                              wait_stream=torch.cuda.current_stream(xs[r].device), comm_stream=rk.stream)

    def reduce_scatter(self, grads, outs, shard_off, **kw):
        for r, rk in enumerate(self.ranks):
            rk.reduce_scatter(grads[r], outs[r], shard_off,
                              wait_stream=torch.cuda.current_stream(grads[r].device), comm_stream=rk.stream, **kw)

    def allgather_(self, bufs, shard_off):
        for r, rk in enumerate(self.ranks):
            rk.allgather_(bufs[r], shard_off, wait_stream=torch.cuda.current_stream(bufs[r].device),
                          comm_stream=rk.stream)

    def bn_register(self, layer_id, channels):
        offs = [rk.bn_register(layer_id, channels) for rk in self.ranks]
        if len(set(offs)) != 1:
            raise RuntimeError("SyncBatchNorm region of layer %d at different arena offsets: %s" % (layer_id, offs))
        return offs[0]

    def bn_stats_exchange(self, layer_id, means, invstds, counts, eps, momentum, mean_outs, invstd_outs, counts_outs,
                          running_means=None, running_vars=None):
        """Rank r's arguments are the r-th entries.  Phase-major on the ranks' own streams (after the current stream):
        push everywhere, then combine everywhere."""
        for ph in (1, 2):
            for r, rk in enumerate(self.ranks):
                if ph == 1:
                    rk.stream.wait_stream(torch.cuda.current_stream(torch.device("cuda", rk.device_index)))
                rk.bn_stats_exchange(layer_id, means[r], invstds[r], counts[r], eps, momentum, mean_outs[r], invstd_outs[r],
                                     counts_outs[r], None if running_means is None else running_means[r],
                                     None if running_vars is None else running_vars[r], stream=rk.stream, phases=ph)

    def bn_grad_exchange(self, layer_id, sum_dys, sum_dy_xmus, sum_dy_outs, sum_dy_xmu_outs):
        for ph in (1, 2):
            for r, rk in enumerate(self.ranks):
                if ph == 1:
                    rk.stream.wait_stream(torch.cuda.current_stream(torch.device("cuda", rk.device_index)))
                rk.bn_grad_exchange(layer_id, sum_dys[r], sum_dy_xmus[r], sum_dy_outs[r], sum_dy_xmu_outs[r],
                                    stream=rk.stream, phases=ph)

    def synchronize(self):
        for rk in self.ranks:
            rk.stream.synchronize()

    def join_current_stream(self):
        """Make the caller's current stream(s) wait for every rank's comm stream."""
        for rk in self.ranks:
            torch.cuda.current_stream(torch.device("cuda", rk.device_index)).wait_stream(rk.stream)

    def close(self):
        self.synchronize()
        for rk in self.ranks:
            rk.ctx.destroy()
        self.ranks = []


# ---- f-2: the optimizer step inside backward, bucket by bucket --------------------------------------------------
class InBackwardOptimizer(torch.optim.Optimizer):
    """Wraps the user's SGD / Adam / AdamW: the step of every DDP bucket's parameters runs on the comm stream right
    behind that bucket's allreduce (b2d_bucket_optim, K14) — overlapped with the rest of backward, no separate pass
    over the parameters afterwards — and ``step()`` only advances the step count.  What torch offers as
    ``_hook_then_optimizer`` (optimizer_overlap_hooks.py:131-163).  Same hyper-parameters (lr schedulers act on this
    object), state per parameter in torch's own state-dict layout.  One backward per step (no gradient accumulation);
    one parameter group."""

    def __init__(self, base, hook_state):
        if len(base.param_groups) != 1:
            raise ValueError("optimizer-in-backward supports one parameter group")
        g = base.param_groups[0]
        kernel_args(type(base), base.defaults, g)      # NotFusable (a ValueError) names what K14 does not implement
        self.kind = 0 if type(base) is torch.optim.SGD else 1
        self._base_cls = type(base)
        d = {k: v for k, v in g.items() if k != "params"}
        d["params"] = list(g["params"])
        super().__init__([d], dict(base.defaults))
        self._steps = 0
        self._pstate = {}       # id(param) -> (state1, state2)
        self._tables = {}       # bucket index -> layout signature
        self.applied = 0
        hook_state.in_backward = self

    def _states(self, p):
        st = self._pstate.get(id(p))
        if st is None:
            g = self.param_groups[0]
            # preserve_format: the state's memory order is the parameter's (channels_last weights stay channels_last)
            s1 = torch.zeros_like(p) if (self.kind == 1 or g.get("momentum", 0) != 0) else None
            s2 = torch.zeros_like(p) if self.kind == 1 else None
            st = self._pstate[id(p)] = (s1, s2)
        return st

    def apply_bucket(self, comm, bucket, buf, stream):
        """Called by b200_allreduce_hook right after the bucket's exchange has been enqueued."""
        params, grads = bucket.parameters(), bucket.gradients()
        sig = tuple((p.data_ptr(), g.data_ptr()) for p, g in zip(params, grads))
        idx = bucket.index()
        if self._tables.get(idx) != sig:
            # The kernel walks parameter, gradient and state in MEMORY order.  For a dense parameter the Reducer lays the
            # bucket view out with the parameter's own strides (reducer.cpp initialize_bucket_views, the "gradient layout
            # contract"), so memory order agrees — also for channels_last weights.  (GradBucket.gradients() re-views the same
            # bytes as contiguous tensors of the parameter's sizes: only their data pointers are used here.)
            for p_ in params:
                dense = p_.is_contiguous() or (p_.dim() == 4 and p_.is_contiguous(memory_format=torch.channels_last)) or \
                    (p_.dim() == 5 and p_.is_contiguous(memory_format=torch.channels_last_3d))
                if p_.dtype != torch.float32 or not dense:
                    raise ValueError("optimizer-in-backward needs dense (contiguous or channels_last) fp32 parameters")
            offs = [(g.data_ptr() - buf.data_ptr()) // 4 for g in grads]
            st = [self._states(p) for p in params]
            comm.ctx.optim_register(idx, [p.data_ptr() for p in params],
                                    None if st[0][0] is None else [s[0].data_ptr() for s in st],
                                    None if st[0][1] is None else [s[1].data_ptr() for s in st],
                                    offs, [p.numel() for p in params])
            self._tables[idx] = sig
        a = kernel_args(self._base_cls, self.defaults, self.param_groups[0])
        hp = AdamParams(lr=a["lr"], beta1=a.get("beta1", 0.0), beta2=a.get("beta2", 0.0), eps=a.get("eps", 0.0),
                        weight_decay=a["weight_decay"], step=self._steps + 1, adamw=a.get("adamw", 0), zero_grads=0)
        comm.ctx.bucket_optim(idx, buf.data_ptr(), buf.numel(), self.kind, hp, a.get("momentum", 0.0), stream)
        self.applied += 1

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self._steps += 1      # the updates themselves ran during backward; DDP's finalize already waited for them
        return loss

    def state_dict(self):
        g = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        params = self.param_groups[0]["params"]
        g["params"] = list(range(len(params)))
        state = {}
        for i, p in enumerate(params):
            st = self._pstate.get(id(p))
            if st is None or self._steps == 0:
                continue
            if self.kind == 0:
                if st[0] is not None:
                    state[i] = {"momentum_buffer": st[0].detach().clone()}
            else:
                state[i] = {"step": torch.tensor(float(self._steps)), "exp_avg": st[0].detach().clone(),
                            "exp_avg_sq": st[1].detach().clone()}
        return {"state": state, "param_groups": [g]}

    def load_state_dict(self, sd):
        self.param_groups[0].update({k: v for k, v in sd["param_groups"][0].items() if k != "params"})
        params = self.param_groups[0]["params"]
        for i, st in sd.get("state", {}).items():
            p = params[int(i)]
            s1, s2 = self._states(p)
            if self.kind == 0 and "momentum_buffer" in st and s1 is not None:
                s1.copy_(st["momentum_buffer"])
                self._steps = max(self._steps, 1)     # K14 reads the buffer instead of starting it from the gradient
            elif self.kind == 1:
                s1.copy_(st["exp_avg"]); s2.copy_(st["exp_avg_sq"])
                self._steps = int(st["step"])


# ---- f-3: DDP's per-forward buffer broadcast through the arena -------------------------------------------------
class ArenaBufferSync:
    """State of ``b200_buffer_hook``: the module's buffers (BatchNorm running statistics, counters ...) live in ONE flat
    region of the symmetric arena; "broadcast from rank 0" is then rank 0 pushing that region into every peer's arena
    (b2d_adam_push with no Adam groups and rank 0 owning everything) — one kernel + a one-warp wait per forward, no
    flatten / unflatten copies and no NCCL call.  Replaces DDP._sync_buffers' coalesced ncclBroadcast
    (torch/nn/parallel/distributed.py `_sync_buffers` / `_default_broadcast_coalesced`)."""

    def __init__(self, hook_state, src=0):
        self.hook_state, self.src = hook_state, src
        self.flat = None
        self.calls = 0

    def adopt(self, buffers):
        """Move every buffer into the arena (same values, same tensor objects).  Collective in the sense that every
        rank must do it with the same buffers; called once, lazily, from the hook."""
        comm = self.hook_state.comm
        items = [(n, b) for n, b in buffers.items() if b is not None and b.numel() > 0]
        offs, cur = [], 0
        for _, b in items:
            offs.append(cur)
            cur += -(-b.numel() * b.element_size() // 32) * 32      # 8 fp32 elements: the push kernel's granule
        self.nbytes = max(cur, 32)
        raw = comm.arena_tensor(self.nbytes // 4, torch.float32)
        self.flat = raw
        as_bytes = raw.view(torch.uint8)
        for (_, b), off in zip(items, offs):
            v = as_bytes[off:off + b.numel() * b.element_size()].view(b.dtype).view(b.shape)
            v.copy_(b.data)
            b.data = v
        n = self.nbytes // 4
        self.shard_off = [0] + [n if r >= self.src else 0 for r in range(comm.world)]

    def sync(self, buffers):
        st = self.hook_state
        if self.flat is None:
            self.adopt(buffers)
        cur = torch.cuda.current_stream(self.flat.device)
        st.comm.adam_push_(self.flat, None, None, None, self.shard_off, [], nvls=False, wait_stream=cur, comm_stream=cur)
        self.calls += 1


def b200_buffer_hook(state: ArenaBufferSync, buffers):
    """DDP buffer comm hook (``DistributedDataParallel._register_buffer_comm_hook``): rank 0's buffers reach every rank
    through libb2d's peer stores instead of a coalesced ncclBroadcast."""
    state.hook_state.ensure(next(iter(buffers.values())).device)
    state.sync(buffers)
    return None


def _pg_timeout_ms(group=None):
    """What torch's own collectives of this process group's backend wait before giving up (10 min for NCCL, 30 for gloo;
    torch exposes no getter for a group's individual timeout) — in ms; None keeps the library default of 10 minutes."""
    try:
        backend = dist.get_backend(group)
        return max(int(dist.distributed_c10d._get_default_timeout(backend).total_seconds() * 1000), 60_000)
    except Exception:
        return None


# ---- the DDP communication hook -----------------------------------------------------------
class B200HookState:
    """State object handed to ``DistributedDataParallel.register_comm_hook``.

    wire  "bf16": same arithmetic contract as torch's ``bf16_compress_hook`` (bf16 on the wire,
                  fp32 accumulate, one rounding of the sum); "fp32": contract of DDP's default
                  allreduce (divide, then fp32 SUM).
    The communicator is created lazily on first use *inside the worker*: the strategy object is
    pickled to every actor (ray_launcher.py:240-245) and must not hold CUDA handles before that.
    """

    def __init__(self, wire="fp32", algo="auto", process_group=None, total_grad_elems=None,
                 arena_bytes=None, mem="ipc", timing=False, max_ctas=None, one_shot_max_bytes=None,
                 nvls="auto", stream_priority=-1, timeout_ms=None, chunk_bytes=None, exch_ctas=None,
                 arena_buckets=False, arena_extra_bytes=0):
        self.wire, self.algo = wire, algo
        self.process_group = process_group
        self.total_grad_elems = total_grad_elems
        self.arena_bytes = arena_bytes
        self.mem, self.timing, self.max_ctas, self.nvls = mem, timing, max_ctas, nvls
        self.one_shot_max_bytes = one_shot_max_bytes
        self.stream_priority = stream_priority
        self.timeout_ms, self.chunk_bytes, self.exch_ctas = timeout_ms, chunk_bytes, exch_ctas
        self.arena_buckets, self.arena_extra_bytes = bool(arena_buckets), int(arena_extra_bytes)
        self.comm = None
        self.stream = None
        self.calls = 0
        self.seen = {}   # bucket index -> elements, as last seen (introspection for benchmarks/tests)
        self.in_arena = {}  # bucket index -> does the Reducer's bucket storage live in the symmetric arena?
        self.in_backward = None   # an InBackwardOptimizer, when the optimizer step rides behind every bucket (f-2)
        self._pool = self._pool_alloc = None

    def ensure(self, device):
        if self.comm is not None:
            return
        world = dist.get_world_size(self.process_group) if dist.is_initialized() else 1
        rank = dist.get_rank(self.process_group) if dist.is_initialized() else 0
        nbytes = self.arena_bytes
        if nbytes is None:
            if self.total_grad_elems is None:
                raise ValueError("B200HookState needs total_grad_elems or arena_bytes")
            nbytes = arena_bytes_for(self.total_grad_elems, extra_bytes=self.arena_extra_bytes, wire=self.wire,
                                     arena_buckets=self.arena_buckets)
        timeout_ms = self.timeout_ms
        if timeout_ms is None:
            # the watchdog follows the process group's own timeout (minutes), like torch's NCCL collectives
            timeout_ms = _pg_timeout_ms(self.process_group)
        self.comm = Communicator(rank, world, device.index, nbytes, group=self.process_group, mem=self.mem,
                                 timing=self.timing, nvls=self.nvls, max_ctas=self.max_ctas,
                                 one_shot_max_bytes=self.one_shot_max_bytes, timeout_ms=timeout_ms,
                                 chunk_bytes=self.chunk_bytes, exch_ctas=self.exch_ctas)
        # a high-priority side stream: the comm kernel's few CTAs get SMs as soon as backward frees any
        self.stream = torch.cuda.Stream(device=device, priority=self.stream_priority)

    # ---- f-1: the arena as the Reducer's bucket storage ---------------------------------------------------
    @contextlib.contextmanager
    def allocate_in_arena(self):
        """Everything THIS thread allocates on the communicator's device inside the block comes out of the symmetric
        arena (torch.cuda.MemPool over b2d_pool_alloc).  Wrapped around DistributedDataParallel(...) and around
        Reducer._rebuild_buckets() it makes the flat bucket tensors (reducer.hpp:347-406) peer-addressable, so the
        fp32 exchange runs in place.  Every rank must allocate the same sizes in the same order."""
        if self._pool is None:
            self._pool_alloc = torch.cuda.memory.CUDAPluggableAllocator(_b2d.lib_path(), "b2d_pool_alloc", "b2d_pool_free")
            self._pool = torch.cuda.MemPool(self._pool_alloc.allocator(), use_on_oom=False, no_split=True)
        self.comm.ctx.pool_bind(True)
        try:
            with torch.cuda.use_mem_pool(self._pool, device=self.comm.device_index):
                yield
        finally:
            self.comm.ctx.pool_bind(False)

    def verify_symmetric_buckets(self):
        """Collective, host side: in-place exchange is only valid when every rank's pool allocations landed at the
        same arena offsets.  Compares a digest of (offset, size) over the control plane; on any mismatch the
        in-place path is switched off everywhere (buckets are then staged like any other tensor)."""
        st = self.comm.stats()
        mine = (int(st["pool_allocs"]), int(st["pool_digest"]))
        if self.comm.world > 1 and dist.is_initialized():
            allv = [None] * self.comm.world
            dist.all_gather_object(allv, mine, group=self.process_group)
        else:
            allv = [mine]
        ok = len(set(allv)) == 1
        self.comm.ctx.set_inplace(ok)
        return ok

    def __getstate__(self):
        d = dict(self.__dict__)
        d["comm"], d["stream"], d["_pool"], d["_pool_alloc"], d["in_backward"] = None, None, None, None, None
        return d

    def close(self):
        if self.comm is not None:
            self.comm.close()
            self.comm = None


def b200_allreduce_hook(state: B200HookState, bucket: dist.GradBucket) -> torch.futures.Future[torch.Tensor]:
    """DDP comm hook: one fused libb2d kernel per bucket on a side stream.

    Replaces (ray_lightning/ray_ddp.py:112-116 -> torch DDP) ``bf16_compress_hook``'s
    cast + div + ncclAllReduce + copy (default_hooks.py:57-93,116-134) or, with wire="fp32",
    the default divide + fp32 allreduce (default_hooks.py:18-54).  Called once per bucket in
    bucket order on the autograd thread (reducer.hpp:112-113); returns a CUDA future that the
    Reducer's finalize_backward turns into a stream wait.
    """
    buf = bucket.buffer()
    state.ensure(buf.device)
    comm = state.comm
    cur = torch.cuda.current_stream(buf.device)
    comm.allreduce_(buf, bucket.index(), wire=state.wire, scale=1.0 / comm.world, algo=state.algo,
                    wait_stream=cur, comm_stream=state.stream)
    state.calls += 1
    state.seen[bucket.index()] = buf.numel()
    state.in_arena[bucket.index()] = comm.owns(buf)
    if state.in_backward is not None:
        state.in_backward.apply_bucket(comm, bucket, buf, state.stream)
    fut = torch.futures.Future(devices=[buf.device])
    with torch.cuda.stream(state.stream):
        fut.set_result(buf)
    return fut
