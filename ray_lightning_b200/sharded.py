"""Sharded data parallelism on libb2d: gradients reduced to their owners WHILE backward runs, partitioned
optimizer step, parameters pushed back to every rank.

What ``RayShardedStrategy`` (ray_lightning/ray_ddp_sharded.py:12-13) gets from FairScale —
``ShardedDataParallel`` reducing every gradient bucket to its owner from the autograd hooks and ``OSS``
stepping the owned shard and broadcasting it — is laid out here GPU-first:

* all trainable parameters live in ONE flat fp32 buffer inside the symmetric arena, grouped by owner rank and,
  inside a rank, by optimizer parameter group; gradients accumulate into a second flat buffer (``param.grad``
  are views);
* parameters are cut into *reduce buckets* in the order their gradients become ready (reverse declaration order,
  ``reduce_bucket_mb`` each).  A post-accumulate hook per parameter counts a bucket down; when it is complete its
  segments are staged (cast + scale, gradients zeroed in the same pass) and every owner pulls its share from all
  ranks into its fp32 reduced-gradient shard (b2d_reduce_to_owner: K11 + K12, NVLS when bound) — on the library's
  side streams, overlapped with the rest of backward;
* ``ShardedOptimizer.step()`` is then ONE kernel for Adam/AdamW (b2d_adam_push: Adam on the owned shard in
  registers, per parameter group, new parameters pushed into every rank's flat buffer) + a one-warp wait; any
  other elementwise optimizer runs ``base.step()`` on views of the owned shard and pushes the result;
* optimizer state exists only for the owned shard (the memory saving OSS is used for) and is consolidated to the
  stock ``torch.optim`` state-dict layout for checkpoints, which can be loaded back at ANY world size;
* gradient clipping acts on the owned shards of the averaged gradient, where the gradients are by then:
  ``clip_grad_norm`` computes the global norm on the device (b2d_clip_norm: K18 + K19) and the coefficient is applied
  inside the fused step (or by one multiply before a generic ``base.step()``); ``clip_grad_value`` clamps the shard.
"""
from typing import List

import torch

from ._optim import NotFusable, kernel_args
from .partition import flat_layout, partition_parameters


class FlatShards:
    """Flat parameter / gradient buffers of one module, the owner table and the reduce buckets."""

    def __init__(self, module: torch.nn.Module, comm, rule: str = "fairscale", group_of=None, wire: str = "bf16",
                 reduce_bucket_mb: float = 25.0):
        self.comm = comm
        self.wire = wire
        self.params: List[torch.nn.Parameter] = [p for p in module.parameters() if p.requires_grad]
        if not self.params:
            raise ValueError("module has no trainable parameters")
        dev = self.params[0].device
        if dev.type != "cuda" and not getattr(comm, "is_test_double", False):
            # a real Communicator cannot exist without CUDA; only the host-logic tests' stand-in gets past here
            raise RuntimeError("FlatShards needs the module on a CUDA device (no CPU fallback)")
        if any(p.dtype != torch.float32 for p in self.params):
            raise ValueError("the sharded path keeps fp32 master parameters; got a non-fp32 parameter")
        self.numels = [p.numel() for p in self.params]
        self.owner = partition_parameters(self.numels, comm.world, rule)
        self.group_of = [0] * len(self.params) if group_of is None else list(group_of)
        self.offsets, self.shard_off, self.total = flat_layout(self.numels, self.owner, comm.world, group_of=self.group_of)
        self.flat_params = comm.arena_tensor(self.total)      # symmetric: owners push new values into it
        self.flat_params.zero_()
        self.flat_grads = torch.zeros(self.total, device=dev)
        for p, off, n in zip(self.params, self.offsets, self.numels):
            self.flat_params[off:off + n].copy_(p.data.reshape(-1))
            p.data = self.flat_params[off:off + n].view(p.shape)
            p.grad = self.flat_grads[off:off + n].view(p.shape)
        lo, hi = self.shard_off[comm.rank], self.shard_off[comm.rank + 1]
        self.own = slice(lo, hi)
        self.reduced = torch.zeros(max(hi - lo, 8), device=dev)   # the owner's averaged gradients, fp32
        self._make_buckets(reduce_bucket_mb)

    # ---- reduce buckets: parameters that become ready together --------------------------------------------
    def _make_buckets(self, cap_mb):
        cap = max(int(cap_mb * (1 << 20)) // 4, 1)
        self.bucket_of = [0] * len(self.params)
        self.buckets = []          # list of parameter-index lists, in firing order
        cur, cur_n = [], 0
        for i in reversed(range(len(self.params))):     # autograd produces gradients roughly in reverse declaration order
            padded = -(-self.numels[i] // 8) * 8
            if cur and cur_n + padded > cap:
                self.buckets.append(cur)
                cur, cur_n = [], 0
            cur.append(i)
            cur_n += padded
        if cur:
            self.buckets.append(cur)
        for b, idxs in enumerate(self.buckets):
            for i in idxs:
                self.bucket_of[i] = b
            segs = [(self.offsets[i], -(-self.numels[i] // 8) * 8, self.owner[i]) for i in idxs]
            self.comm.register_bucket(b, segs, self.wire)
        self.bucket_elems = [sum(-(-self.numels[i] // 8) * 8 for i in idxs) for idxs in self.buckets]

    def rebind_grads(self):
        """Point every ``param.grad`` back at its slice of the flat buffer (after a set_to_none)."""
        for p, off, n in zip(self.params, self.offsets, self.numels):
            if p.grad is None or p.grad.data_ptr() != self.flat_grads[off:off + n].data_ptr():
                p.grad = self.flat_grads[off:off + n].view(p.shape)


def _fusable(opt: torch.optim.Optimizer) -> bool:
    """K13 steps Adam / AdamW with up to 8 parameter groups, each of a configuration kernel_args() accepts."""
    if type(opt) not in (torch.optim.Adam, torch.optim.AdamW) or len(opt.param_groups) > 8:
        return False
    try:
        for g in opt.param_groups:
            kernel_args(type(opt), opt.defaults, g)
    except NotFusable:
        return False
    return True


def group_index_of(params, opt):
    """Optimizer parameter group of every parameter in ``params`` (module order)."""
    where = {}
    for gi, g in enumerate(opt.param_groups):
        for p in g["params"]:
            where[id(p)] = gi
    missing = [i for i, p in enumerate(params) if id(p) not in where]
    if missing:
        raise ValueError("%d trainable parameter(s) are in no optimizer parameter group: the sharded path steps every "
                         "parameter it reduces" % len(missing))
    return [where[id(p)] for p in params]


class ShardedOptimizer(torch.optim.Optimizer):
    """Wraps the user's optimizer the way PL wraps it in FairScale ``OSS``: same parameter groups and
    hyper-parameters (lr schedulers act on THIS object), state only for the owned shard, parameters whole again
    after every ``step()``.  ``overlap=True`` reduces every bucket to its owner from autograd hooks during backward."""

    def __init__(self, base: torch.optim.Optimizer, shards: FlatShards, wire: str = "bf16", stream=None, overlap=True,
                 nvls=False):
        self.shards, self.comm, self.wire = shards, shards.comm, wire
        self.stream = stream
        self.nvls = bool(nvls)
        self.fused = _fusable(base)
        self._base_cls = type(base)
        sh = shards
        group_of = group_index_of(sh.params, base)
        if group_of != sh.group_of:
            raise ValueError("FlatShards was laid out for other parameter groups than this optimizer's")
        groups = []
        for g in base.param_groups:
            d = {k: v for k, v in g.items() if k != "params"}
            d["params"] = list(g["params"])
            groups.append(d)
        super().__init__(groups, dict(base.defaults))
        self._steps = 0
        n_own = sh.own.stop - sh.own.start
        dev = sh.flat_params.device
        # the part of the own shard each parameter group covers: contiguous by construction of the flat layout
        self.group_range = []
        for gi in range(len(groups)):
            mine = [(sh.offsets[i], -(-sh.numels[i] // 8) * 8) for i in range(len(sh.params))
                    if sh.owner[i] == self.comm.rank and sh.group_of[i] == gi]
            lo = min((o for o, _ in mine), default=sh.own.start) - sh.own.start
            hi = max((o + n for o, n in mine), default=sh.own.start) - sh.own.start
            self.group_range.append((lo, max(hi, lo)))
        # state_dict numbering: torch numbers parameters group by group
        order = [i for gi in range(len(groups)) for i in range(len(sh.params)) if sh.group_of[i] == gi]
        self._sd_index = {i: k for k, i in enumerate(order)}
        if self.fused:
            self.exp_avg = torch.zeros(max(n_own, 8), device=dev)
            self.exp_avg_sq = torch.zeros(max(n_own, 8), device=dev)
            self._base = None
        else:
            # any elementwise optimizer, run on the owned shard viewed as one flat parameter per group
            self._own_params, bgroups = [], []
            for gi, (lo, hi) in enumerate(self.group_range):
                p = torch.nn.Parameter(sh.flat_params[sh.own][lo:hi], requires_grad=True)
                p.grad = sh.reduced[lo:hi]
                self._own_params.append(p)
                bgroups.append({"params": [p], **{k: v for k, v in groups[gi].items() if k != "params"}})
            self._base = self._base_cls(bgroups)
        # ---- backward overlap -----------------------------------------------------------------------------
        self.overlap = bool(overlap)
        self._left = [len(b) for b in sh.buckets]
        self._next = 0                      # buckets fire in index order on every rank, whatever autograd's order
        self._backward_seen = False         # a backward has reduced since the last step
        self._accumulating = False
        self._discard = False
        self._pass_done = False
        self._grads_clean = True
        self._clip_bufs = None              # (norm, coef) device scalars, once the clip region is registered
        self._coef = None                   # the clip coefficient the next step() applies
        self._clipped = False               # gradients have been clipped since the last step
        self._hooks = []
        if self.overlap:
            for i, p in enumerate(sh.params):
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(i)))

    # ---- the reduce side ---------------------------------------------------------------------------------
    def _make_hook(self, i):
        b = self.shards.bucket_of[i]

        def hook(param):
            self._left[b] -= 1
            if self._left[b] == 0:
                self._fire_ready()
        return hook

    def _streams(self):
        on_gpu = self.shards.flat_params.is_cuda
        cur = torch.cuda.current_stream(self.shards.flat_params.device) if on_gpu else None
        side = self.stream if self.stream is not None else cur
        return cur, side

    def _fire(self, b):
        sh = self.shards
        cur, side = self._streams()
        if b == 0:
            if self._clipped:
                raise RuntimeError("a backward pass started after the gradients were clipped and before optimizer.step(): "
                                   "clip once, right before the step (or call zero_grad() first)")
            if self._backward_seen:
                # gradient accumulation: a second backward without a step in between.  The parameter exchange that
                # normally fences the staging regions between two uses has not happened: fence explicitly, and add.
                self.comm.device_barrier(side)
                self._accumulating = not self._discard
            self._discard = False
            self._backward_seen = True
        self.comm.reduce_to_owner(b, sh.flat_grads, sh.reduced, sh.shard_off, zero_grads=True,
                                  accumulate=self._accumulating, nvls=self.nvls, wait_stream=cur, comm_stream=side)

    def _fire_ready(self):
        while self._next < len(self._left) and self._left[self._next] <= 0:
            self._fire(self._next)
            self._next += 1
        if self._next == len(self._left):      # this backward pass is complete: arm the counters for the next one
            self._left = [len(b) for b in self.shards.buckets]
            self._next = 0
            self._pass_done = True

    def _flush(self):
        """Everything not reduced yet (no overlap, or parameters that received no gradient), in bucket order."""
        if self._pass_done and self._next == 0:
            return
        while self._next < len(self._left):
            self._fire(self._next)
            self._next += 1

    def zero_grad(self, set_to_none: bool = False):
        self._coef, self._clipped = None, False     # a pending clip coefficient belongs to the gradients dropped here
        if self._backward_seen:
            self._discard = True      # gradients reduced since the last step are being thrown away, not accumulated
        if not self._grads_clean:
            self.shards.flat_grads.zero_()
            self._grads_clean = True
        self.shards.rebind_grads()

    # ---- gradient clipping: on the averaged gradient, i.e. the owned shards ------------------------------------------
    def _own_grads(self):
        sh = self.shards
        return sh.reduced[:sh.own.stop - sh.own.start]

    @torch.no_grad()
    def clip_grad_norm(self, max_norm, norm_type=2.0):
        """Collective (every rank calls it at the same step), like FairScale's ``OSS.clip_grad_norm``: the 2-norm of the
        whole averaged gradient over all ranks, returned as a device tensor valid on the current stream.  The gradients
        are scaled by ``min(max_norm / (norm + 1e-6), 1)`` — torch's ``clip_grad_norm_`` — inside the next ``step()``;
        no host synchronisation."""
        if float(norm_type) != 2.0:
            raise ValueError("ShardedOptimizer.clip_grad_norm supports norm_type=2 only (got %r)" % (norm_type,))
        sh = self.shards
        cur, side = self._streams()
        self._flush()                  # every bucket reduced: the shard holds the whole averaged gradient
        if self._clip_bufs is None:
            self.comm.clip_register()  # collective point: compares the region's offset across ranks once
            dev = sh.flat_params.device
            self._clip_bufs = (torch.zeros(1, device=dev), torch.zeros(1, device=dev))
        norm, coef = self._clip_bufs
        # waits for the current stream too: the returned norm of a previous call is read there
        self.comm.clip_norm_(self._own_grads(), max_norm, norm, coef, wait_stream=cur, comm_stream=side)
        self._coef = coef
        self._clipped = True
        if side is not cur:
            cur.wait_stream(side)
        return norm.clone()

    @torch.no_grad()
    def clip_grad_value(self, clip_value):
        """``clip_grad_value_`` on the averaged gradient: element-wise, so clamping every owned shard is the same."""
        v = float(clip_value)
        cur, side = self._streams()
        self._flush()
        if side is not None and side is not cur:
            with torch.cuda.stream(side):
                self._own_grads().clamp_(min=-v, max=v)
            cur.wait_stream(side)
        else:
            self._own_grads().clamp_(min=-v, max=v)
        self._clipped = True

    # ---- the step ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        sh = self.shards
        self._steps += 1
        cur, side = self._streams()
        self._flush()                  # staging zeroes the gradients it ships: after this the flat buffer is clean
        self._grads_clean = True
        if side is not None and side is not cur:
            side.wait_stream(cur)      # the step rewrites parameters and state that work queued before it may still read

        if self.fused:
            groups = []
            for g, (lo, hi) in zip(self.param_groups, self.group_range):
                if hi > lo:
                    groups.append((lo, hi, dict(kernel_args(self._base_cls, self.defaults, g), step=self._steps)))
            clip = {} if self._coef is None else {"grad_scale": self._coef}
            self.comm.adam_push_(sh.flat_params, self.exp_avg, self.exp_avg_sq, sh.reduced, sh.shard_off, groups,
                                 nvls=self.nvls, wait_stream=side, comm_stream=side, **clip)
        else:
            for g, bg in zip(self.param_groups, self._base.param_groups):   # lr schedulers edit OUR groups: mirror them
                for k, v in g.items():
                    if k != "params":
                        bg[k] = v
            if side is not None:
                with torch.cuda.stream(side):
                    if self._coef is not None:
                        self._own_grads().mul_(self._coef)
                    self._base.step()
            else:
                if self._coef is not None:
                    self._own_grads().mul_(self._coef)
                self._base.step()
            self.comm.adam_push_(sh.flat_params, None, None, None, sh.shard_off, [], nvls=self.nvls,
                                 wait_stream=side, comm_stream=side)
        if side is not cur:
            cur.wait_stream(side)
        self._left = [len(b) for b in sh.buckets]
        self._next = 0
        self._backward_seen = False
        self._accumulating = False
        self._discard = False
        self._pass_done = False
        self._coef, self._clipped = None, False
        return loss

    # ---- checkpoints: stock torch.optim layout (SURVEY §8 f-4) -------------------------------------
    def _gather_full(self, own_vec):
        sh = self.shards
        if not hasattr(self, "_gather_buf"):
            self._gather_buf = self.comm.arena_tensor(sh.total)
        buf = self._gather_buf
        buf[sh.own] = own_vec[:sh.own.stop - sh.own.start]
        if buf.is_cuda:
            torch.cuda.current_stream().synchronize()
        self.comm.allgather_(buf, sh.shard_off)
        if buf.is_cuda:
            torch.cuda.current_stream().synchronize()
        return buf.clone()

    def consolidated_state_dict(self):
        """Collective (every rank must call it): the state dict ``type(base)`` would have produced
        had it stepped all parameters on one device."""
        sh = self.shards
        pgs = []
        for gi, g in enumerate(self.param_groups):
            d = {k: v for k, v in g.items() if k != "params"}
            d["params"] = [self._sd_index[i] for i in range(len(sh.params)) if sh.group_of[i] == gi]
            pgs.append(d)
        state = {}
        if self.fused:
            m, v = self._gather_full(self.exp_avg), self._gather_full(self.exp_avg_sq)
            if self._steps > 0:
                for i, (off, n, p) in enumerate(zip(sh.offsets, sh.numels, sh.params)):
                    state[self._sd_index[i]] = {"step": torch.tensor(float(self._steps)),
                                                "exp_avg": m[off:off + n].view(p.shape).cpu(),
                                                "exp_avg_sq": v[off:off + n].view(p.shape).cpu()}
        else:
            n_own = sh.own.stop - sh.own.start
            keys = sorted({k for p in self._own_params for k in self._base.state.get(p, {})})
            for key in keys:
                vals = [self._base.state.get(p, {}).get(key) for p in self._own_params]
                first = next((v for v in vals if v is not None), None)
                if isinstance(first, torch.Tensor) and first.dim() > 0:
                    own_vec = torch.zeros(max(n_own, 8), device=sh.flat_params.device)
                    for (lo, hi), v in zip(self.group_range, vals):
                        if v is not None and hi > lo:
                            own_vec[lo:hi] = v.reshape(-1).float()
                    full = self._gather_full(own_vec)
                    for i, (off, n, p) in enumerate(zip(sh.offsets, sh.numels, sh.params)):
                        state.setdefault(self._sd_index[i], {})[key] = full[off:off + n].view(p.shape).cpu()
                else:
                    # scalars (step counters ...): identical on every rank, also on ranks that own nothing of a group
                    box = first if first is not None else torch.tensor(float(self._steps))
                    for i in range(len(sh.params)):
                        state.setdefault(self._sd_index[i], {})[key] = box.clone() if isinstance(box, torch.Tensor) else box
        return {"state": state, "param_groups": pgs}

    def state_dict(self):
        return self.consolidated_state_dict()

    def load_state_dict(self, sd):
        """Accepts the consolidated layout (written by any previous world size) and keeps the owned slice —
        the resume-with-fewer-workers contract of ray_lightning/tests/test_ddp_sharded.py:118-137."""
        sh = self.shards
        for g, saved in zip(self.param_groups, sd["param_groups"]):
            g.update({k: v for k, v in saved.items() if k != "params"})
        st = {int(k): v for k, v in sd.get("state", {}).items()}
        if not st:
            return
        lo = sh.own.start
        mine = [(i, off, n) for i, (off, n) in enumerate(zip(sh.offsets, sh.numels)) if sh.owner[i] == self.comm.rank]
        for i, _, _ in mine:
            if self._sd_index[i] not in st:
                raise ValueError("optimizer state for parameter %d is missing from the checkpoint" % self._sd_index[i])
        if self.fused:
            for i, off, n in mine:
                s = st[self._sd_index[i]]
                self.exp_avg[off - lo:off - lo + n].copy_(s["exp_avg"].reshape(-1))
                self.exp_avg_sq[off - lo:off - lo + n].copy_(s["exp_avg_sq"].reshape(-1))
            any_state = next(iter(st.values()))
            self._steps = int(any_state["step"])
            return
        # any other elementwise optimizer: every full-size per-parameter state tensor is cut to the owned range of its
        # parameter group; scalars (step counts, ...) are taken as they are
        any_state = next(iter(st.values()))
        for gi, (p, (glo, ghi)) in enumerate(zip(self._own_params, self.group_range)):
            own_state = {}
            members = [(i, off, n) for i, off, n in mine if sh.group_of[i] == gi]
            for key, first in any_state.items():
                if isinstance(first, torch.Tensor) and first.dim() > 0:
                    flat = torch.zeros(max(ghi - glo, 1), device=sh.flat_params.device)
                    for i, off, n in members:
                        v = st[self._sd_index[i]][key]
                        if not isinstance(v, torch.Tensor) or v.numel() != n:
                            raise ValueError("optimizer state %r of parameter %d has an unexpected shape" % (key, self._sd_index[i]))
                        flat[off - lo - glo:off - lo - glo + n].copy_(v.reshape(-1))
                    own_state[key] = flat[:ghi - glo].view_as(p)
                else:
                    own_state[key] = first.clone() if isinstance(first, torch.Tensor) else first
            self._base.state[p] = own_state
        if "step" in any_state:
            self._steps = int(any_state["step"])
